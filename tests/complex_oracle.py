"""Reference product of complex sparse matrices, the spmv_ops_impl<std::complex<T>, std::complex<T>> of the reference's
examples/complex_spmv.cpp with every product and sum rounded on its own:

    for each stored entry a + bi of row i, in storage order, with x_c = xr + xi i:
        tr = a*xr - b*xi;  s_re = s_re + tr
        ti = a*xi + b*xr;  s_im = s_im + ti
    y_i = alpha * s  or  y_i + alpha * s        (per component, alpha real)

in the real type of val (float64 for complex128, float32 for complex64).  x and y are real arrays of interleaved
(re, im) pairs, the bytes of std::complex<T>[].  Vectorised over rows, one pass per position within a row, as
tests/block_oracle.py is.  Test infrastructure: the product never imports it.
"""
from __future__ import annotations

import numpy as np

from block_oracle import block_stencil


def real_of(val) -> type:
    return np.float64 if np.asarray(val).dtype == np.complex128 else np.float32


def zsr_spmv(ptr, col, val, x, y=None, alpha=1.0, append=False) -> np.ndarray:
    """y (=|+=) alpha * A x.  val: nnz complex values; x: 2*ncols real values; y: 2*nrows real values.  Returns a new flat
    real array.  With no stored entry, y += A*x leaves y as it is (as vexb_spmv does)."""
    val = np.asarray(val)
    dt = np.dtype(real_of(val))
    a, b = val.real.astype(dt), val.imag.astype(dt)
    ptr = np.asarray(ptr, dtype=np.int64)
    ptr = ptr - ptr[0]
    col = np.asarray(col, dtype=np.int64)
    n = ptr.size - 1
    xz = np.asarray(x, dtype=dt).reshape(-1, 2)
    xr, xi = xz[:, 0], xz[:, 1]
    y0 = np.zeros(2 * n, dt) if y is None else np.array(y, dtype=dt).reshape(2 * n)
    if append and ptr[-1] == 0:
        return y0
    sr, si = np.zeros(n, dt), np.zeros(n, dt)
    width = np.diff(ptr)
    for k in range(int(width.max()) if n else 0):
        rows = np.nonzero(width > k)[0]
        j = ptr[rows] + k
        c = col[j]
        tr = a[j] * xr[c] - b[j] * xi[c]
        ti = a[j] * xi[c] + b[j] * xr[c]
        sr[rows] = sr[rows] + tr
        si[rows] = si[rows] + ti
    res = np.empty(2 * n, dt)
    res[0::2] = dt.type(alpha) * sr
    res[1::2] = dt.type(alpha) * si
    return y0 + res if append else res


def as_blocks(val) -> np.ndarray:
    """Each entry a + bi as the real 2x2 block [[a, -b], [b, a]]: the same matrix for tests/block_oracle.py and vexb_bspmv."""
    val = np.asarray(val)
    dt = real_of(val)
    a, b = val.real.astype(dt), val.imag.astype(dt)
    return np.stack([np.stack([a, -b], axis=1), np.stack([b, a], axis=1)], axis=1)


def complex_stencil(nx: int, dtype=np.complex128, seed: int = 0):
    """7-point stencil on an nx^3 grid (the pattern of block_oracle.block_stencil), values seeded U(-1, 1) + U(-1, 1) i.
    Returns int32 ptr and col and the complex values."""
    ptr, col, _ = block_stencil(nx, 1, np.float64, seed)
    rng = np.random.default_rng(seed)
    val = (rng.uniform(-1.0, 1.0, col.size) + 1j * rng.uniform(-1.0, 1.0, col.size)).astype(dtype)
    return ptr, col, val
