"""Reference product of block sparse matrices (B x B values), the loop of the reference's
tests/sparse_matrices.cpp custom_values case (:271-281) for any B:

    for each stored block j of block row i, in storage order, and each row r of the block:
        t = a_r0 * x_0;  t = t + a_r1 * x_1;  ...;  s_r = s_r + t
    y_i = alpha * s  or  y_i + alpha * s

in the dtype of val, every product and sum rounded on its own.  Vectorised over block rows, one pass per
position within a row.  Test infrastructure, like the oracle package: the product never imports it.
"""
from __future__ import annotations

import numpy as np


def bsr_spmv(ptr, col, val, x, y=None, alpha=1.0, append=False) -> np.ndarray:
    """y (=|+=) alpha * A x.  ptr/col count block rows/columns; val: (nnzb, B, B); x: ncols*B values; y: nrows*B values.
    Returns a new flat array.  With no stored block, y += A*x leaves y as it is (as vexb_spmv does)."""
    val = np.asarray(val)
    dt = val.dtype
    B = val.shape[1]
    ptr = np.asarray(ptr, dtype=np.int64)
    ptr = ptr - ptr[0]
    col = np.asarray(col, dtype=np.int64)
    n = ptr.size - 1
    xb = np.asarray(x, dtype=dt).reshape(-1, B)
    y0 = np.zeros(n * B, dt) if y is None else np.array(y, dtype=dt).reshape(n * B)
    if append and ptr[-1] == 0:
        return y0
    s = np.zeros((n, B), dt)
    width = np.diff(ptr)
    for k in range(int(width.max()) if n else 0):
        rows = np.nonzero(width > k)[0]
        j = ptr[rows] + k
        a, xv = val[j], xb[col[j]]
        t = a[:, :, 0] * xv[:, None, 0]
        for q in range(1, B):
            t = t + a[:, :, q] * xv[:, None, q]
        s[rows] = s[rows] + t
    res = (dt.type(alpha) * s).reshape(n * B)
    return y0 + res if append else res


def block_stencil(nx: int, B: int, dtype=np.float64, seed: int = 0):
    """7-point stencil on an nx^3 grid of block rows (columns ascending: z-1, y-1, x-1, self, x+1, y+1, z+1).  Off-diagonal
    blocks are seeded U(-1, 1); diagonal blocks U(-1, 1) + 7B on their diagonal, so every row is diagonally dominant.
    Returns int32 ptr and col and val of shape (nnzb, B, B)."""
    n = nx ** 3
    i = np.arange(n, dtype=np.int64)
    x, y, z = i % nx, (i // nx) % nx, i // (nx * nx)
    offs = ((-nx * nx, z > 0), (-nx, y > 0), (-1, x > 0), (0, np.ones(n, bool)),
            (1, x < nx - 1), (nx, y < nx - 1), (nx * nx, z < nx - 1))
    ok = np.stack([m for _, m in offs], axis=1)                          # (n, 7)
    cols = i[:, None] + np.array([d for d, _ in offs], np.int64)[None, :]
    col = cols[ok].astype(np.int32)
    is_diag = np.broadcast_to(np.arange(7) == 3, ok.shape)[ok]
    ptr = np.zeros(n + 1, np.int32)
    ptr[1:] = np.cumsum(ok.sum(axis=1))
    rng = np.random.default_rng(seed)
    val = rng.uniform(-1.0, 1.0, (col.size, B, B)).astype(dtype)
    val[is_diag] += (7 * B * np.eye(B)).astype(dtype)
    return ptr, col, val


def expand(ptr, col, val, chunk: int = 1 << 20):
    """The same matrix as scalar CSR (nrows*B rows): row r of block row i holds a_rq at column col*B + q, blocks in
    storage order.  Returns int64 row, int32 col and val in its own dtype (built chunk by chunk: the 128^3 stencil with
    B = 4 expands to 233 M entries)."""
    val = np.asarray(val)
    B = val.shape[1]
    ptr = np.asarray(ptr, dtype=np.int64)
    ptr = ptr - ptr[0]
    col = np.asarray(col, dtype=np.int64)
    n, nnzb = ptr.size - 1, int(ptr[-1])
    width = np.diff(ptr)
    row = np.zeros(n * B + 1, np.int64)
    row[1:] = np.cumsum(np.repeat(width * B, B))
    ecol = np.empty(nnzb * B * B, np.int32)
    evals = np.empty(nnzb * B * B, val.dtype)
    blk_all = np.repeat(np.arange(n), width)                 # block row of each stored block
    r = np.arange(B)
    for j0 in range(0, nnzb, chunk):
        j = np.arange(j0, min(j0 + chunk, nnzb))
        blk = blk_all[j]
        # entry (block j, row r, column q) goes to row[blk*B] + r*width*B + (j - ptr[blk])*B + q
        dst = (row[blk * B] + (j - ptr[blk]) * B)[:, None, None] + (r[None, :, None] * (width[blk] * B)[:, None, None]) \
            + r[None, None, :]
        ecol[dst.ravel()] = np.broadcast_to((col[j] * B)[:, None, None] + r[None, None, :], dst.shape).ravel()
        evals[dst.ravel()] = val[j].reshape(-1)
    return row, ecol, evals
