"""The stencil kernels' launch geometry, window and writes, restated on the CPU.

`csrc/stencil.cu` computes, per output of a device slice,

    y[i] (=|+=) alpha * sum_{k < width} s[k] * X(i + k - center)        (stencil_kernel, stencil_pipe_kernel)
    y[i] (=|+=) alpha * f(&X(i))                                         (vexb_stencil_op, body f supplied at run time)

with X(j) = x[j] inside the slice, the caller's `left` / `right` halo outside it, and the slice's first / last element
where no halo is given.  Every product and sum is rounded on its own in the slice's precision, in tap order, then the
kernel multiplies by alpha and adds y on append.  `oracle/stencil.py::convolve` is that arithmetic over a whole vector;
this module adds what a single call of the C ABI sees:

  stencil_launch     wlen = 1024 + ceil8(width) window positions per 1024-output tile,
                     smem = (st_pad(wlen) + 1 + ceil8(width)) * sizeof(T), st_pad(p) = p + p / 8;
                     smem > 200 KB is refused (VEXB_ERR_UNSUPPORTED), smem > 48 KB raises the attribute first;
                     smem2 = (2 * (st_pad(wlen) + 1) + ceil8(width)) * sizeof(T) for the two windows of the pipe kernel,
                     which runs only when stencil.kernel == 0, smem2 <= 100 KB and there are more tiles than resident blocks;
                     a tile is `inside` (direct loads, no clamps) when b0 - center >= 0 and b0 - center + wlen <= n
  vexb_stencil_op    256 outputs per block, a shared window of 256 + WIDTH - 1 positions starting at b0 - CENTER:
                     position j < 0 from left[CENTER + j] (x[0] without a left halo), j >= n from
                     right[min(j - n, RHALO - 1)] (x[n - 1] without a right halo); then v = alpha * f(X),
                     y = append ? y + v : v
  exchange_halos     (api.py stencil.exchange_halos, include/vexcl/stencil.hpp detail::stencil_halos) a slice that is not
                     at the start of the vector gets a left halo of `center` elements, one not at the end a right halo of
                     `width - 1 - center`; where the vector runs out they are padded with x[0] and x[n - 1], also when a
                     neighbouring slice is shorter than the halo or empty

The operator bodies used by the tests are restated in `BODIES`: C source for NVRTC (compiled with --fmad=false) next to
the same operations on numpy arrays of the slice's dtype, which round each operation like C does.  They use only +, -,
*, fmin, fmax and constants exact in T, cast to T, so that the device result is exactly defined.
"""
from __future__ import annotations

import numpy as np

from oracle.stencil import convolve

ST_B = 1024                          # outputs per stencil_kernel tile (128 threads x 8 consecutive outputs)
OP_B = 256                           # outputs per vexb_stencil_op block
SMEM_LIMIT = 200 * 1024              # bytes of dynamic shared memory stencil_kernel may ask for
SMEM_DEFAULT = 48 * 1024             # above this the kernel's attribute is raised before the launch
PIPE_LIMIT = 100 * 1024              # bytes of the pipe kernel's two windows and taps
OP_MAX_WIDTH = 4096                  # widest operator vexb_stencil_operator_register accepts

__all__ = ["convolve", "ceil8", "st_pad", "smem_bytes", "pipe_smem_bytes", "accepted", "attribute_path", "pipe_fits",
           "uses_pipe", "tiles", "tile_inside", "window", "finish", "convolve_slice", "op_window", "apply_operator", "BODIES",
           "slice_halos", "convolve_slices"]


def ceil8(width: int) -> int:
    return (width + 7) & ~7


def st_pad(p: int) -> int:
    """One pad word per 8 window positions, so the stride-8 reads of neighbouring lanes fall in distinct banks."""
    return p + (p >> 3)


def wlen(width: int) -> int:
    return ST_B + ceil8(width)


def smem_bytes(width: int, dtype) -> int:
    return (st_pad(wlen(width)) + 1 + ceil8(width)) * np.dtype(dtype).itemsize


def pipe_smem_bytes(width: int, dtype) -> int:
    return (2 * (st_pad(wlen(width)) + 1) + ceil8(width)) * np.dtype(dtype).itemsize


def accepted(width: int, dtype) -> bool:
    return smem_bytes(width, dtype) <= SMEM_LIMIT


def attribute_path(width: int, dtype) -> bool:
    return smem_bytes(width, dtype) > SMEM_DEFAULT


def pipe_fits(width: int, dtype) -> bool:
    return pipe_smem_bytes(width, dtype) <= PIPE_LIMIT


def tiles(n: int) -> int:
    return -(-n // ST_B)


def uses_pipe(width: int, n: int, dtype, kernel: int, per_sm: int, sms: int) -> bool:
    """Whether stencil_launch runs stencil_pipe_kernel; per_sm: resident blocks per SM after stencil.blocks_per_sm."""
    return kernel == 0 and pipe_fits(width, dtype) and tiles(n) > max(per_sm, 1) * sms


def tile_inside(tile: int, n: int, width: int, center: int) -> bool:
    b0 = tile * ST_B
    return b0 - center >= 0 and b0 - center + wlen(width) <= n


def window(x, center: int, rhalo: int, lo: int, hi: int, left=None, right=None) -> np.ndarray:
    """X(j) for j in [lo, hi), as both kernels stage it from one slice and its optional halos."""
    x = np.asarray(x)
    n = x.size
    j = np.arange(lo, hi, dtype=np.int64)
    out = x[np.clip(j, 0, n - 1)]
    if left is not None:
        m = j < 0
        out[m] = np.asarray(left)[center + j[m]]
    if right is not None and rhalo > 0:
        m = j >= n
        out[m] = np.asarray(right)[np.minimum(j[m] - n, rhalo - 1)]
    return out


def finish(acc, alpha, y, append):
    """The kernels' write: v = alpha * acc rounded in T, then y + v on append."""
    v = acc.dtype.type(alpha) * acc
    return np.asarray(y, dtype=acc.dtype) + v if append else v


def convolve_slice(s, center: int, x, left=None, right=None, y=None, alpha=1.0, append=False) -> np.ndarray:
    """One vexb_stencil_apply call on one slice: taps added in order to +0, then alpha, then y on append."""
    s = np.asarray(s)
    x = np.asarray(x)
    n, width = x.size, s.size
    ext = window(x, center, width - 1 - center, -center, n + width - 1 - center, left, right)
    acc = np.zeros(n, dtype=x.dtype)
    for k in range(width):
        acc = acc + s[k] * ext[k:k + n]
    return finish(acc, alpha, y, append)


def op_window(x, block: int, width: int, center: int, left=None, right=None) -> np.ndarray:
    """The shared window of vexb_stencil_op's block `block`, literally: 256 + WIDTH - 1 positions from b0 - CENTER."""
    x = np.asarray(x)
    n, rhalo, b0 = x.size, width - 1 - center, block * OP_B
    win = np.empty(OP_B + width - 1, dtype=x.dtype)
    for p in range(win.size):
        j = b0 - center + p
        if j < 0:
            win[p] = left[center + j] if left is not None else x[0]
        elif j >= n:
            win[p] = right[min(j - n, rhalo - 1)] if (right is not None and rhalo > 0) else x[n - 1]
        else:
            win[p] = x[j]
    return win


def apply_operator(body: str, width: int, center: int, x, left=None, right=None, y=None, alpha=1.0,
                   append=False) -> np.ndarray:
    """One vexb_stencil_operator_apply call with the registered BODIES[body], vectorised over the slice."""
    x = np.asarray(x)
    n = x.size
    ext = window(x, center, width - 1 - center, -center, n + width - 1 - center, left, right)
    f = BODIES[body][1]
    acc = f(lambda k: ext[center + k:center + k + n], x.dtype.type, width, center)
    return finish(np.asarray(acc, dtype=x.dtype), alpha, y, append)


def _sum_squares(X, T, width, center):
    s = None
    for k in range(-center, width - center):
        t = X(k) * X(k)
        s = T(0) + t if s is None else s + t
    return s


# name -> (C body of `T stencil_oper(const T *X)`, the same operations on numpy arrays; X(k) is the slice shifted by k)
BODIES = {
    "second_difference": ("return X[-1] - (T)2 * X[0] + X[1];",
                          lambda X, T, w, c: X(-1) - T(2) * X(0) + X(1)),
    "forward": ("return (T)0.5 * (X[3] - X[0]) + X[1] * X[2];",
                lambda X, T, w, c: T(0.5) * (X(3) - X(0)) + X(1) * X(2)),
    "backward": ("return X[0] - (T)0.75 * X[-1] + (T)0.25 * X[-3] * X[-2];",
                 lambda X, T, w, c: X(0) - T(0.75) * X(-1) + T(0.25) * X(-3) * X(-2)),
    "min_max": ("return fmax(X[-1], X[1]) - fmin(X[0], (T)0.5 * X[1]);",
                lambda X, T, w, c: np.fmax(X(-1), X(1)) - np.fmin(X(0), T(0.5) * X(1))),
    "sum_squares": ("T s = (T)0;\nfor (int k = -CENTER; k <= RHALO; ++k) s = s + X[k] * X[k];\nreturn s;",
                    _sum_squares),
}


def slice_halos(x, bounds, center: int, width: int):
    """The halos the exchange gives each slice [bounds[k], bounds[k + 1]): a list of (left or None, right or None)."""
    x = np.asarray(x)
    n, rhalo, nparts = x.size, width - 1 - center, len(bounds) - 1
    out = []
    for k in range(nparts):
        start, size = int(bounds[k]), int(bounds[k + 1] - bounds[k])
        left = right = None
        if nparts > 1 and width > 1 and size:
            if start > 0 and center:
                g = np.arange(start - center, start)
                left = np.where(g < 0, x[0], x[np.maximum(g, 0)]).astype(x.dtype)
            if start + size < n and rhalo:
                g = np.arange(start + size, start + size + rhalo)
                right = np.where(g >= n, x[n - 1], x[np.minimum(g, n - 1)]).astype(x.dtype)
        out.append((left, right))
    return out


def convolve_slices(s, center: int, x, bounds, y=None, alpha=1.0, append=False) -> np.ndarray:
    """stencil.apply over several slices: the halo exchange, then one convolve_slice per slice, concatenated."""
    x = np.asarray(x)
    s = np.asarray(s)
    parts = []
    for k, (left, right) in enumerate(slice_halos(x, bounds, center, s.size)):
        a, b = int(bounds[k]), int(bounds[k + 1])
        if a < b:
            parts.append(convolve_slice(s, center, x[a:b], left, right, None if y is None else np.asarray(y)[a:b],
                                        alpha, append))
    return np.concatenate(parts) if parts else np.zeros(0, dtype=x.dtype)
