"""The order of additions of the fused product + dot on a sliced-ELL strip, and of CGFused on such a matrix, restated on
the CPU (every operation rounded in the result dtype, as in reduce_order).

dist_apply_kernel<T, 0, SellCol<C>, true> on one part gives interior block b the slices 8 b .. 8 b + 7, warp w of the
block slice 8 b + w, lane l of the warp the stored row perm[32 s + l] of slice s (sell_layout, the strip's sigma).  A live
lane's term is w[r] * y[r] for the y it wrote; a padding lane (perm -1) and a warp past the last slice contribute +0.
The block partial is reduce_order's epilogue (a shuffle tree per warp, then the 8 warp sums in order) and
dot_fold_kernel folds the partials as it does for hybrid ELL."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle
import reduce_order as ro
from vexcl_b200 import _lib as L

SLICES_PER_BLOCK = 8


def sell_layout(row, sigma: int):
    """perm (32 per slice, -1 = padding lane) of the strip VEXB_FMT_SELL builds from these row pointers."""
    row = np.ascontiguousarray(row, np.int64)
    n = row.size - 1
    ns, slots = C.c_size_t(0), C.c_size_t(0)
    L.check(L.lib().vexb_csr_sell_layout(n, row.ctypes.data, 8, sigma, C.byref(ns), C.byref(slots), None, None))
    perm = np.empty(ns.value * 32, np.int32)
    sptr = np.empty(ns.value + 1, np.int32)
    L.check(L.lib().vexb_csr_sell_layout(n, row.ctypes.data, 8, sigma, C.byref(ns), C.byref(slots), perm.ctypes.data, sptr.ctypes.data))
    return perm


def interior_blocks(perm) -> int:
    return -(-(perm.size // 32) // SLICES_PER_BLOCK)


def dot_partials(w, y, perm) -> np.ndarray:
    """The per-block partials: lane terms in storage order, blocks of 8 warps of 32 lanes."""
    G = interior_blocks(perm)
    terms = np.zeros(G * ro.THREADS, y.dtype)
    live = perm >= 0
    idx = np.nonzero(live)[0]
    terms[idx] = np.asarray(w, y.dtype)[perm[idx]] * y[perm[idx]]
    return ro._warps_in_order(ro.warp_tree(terms.reshape(G, SLICES_PER_BLOCK, 32)))


def fused_dot(w, y, perm):
    """The value SpMat.apply_dot leaves in its DeviceScalar on one part of a sliced-ELL strip."""
    return ro.dot_fold(dot_partials(w, y, perm))


def cg_fused(row, col, val, b, iters: int, sms: int, perm, bps: int = 8):
    """solvers.CGFused from x = 0 on one part, float64, on a sliced-ELL strip with layout perm: the sliced-ELL product
    adds a row's products in storage order from +0 (oracle.csr_spmv's bits), the dot in the order above, the r sweep
    and the x / p sweep as reduce_order.  Returns x and the history of rho'."""
    b = np.asarray(b, np.float64)
    x, r = np.zeros_like(b), b.copy()
    p = r.copy()
    rho = ro.reduce_sum(r * r, False, "sweep", sms, bps)
    hist = []
    for _ in range(iters):
        q = oracle.csr_spmv(row, col, val, p)
        pq = fused_dot(p, q, perm)
        r, rho_new = ro.cg_update_r(r, q, rho, pq, sms, bps)
        x, p = ro.cg_update_xp(x, p, r, rho, pq, rho_new)
        rho = rho_new
        hist.append(rho)
    return x, hist
