"""The order of additions of the reduction kernels, the fused dot and the fused CG iteration, restated on the CPU.

Every kernel here rounds each add, subtract, multiply and divide on its own (`__dadd_rn`, `__fadd_rn`, `__ddiv_rn`, ...),
and its grid depends only on n, `reduce.blocks_per_sm` and the SM count.  So its result is predictable bit for bit:
this module adds the same terms in the same order, every operation rounded in the result dtype (numpy rounds each
operation on float64 / float32 arrays to nearest and never fuses), vectorised over accumulators.  It restates
`csrc/reduce.cu` and `csrc/distapply.cu`:

  vexb_reduce_all     sweep path (float or double, one of the five reduce shapes, 32-byte-aligned operands, no
                      scalars, eval.force_interp = 0): reduce_sweep_kernel, U = 2 vectors of E = 32 / sizeof(T)
                      elements per thread and turn, min(max(1, ceil(floor(n / E) / 512)), cap) blocks;
                      interpreter path (everything else): reduce_interp_kernel, U = 4 elements per thread and turn,
                      min(ceil(n / 1024), cap) blocks; cap = SMs * clamp(reduce.blocks_per_sm, 1, 16)
  vexb_reduce_multi   reduce_multi_kernel (vex::CombineReductors): the interpreter geometry, ONE accumulator per
                      thread and reduction taking the thread's U elements of each turn in order
  vexb_cg_update_r    the sweep geometry over r_new^2
  block_finish        per warp a shuffle tree (offsets 16, 8, 4, 2, 1: lane l adds lane l + off), thread 0 adds the
                      8 warp sums in order; the last block: thread t adds partials t, t + 256, ... to +0, then the
                      same trees and the same warp order
  dist_apply_kernel   (fused dot, one part) one row per thread, term w[r] * y[r] (+0 past n), a shuffle tree per warp,
                      then s_part[0] + s_part[1] + ... + s_part[7]; dot_fold_kernel: 1024 threads, thread t adds
                      partials t, t + 1024, ... to +0, a tree per warp, then one tree over the 32 warp sums

SUM_KAHAN compensates only inside a thread's accumulator (take: y = v - c, t = s + y, c = (t - s) - y, s = t); every
merge after that is a plain add, so an accumulator's compensation first matters at its third term.
"""
from __future__ import annotations

import math

import numpy as np

import oracle

THREADS = 256                       # every kernel here runs 256-thread blocks (dot_fold_kernel: one block of 1024)
MAX_BLOCKS_PER_SM = 16
SWEEP_U, INTERP_U = 2, 4
SWEEP_SHAPES = ("copy", "mul", "sqr", "sub", "absdiff")


def lanes(dtype) -> int:
    """E: elements per 32-byte vector access."""
    return 32 // np.dtype(dtype).itemsize


def clamp_bps(bps: int) -> int:
    return min(max(int(bps), 1), MAX_BLOCKS_PER_SM)


def sweep_blocks(n: int, dtype, sms: int, bps: int) -> int:
    """Grid of reduce_sweep_kernel and cg_update_r_kernel (0: n == 0 launches only the identity)."""
    if n == 0:
        return 0
    want = max(1, -(-(n // lanes(dtype)) // 512))
    return min(want, sms * clamp_bps(bps))


def interp_blocks(n: int, sms: int, bps: int) -> int:
    """Grid of reduce_interp_kernel and reduce_multi_kernel (0: n == 0 launches only the identity)."""
    if n == 0:
        return 0
    return min(-(-n // 1024), sms * clamp_bps(bps))


def reduce_path(dtype, shape, force_interp: bool = False) -> str:
    """The kernel vexb_reduce_all picks: "sweep" or "interp".  `shape` is one of SWEEP_SHAPES or None (any other
    expression); operands are taken to be 32-byte aligned, as every vector's slice is."""
    floating = np.dtype(dtype) in (np.dtype(np.float64), np.dtype(np.float32))
    return "sweep" if floating and shape in SWEEP_SHAPES and not force_interp else "interp"


# ------------------------------------------------------------------------------------------------ per-thread folds

def kahan_take(s, c, v):
    """One step of Fold::take for SUM_KAHAN, each operation rounded in the dtype of its operands."""
    y = v - c
    t = s + y
    return t, (t - s) - y


def _take(s, c, v, kahan):
    """Accumulators s (compensations c) take v, in place."""
    if not kahan:
        s += v
        return
    y = v - c
    t = s + y
    np.subtract(t, s, out=c)
    c -= y
    s[...] = t


def _fold_turns(s, c, v, kahan):
    """The grid-stride loop over flat accumulators s, c: turn `it` hands term it * s.size + i to accumulator i; the
    last turn may stop part-way, and the accumulators past its end take nothing."""
    for lo in range(0, v.shape[0], s.shape[0]):
        chunk = v[lo:lo + s.shape[0]]
        _take(s[:chunk.shape[0]], c[:chunk.shape[0]], chunk, kahan)


def sweep_thread_sums(v, kahan: bool, grid: int) -> np.ndarray:
    """reduce_sweep_kernel up to block_finish: each thread's value, shape (grid, 256).

    Thread (b, t) owns acc[u][j] (u < U = 2, j < E).  On turn `it` acc[u][j] takes element iv * E + j with
    iv = it * grid * 256 * U + b * 256 * U + u * 256 + t, while iv < floor(n / E); the last n mod E elements go to
    block 0, element floor(n / E) * E + t into thread t's acc[0][0].  The thread then adds acc[0][0] and the others in
    u-major order (plain adds)."""
    E = lanes(v.dtype)
    n = v.size
    nvec = n // E
    shape = (grid, SWEEP_U, THREADS, E)
    s = np.zeros(shape, v.dtype)
    c = np.zeros(shape, v.dtype)
    _fold_turns(s.reshape(-1, E), c.reshape(-1, E), v[:nvec * E].reshape(nvec, E), kahan)
    tail = n - nvec * E
    if tail:
        _take(s[0, 0, :tail, 0], c[0, 0, :tail, 0], v[nvec * E:], kahan)
    f = s[:, 0, :, 0].copy()
    for u in range(SWEEP_U):
        for j in range(E):
            if u or j:
                f = f + s[:, u, :, j]
    return f


def interp_thread_sums(v, kahan: bool, grid: int) -> np.ndarray:
    """reduce_interp_kernel up to block_finish: acc[k] of thread (b, t) takes element b * 1024 + it * grid * 1024 +
    k * 256 + t on turn `it`; the thread adds acc[0] + acc[1] + acc[2] + acc[3]."""
    s = np.zeros((grid, INTERP_U, THREADS), v.dtype)
    c = np.zeros_like(s)
    _fold_turns(s.reshape(-1), c.reshape(-1), v, kahan)
    f = s[:, 0].copy()
    for k in range(1, INTERP_U):
        f = f + s[:, k]
    return f


def multi_thread_sums(v, kahan: bool, grid: int) -> np.ndarray:
    """reduce_multi_kernel up to block_finish: one accumulator per thread, which takes the elements of the interpreter
    geometry turn by turn, and within a turn u = 0, 1, 2, 3 (element b * 1024 + it * grid * 1024 + u * 256 + t)."""
    s = np.zeros((grid, THREADS), v.dtype)
    c = np.zeros_like(s)
    per_turn = grid * INTERP_U * THREADS
    for lo in range(0, v.size, per_turn):
        chunk = v[lo:lo + per_turn]
        if chunk.size == per_turn:
            vals = chunk.reshape(grid, INTERP_U, THREADS)
            for u in range(INTERP_U):
                _take(s, c, vals[:, u], kahan)
            continue
        for u in range(INTERP_U):                     # the last turn: block b, slot u holds chunk[b * 1024 + u * 256 + t]
            for b in range(grid):
                part = chunk[b * INTERP_U * THREADS + u * THREADS:b * INTERP_U * THREADS + (u + 1) * THREADS]
                _take(s[b, :part.size], c[b, :part.size], part, kahan)
    return s


def first_takes(n: int, dtype, path: str, sms: int, bps: int) -> list:
    """Indices of the elements that element 0's accumulator takes, in the order it takes them."""
    if n == 0:
        return []
    if path == "sweep":
        E = lanes(dtype)
        G = sweep_blocks(n, dtype, sms, bps)
        nvec = n // E
        out = [iv * E for iv in range(0, nvec, G * SWEEP_U * THREADS)]
        return out + ([nvec * E] if n % E else [])
    G = interp_blocks(n, sms, bps)
    step = G * INTERP_U * THREADS
    if path == "interp":
        return list(range(0, n, step))
    return [i for base in range(0, n, step) for i in range(base, min(base + INTERP_U * THREADS, n), THREADS)]


# ------------------------------------------------------------------------------------------------ block_finish

def warp_tree(a) -> np.ndarray:
    """__shfl_down_sync tree over the last axis (32 lanes): for off = 16, 8, 4, 2, 1 lane l adds lane l + off; lane 0's
    value."""
    assert a.shape[-1] == 32
    for off in (16, 8, 4, 2, 1):
        a = a[..., :off] + a[..., off:2 * off]
    return a[..., 0]


def _warps_in_order(w) -> np.ndarray:
    """Thread 0: warp 0's value, then warps 1..7 added in order (last axis)."""
    tot = w[..., 0].copy()
    for k in range(1, w.shape[-1]):
        tot = tot + w[..., k]
    return tot


def block_partials(f) -> np.ndarray:
    """block_finish's first half: each block's partial from its threads' values f (grid, 256)."""
    return _warps_in_order(warp_tree(f.reshape(f.shape[0], THREADS // 32, 32)))


def last_block(parts):
    """block_finish's last block: thread t adds partials t, t + 256, ... to +0, then the warp trees and the warps in
    order."""
    g = np.zeros(THREADS, parts.dtype)
    for lo in range(0, parts.size, THREADS):
        chunk = parts[lo:lo + THREADS]
        g[:chunk.size] = g[:chunk.size] + chunk
    return _warps_in_order(warp_tree(g.reshape(THREADS // 32, 32)))


def block_finish(f):
    return last_block(block_partials(f))


# ------------------------------------------------------------------------------------------------ whole reductions

def reduce_sum(v, kahan: bool = False, path: str = "sweep", sms: int = 132, bps: int = 8):
    """SUM (kahan=False) or SUM_KAHAN of the evaluated terms v (their dtype is the result dtype) through one slot of
    vexb_reduce_all (path "sweep" or "interp") or vexb_reduce_multi (path "multi")."""
    v = np.ascontiguousarray(v)
    typ = v.dtype.type
    if v.size == 0:
        return typ(0)
    if path == "sweep":
        f = sweep_thread_sums(v, kahan, sweep_blocks(v.size, v.dtype, sms, bps))
    elif path == "interp":
        f = interp_thread_sums(v, kahan, interp_blocks(v.size, sms, bps))
    elif path == "multi":
        f = multi_thread_sums(v, kahan, interp_blocks(v.size, sms, bps))
    else:
        raise ValueError(path)
    return typ(block_finish(f))


def host_fold(values):
    """Reductor's fold of the slots' values (slot order, in the result dtype) when no peer group or communicator
    combines them."""
    acc = values[0]
    for v in values[1:]:
        acc = acc + v
    return acc


def slots_sum(v, part, kahan: bool = False, path: str = "sweep", sms: int = 132, bps: int = 8):
    """The sum over several slots of one device: each slot reduces its own slice part[k]:part[k + 1], then
    host_fold."""
    v = np.ascontiguousarray(v)
    return host_fold([reduce_sum(v[part[k]:part[k + 1]], kahan, path, sms, bps) for k in range(len(part) - 1)])


def sum_depth(n: int, dtype, path: str, sms: int, bps: int) -> int:
    """Largest number of additions between a term and the result (adds to the initial +0 included)."""
    if n == 0:
        return 0
    E = lanes(dtype)
    if path == "sweep":
        G = sweep_blocks(n, dtype, sms, bps)
        takes = -(-n // E // (G * SWEEP_U * THREADS)) + (1 if n % E else 0)
        merge = SWEEP_U * E - 1
    else:
        G = interp_blocks(n, sms, bps)
        turns = -(-n // (G * INTERP_U * THREADS))
        takes, merge = (turns, INTERP_U - 1) if path == "interp" else (turns * INTERP_U, 0)
    trees = 2 * (5 + THREADS // 32 - 1)
    return takes + merge + trees + -(-G // THREADS)


# ------------------------------------------------------------------------------------------------ fused dot

def dot_partials(w, y) -> np.ndarray:
    """dist_apply_kernel's per-block partials of dot(w, y) on one part: block b covers rows 256 b ..."""
    n = y.size
    G = -(-n // THREADS)
    terms = np.zeros(G * THREADS, y.dtype)
    terms[:n] = w * y
    return _warps_in_order(warp_tree(terms.reshape(G, THREADS // 32, 32)))


def dot_fold(parts):
    """dot_fold_kernel: thread t of 1024 adds partials t, t + 1024, ... to +0; a tree per warp; warp 0's tree over the
    32 warp sums."""
    g = np.zeros(1024, parts.dtype)
    for lo in range(0, parts.size, 1024):
        chunk = parts[lo:lo + 1024]
        g[:chunk.size] = g[:chunk.size] + chunk
    return parts.dtype.type(warp_tree(warp_tree(g.reshape(32, 32))))


def fused_dot(w, y):
    """The value SpMat.apply_dot leaves in its DeviceScalar on one part, from the y the product wrote."""
    return dot_fold(dot_partials(np.asarray(w, y.dtype), y))


# ------------------------------------------------------------------------------------------------ CG

def cg_update_r(r, q, rho, pq, sms: int, bps: int = 8):
    """vexb_cg_update_r: alpha = rho / pq; r_new = r - alpha q; rho' = (r_new, r_new) in the sweep geometry."""
    typ = r.dtype.type
    alpha = typ(rho) / typ(pq)
    rn = r - alpha * q
    return rn, reduce_sum(rn * rn, False, "sweep", sms, bps)


def cg_update_xp(x, p, r, rho, pq, rho_new):
    """vexb_cg_update_xp: beta = rho' / rho; x += alpha p; p = r + beta p (r already updated)."""
    typ = x.dtype.type
    alpha, beta = typ(rho) / typ(pq), typ(rho_new) / typ(rho)
    return x + alpha * p, r + beta * p


def cg_fused(row, col, val, b, iters: int, sms: int, bps: int = 8):
    """solvers.CGFused from x = 0 on one part, float64: r = b, p = r, rho = (r, r) (sweep geometry); each iteration
    q = A p (the hybrid-ELL product equals oracle.csr_spmv bit for bit in float64 on one part), pq = the fused dot
    (p, q), then the r sweep and the x / p sweep.  Returns x and the history of rho'."""
    b =np.asarray(b, np.float64)
    x, r = np.zeros_like(b), b.copy()
    p = r.copy()
    rho = reduce_sum(r * r, False, "sweep", sms, bps)
    hist = []
    for _ in range(iters):
        q = oracle.csr_spmv(row, col, val, p)
        pq = fused_dot(p, q)
        r, rho_new = cg_update_r(r, q, rho, pq, sms, bps)
        x, p = cg_update_xp(x, p, r, rho, pq, rho_new)
        rho = rho_new
        hist.append(rho)
    return x, hist


def laplacian(n: int):
    """7-point Laplacian on an n^3 grid with the Dirichlet neighbours dropped (symmetric positive definite), as
    int64 row / col and float64 val, columns sorted."""
    N = n ** 3
    i = np.arange(N, dtype=np.int64)
    coord = (i // (n * n), (i // n) % n, i % n)
    offsets, inside = [], []
    for ax, step in ((0, n * n), (1, n), (2, 1)):
        offsets += [-step, step]
        inside += [coord[ax] > 0, coord[ax] < n - 1]
    offsets.append(0)
    inside.append(np.ones(N, bool))
    order = np.argsort(offsets)
    offsets = np.array(offsets)[order]
    inside = np.stack(inside, axis=1)[:, order]
    cols = i[:, None] + offsets[None, :]
    vals = np.where(offsets == 0, 6.0, -1.0)[None, :].repeat(N, axis=0)
    row = np.zeros(N + 1, np.int64)
    np.cumsum(inside.sum(axis=1), out=row[1:])
    return row, cols[inside], vals[inside], N


def error_bound(v, depth: int) -> float:
    """(depth - 1) u sum |v_i|: the bound on a sum whose terms each pass through at most `depth` additions."""
    u = np.finfo(v.dtype).eps / 2
    return (depth - 1) * float(u) * math.fsum(np.abs(v.astype(np.float64)))
