"""CSR strips at the edges of their tiles, row modes and persistent loops.

A CSR strip (VEXB_FMT_CSR) is multiplied by one of seven kernels (`spmv.kernel`):

  0 csr_stream_kernel, 1 csr_pipe_kernel, 2 csr_direct_kernel, 6 csr_window_kernel -- CTA tiles (<= spmv.tile_nnz
    entries, <= spmv.tile_rows rows).  A tile holding one row longer than tile_nnz is added by 256 threads striding by
    256, a shuffle tree per warp and the 8 warp sums in order; any other tile adds each row in storage order by one
    thread if cnt <= 12 nr, else by a 32-lane shuffle tree;
  3 csr_scalar_kernel -- one thread per row, storage order;
  4 csr_warp_kernel, 5 csr_ring_kernel -- warp tiles (<= 256 entries, <= 256 rows).  A row longer than 256 entries is
    added by a 32-lane tree, any other row by G = 1, 4, 8 or 32 lanes (warp_tile_group: cnt <= 6 nr, 24 nr, 64 nr);
 -1 the strip's own choice: 3 for short even rows, else 4.

Products and sums are rounded separately (no contraction), so `csr_kernel_ref`, which restates the tile cut and each
kernel's order of additions in numpy, predicts y bit for bit, in float64 and float32, on one part and on the boundary
and ghost strips of 2 and 3 parts (copy-engine halo, row-mapped strips).  The shapes aim at the tile cut (tile_nnz and
tile_rows, +- 1), the long-row branches (tile_nnz, tile_nnz + 1, 256, 257 entries), the row-mode thresholds (12 nr,
6 nr, 24 nr, 64 nr, each + 1), empty rows and strips, a rectangular strip whose last x window would pass the end of x,
every tile parameter, and matrices long enough for every persistent CTA and warp to wrap its ring many times."""
import ctypes as C

import numpy as np
import pytest

import oracle
import vexcl_b200 as vx
from vexcl_b200 import _lib as L

# ------------------------------------------------------------------------------------------------ references

WARP_TILE = 256                                 # kWarpTileNnz = kWarpTileRows
CTA_THREADS = 256


def clamp_tiles(tile_nnz, tile_rows):
    """The tile size build() uses for spmv.tile_nnz / spmv.tile_rows."""
    return max(64, min(tile_nnz, 8192)) & ~3, max(32, min(tile_rows, 4096)) & ~3


def csr_tiles(row, tile_nnz=2048, tile_rows=512, clamp=True):
    """First row of every tile, then n: build()'s cut.  A tile takes rows while it holds <= tile_nnz entries and
    <= tile_rows rows; a row that does not fit alone is a tile of its own."""
    row = np.asarray(row, np.int64)
    n = row.size - 1
    if clamp:
        tile_nnz, tile_rows = clamp_tiles(tile_nnz, tile_rows)
    starts, r = [], 0
    while r < n:
        k = int(np.searchsorted(row, row[r] + tile_nnz, side="right")) - 1      # last e with row[e] - row[r] <= tile_nnz
        e = min(n, r + tile_rows, k)
        if e == r:
            e = r + 1
        starts.append(r)
        r = e
    starts.append(n)
    return np.array(starts, np.int64)


def default_kernel(row):
    """build()'s choice for a strip: thread per row (3) when the mean row is <= 8 and the longest <= 2 mean + 2."""
    n = row.size - 1
    cnt = np.diff(np.asarray(row, np.int64))
    mean = float(row[-1] - row[0]) / n if n else 0.0
    maxw = int(cnt.max()) if n else 0
    return 3 if mean <= 8.0 and maxw <= 2.0 * mean + 2.0 else 4


def row_lanes(kernel, row, tile_nnz=2048, tile_rows=512):
    """Lanes that add each row: 1 (storage order), 4, 8, 32 (a shuffle tree over lanes striding by G), or 256 (the
    CTA long-row fold)."""
    row = np.asarray(row, np.int64)
    n = row.size - 1
    if kernel == -1:
        kernel = default_kernel(row)
    if kernel == 3:
        return np.ones(n, np.int64)
    if kernel in (4, 5):
        t = csr_tiles(row, WARP_TILE, WARP_TILE)
        nr, cnt = np.diff(t), row[t[1:]] - row[t[:-1]]
        g = np.where(cnt > WARP_TILE, 32, np.where(cnt <= 6 * nr, 1, np.where(cnt <= 24 * nr, 4, np.where(cnt <= 64 * nr, 8, 32))))
    else:
        tn, tr = clamp_tiles(tile_nnz, tile_rows)
        t = csr_tiles(row, tn, tr)
        nr, cnt = np.diff(t), row[t[1:]] - row[t[:-1]]
        g = np.where(cnt > tn, CTA_THREADS, np.where(cnt <= 12 * nr, 1, 32))
    return np.repeat(g, nr)


def lane_sums(start, length, prod, G):
    """(rows, G): lane l of each row adds the row's entries l, l + G, l + 2G, ... in order, from 0.  Rows are taken
    longest first, so every step works on the rows that still have entries."""
    order = np.argsort(-length, kind="stable")
    a, n_ = start[order], length[order]
    P = np.zeros((a.size, G), prod.dtype)
    lanes = np.arange(G)
    steps = -(-int(n_[0]) // G) if a.size else 0
    for k in range(steps):
        m = int(np.count_nonzero(n_ > k * G))
        off = k * G + lanes
        ok = off[None, :] < n_[:m, None]
        sub = P[:m]
        sub[ok] = sub[ok] + prod[(a[:m, None] + off[None, :])[ok]]
    out = np.empty_like(P)
    out[order] = P
    return out


def shuffle_tree(P):
    """__shfl_down_sync over the last axis: p[:off] += p[off:2 off] for off = G/2, ..., 1; lane 0 holds the sum."""
    P = P.copy()
    off = P.shape[-1] // 2
    while off:
        P[..., :off] = P[..., :off] + P[..., off:2 * off]
        off //= 2
    return P[..., 0]


def csr_kernel_ref(kernel, row, col, val, x, dtype, tile_nnz=2048, tile_rows=512):
    """The y = A*x that CSR kernel `kernel` computes, bit for bit: every product and sum rounded in `dtype`."""
    dt = np.dtype(dtype).type
    row = np.asarray(row, np.int64)
    n = row.size - 1
    col = np.asarray(col, np.int64)
    prod = (np.asarray(val).astype(dt) * np.asarray(x).astype(dt)[col]).astype(dt)
    cnt = np.diff(row)
    g = row_lanes(kernel, row, tile_nnz, tile_rows)
    s = np.zeros(n, dt)
    for G in np.unique(g):
        r = np.nonzero(g == G)[0]
        if G == CTA_THREADS:
            warp = shuffle_tree(lane_sums(row[r], cnt[r], prod, CTA_THREADS).reshape(r.size, CTA_THREADS // 32, 32))
            tot = warp[:, 0]
            for w in range(1, CTA_THREADS // 32):
                tot = tot + warp[:, w]
            s[r] = tot
        else:
            s[r] = shuffle_tree(lane_sums(row[r], cnt[r], prod, int(G)))
    return s


def store_ref(y0, s, alpha, append, dtype):
    """store_y: dtype(alpha s), then dtype(y0 + that) when appending."""
    dt = np.dtype(dtype).type
    v = (dt(alpha) * s.astype(dt)).astype(dt)
    return (np.asarray(y0).astype(dt) + v).astype(dt) if append else v


# ------------------------------------------------------------------------------------------------ generators

SEP_CTA, SEP_WARP = 2100, 300          # a row longer than a CTA / warp tile: ends the tile before it, is one of its own


def alt(nr, a, b):
    return [a if i % 2 == 0 else b for i in range(nr)]


def from_lengths(lengths, m=None, seed=0, dtype=np.float64, idx=np.int64, band=None):
    """CSR with the given row lengths: columns uniform on [0, m) (or within +-band of row i * m / n), sorted within a
    row, repeats allowed; values of mixed magnitude so that the order of a sum shows in its last bits."""
    cnt = np.asarray(lengths, np.int64)
    n = cnt.size
    m = m or max(n, 64)
    rng = np.random.default_rng(seed)
    row = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=row[1:])
    nnz = int(row[-1])
    rid = np.repeat(np.arange(n), cnt)
    if band is None:
        col = rng.integers(0, m, nnz)
    else:
        col = np.clip(rid * m // n + rng.integers(-band, band + 1, nnz), 0, m - 1)
    col = col[np.lexsort((col, rid))]
    val = (rng.random(nnz) - 0.5) * 2.0 ** rng.integers(-5, 6, nnz)
    return row.astype(idx), col.astype(idx), val.astype(dtype), m


def rectangular(dtype=np.float64, idx=np.int64):
    """3000 x 2047 (m odd: no multiple of 2 or 4), a band along the scaled diagonal; the last rows reach column m - 1,
    so the last tile's x window, rounded up to 16 bytes, would pass the end of x."""
    n, m = 3000, 2047
    rng = np.random.default_rng(11)
    lengths = rng.integers(0, 30, n)
    lengths[-5:] = 9
    row, col, val, _ = from_lengths(lengths, m, seed=12, dtype=dtype, idx=idx, band=15)
    col = col.astype(np.int64)
    col[int(row[-2]):] = np.arange(m - 9, m)                       # last row: columns m - 9 .. m - 1
    return row, col.astype(idx), val, m


def mixed_lengths(n, seed, long_every=2000, long_len=(2049, 5000), runs=20, run_len=600):
    """Short rows, medium rows, long rows (> a CTA tile) and runs of empty rows longer than a tile's rows."""
    rng = np.random.default_rng(seed)
    w = np.where(rng.random(n) < 0.75, rng.integers(0, 12, n), rng.integers(12, 60, n))
    w[rng.integers(0, n, max(1, n // long_every))] = rng.integers(long_len[0], long_len[1], max(1, n // long_every))
    w[rng.integers(0, n, max(1, n // 500))] = rng.choice([256, 257, 1024, 1025, 1500, 2048], max(1, n // 500))
    for s in rng.integers(0, max(1, n - run_len), runs):
        w[s:s + run_len] = 0
    return w


CASES = {
    # tiles of exactly tile_nnz and tile_nnz + 1 entries (the second row then starts the next, storage-order, tile);
    # exactly tile_rows and tile_rows + 1 rows
    "tile_cut": ([SEP_CTA] + [2040, 8] + [1] * 60 + [SEP_CTA] + [2040, 9] + [1] * 60) * 8
                + [SEP_CTA] + [3] * 512 + [SEP_CTA] + [3] * 513 + [SEP_CTA] + [2] * 10,
    # a long row first and last, tile_nnz (normal tile) against tile_nnz + 1 (long-row branch), two long rows back to
    # back, empty rows on both sides of a long row; the same at the warp tile's 256 / 257
    "long_rows": [2049, 5, 7, 2048, 3, 0, 0, 2200, 0, 0, 4, 2100, 2500, 6, 256, 1, 257, 0, 0, 300, 0, 0, 9, 255, 258, 3000],
    # CTA tiles at cnt = 12 nr and 12 nr + 1 (100 rows)
    "cta_modes": ([SEP_CTA] + alt(100, 2, 22) + [SEP_CTA] + alt(99, 2, 22) + [23]) * 4 + [SEP_CTA],
    # warp tiles at cnt = 6 nr, 24 nr, 64 nr and each + 1; 42 rows of 6 (a natural 6 nr tile); rows of 256 and 257
    "warp_modes": ([SEP_WARP] + alt(32, 1, 11) + [SEP_WARP] + alt(31, 1, 11) + [12]
                   + [SEP_WARP] + alt(8, 4, 44) + [SEP_WARP] + alt(7, 4, 44) + [45]
                   + [SEP_WARP] + [60, 64, 68] + [SEP_WARP] + [60, 64, 69]
                   + [SEP_WARP] + [6] * 42 + [SEP_WARP] + [256] + [SEP_WARP] + [257]) * 3 + [SEP_WARP],
    "one_row": [5],
    "no_entry": [0] * 50,
    # tiles of empty rows only (CTA: 512 rows, warp: 256 rows)
    "empty_tiles": [3] * 5 + [0] * 1100 + [3] * 5 + [0] * 300 + [2],
    "rectangular": None,
}


def case_matrix(name, dtype=np.float64, idx=np.int64):
    if name == "rectangular":
        return rectangular(dtype, idx)
    lengths = CASES[name]
    return from_lengths(lengths, 7 if name == "one_row" else None, seed=len(lengths), dtype=dtype, idx=idx)


# ------------------------------------------------------------------------------------------------ CPU self-checks

@pytest.mark.parametrize("name", ["tile_cut", "long_rows", "cta_modes", "warp_modes", "empty_tiles", "rectangular"])
def test_storage_order_ref_is_csr_spmv(name):
    row, col, val, m = case_matrix(name)
    x = oracle.uniform_real(5, m) - 0.5
    want = oracle.csr_spmv(row.astype(np.int64), col.astype(np.int64), val, x)
    assert np.array_equal(csr_kernel_ref(3, row, col, val, x, np.float64), want)
    # every row added in storage order: the G = 1 path of the tile kernels gives the same bits
    g = row_lanes(0, row)
    s = csr_kernel_ref(0, row, col, val, x, np.float64)
    assert np.array_equal(s[g == 1], want[g == 1])


def _cut(lengths, tn=2048, tr=512, clamp=True):
    row = np.concatenate([[0], np.cumsum(lengths)])
    return list(csr_tiles(row, tn, tr, clamp))


def test_csr_tiles_at_the_cut():
    assert _cut([2040, 8] + [1] * 60) == [0, 2, 62]                    # exactly tile_nnz: one tile
    assert _cut([2040, 9] + [1] * 60) == [0, 1, 62]                    # tile_nnz + 1: the second row starts a tile
    assert _cut([3] * 512) == [0, 512] and _cut([3] * 513) == [0, 512, 513]
    assert _cut([2049]) == [0, 1] and _cut([2048, 1]) == [0, 1, 2] and _cut([1, 2049, 1]) == [0, 1, 2, 3]
    assert _cut([0] * 600) == [0, 512, 600]
    assert _cut([6] * 43, 256, 256) == [0, 42, 43]                     # warp tiles: 252 entries, then 258 > 256
    assert _cut([1] * 257, 256, 256) == [0, 256, 257]
    assert _cut([256, 1, 257, 0], 256, 256) == [0, 1, 2, 3, 4]         # a row over the tile stays alone, even before an empty row
    # clamps: 64..8192 and 32..4096, each rounded down to a multiple of 4
    assert clamp_tiles(10, 5) == (64, 32) and clamp_tiles(10000, 5000) == (8192, 4096) and clamp_tiles(1027, 514) == (1024, 512)
    assert _cut([30] * 5, 10, 10) == [0, 2, 4, 5]                      # tile_nnz 10 is 64: two rows of 30 per tile
    assert _cut([1] * 70, 2048, 33) == [0, 32, 64, 70]                 # tile_rows 33 is 32


def test_row_lanes_at_the_thresholds():
    row = np.concatenate([[0], np.cumsum(CASES["warp_modes"])])
    g = row_lanes(4, row)
    t = csr_tiles(row, 256, 256)
    got = [(int(t[i + 1] - t[i]), int(row[t[i + 1]] - row[t[i]]), int(g[t[i]])) for i in range(11)]
    assert got == [(1, 300, 32), (32, 192, 1), (1, 300, 32), (32, 193, 4), (1, 300, 32), (8, 192, 4), (1, 300, 32),
                   (8, 193, 8), (1, 300, 32), (3, 192, 8), (1, 300, 32)]
    assert int(g[t[11]]) == 32                                         # 3 rows, 193 entries: > 64 nr
    row = np.concatenate([[0], np.cumsum(CASES["cta_modes"])])
    g, t = row_lanes(0, row), csr_tiles(row)
    assert [int(g[t[i]]) for i in range(5)] == [CTA_THREADS, 1, CTA_THREADS, 32, CTA_THREADS]
    assert [int(row[t[i + 1]] - row[t[i]]) for i in (1, 3)] == [1200, 1201]


def test_shuffle_tree_is_the_pairwise_sum():
    """A 32-entry row on a 32-lane tree (one entry per lane) against the pairwise sum written out by hand, in float32."""
    rng = np.random.default_rng(3)
    differs = 0
    for trial in range(20):
        p = ((rng.random(32) - 0.5) * 2.0 ** rng.integers(-8, 9, 32)).astype(np.float32)
        row, col, x = np.array([0, 32]), np.arange(32), np.ones(32, np.float32)
        got = csr_kernel_ref(0, row, col, p, x, np.float32)[0]             # CTA tile, 1 row of 32 > 12 nr: 32 lanes
        t = [p[i] for i in range(32)]
        for off in (16, 8, 4, 2, 1):
            t = [np.float32(t[i] + t[i + off]) for i in range(off)]
        assert got == t[0] and got.dtype == np.float32
        seq = np.float32(0)
        for v in p:
            seq = np.float32(seq + v)
        differs += got != seq
    assert differs > 0                                                      # the tree is not storage order


def test_cta_long_row_fold_by_hand():
    """A 600-entry row in a CTA long-row tile: thread t adds entries t, t + 256, t + 512; each warp's tree; then the 8
    warp sums in order."""
    rng = np.random.default_rng(4)
    p = ((rng.random(600) - 0.5) * 2.0 ** rng.integers(-8, 9, 600)).astype(np.float32)
    row, col, x = np.array([0, 600]), np.arange(600), np.ones(600, np.float32)
    got = csr_kernel_ref(0, row, col, p, x, np.float32, tile_nnz=512)[0]
    th = []
    for t in range(256):
        s = np.float32(0)
        for j in range(t, 600, 256):
            s = np.float32(s + p[j])
        th.append(s)
    red = []
    for w in range(8):
        v = th[32 * w:32 * w + 32]
        for off in (16, 8, 4, 2, 1):
            v = [np.float32(v[i] + v[i + off]) for i in range(off)]
        red.append(v[0])
    tot = red[0]
    for w in range(1, 8):
        tot = np.float32(tot + red[w])
    assert got == tot


def test_store_ref_rounds_twice():
    y0, s = np.array([1.0], np.float32), np.array([2.0 ** -24 * 3], np.float32)
    assert store_ref(y0, s, 0.5, True, np.float32)[0] == np.float32(1.0) + np.float32(0.5 * s[0])
    assert store_ref(y0, s, -1.0, False, np.float32)[0] == -s[0]


def test_default_kernel_rule():
    assert default_kernel(np.array([0, 8, 16])) == 3 and default_kernel(np.array([0, 8, 17])) == 4     # mean 8 / 8.5
    assert default_kernel(np.array([0, 1, 2, 3, 10])) == 3                 # max 7 = 2 mean + 2
    assert default_kernel(np.array([0, 1, 2, 3, 11])) == 4                 # max 8 > 2 * 2.75 + 2


# ------------------------------------------------------------------------------------------------ GPU helpers

KERNELS = [-1, 0, 1, 2, 3, 4, 5, 6]
CTA_KERNELS, WARP_KERNELS = (0, 1, 2, 6), (4, 5)
OPS = {"set": (1.0, False), "add": (1.0, True), "sub": (-1.0, True), "half_append": (0.5, True)}
DEFAULTS = {"spmv.kernel": -1, "spmv.tile_nnz": 2048, "spmv.tile_rows": 512, "spmv.xwin": 2048, "spmv.stages": 4,
            "spmv.ring_stages": 3, "spmv.ring_warps": 8, "spmv.ctas_per_sm": 0}


@pytest.fixture
def params(built):
    """vx.set_param, with every CSR parameter back at its default afterwards."""
    try:
        yield vx.set_param
    finally:
        for k, v in DEFAULTS.items():
            vx.set_param(k, v)


def family(kernel, row):
    """Kernels that add in the same order share one reference."""
    if kernel == -1:
        kernel = default_kernel(np.asarray(row, np.int64))
    return "cta" if kernel in CTA_KERNELS else "warp" if kernel in WARP_KERNELS else "seq"


class Refs:
    """csr_kernel_ref per order family, computed once."""

    def __init__(self, row, col, val, x, dtype, tile_nnz=2048, tile_rows=512):
        self.args = (row, col, val, x, dtype, tile_nnz, tile_rows)
        self.row, self.memo = row, {}

    def __call__(self, kernel):
        f = family(kernel, self.row)
        if f not in self.memo:
            self.memo[f] = csr_kernel_ref({"cta": 0, "warp": 4, "seq": 3}[f], *self.args)
        return self.memo[f]


def assert_same(got, want, what):
    assert got.dtype == want.dtype, what
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} rows differ, first {bad[:8].tolist()}"


def run_ops(ctx, A, X, Y0):
    """Every op through SpMat.apply; y starts from Y0 each time."""
    x, out = vx.vector(ctx, X), {}
    for op, (alpha, append) in OPS.items():
        y = vx.vector(ctx, Y0)
        A.apply(x, y, alpha, append)
        out[op] = y.read()
    return out


def check_kernels(ctx, A, row, col, val, m, dtype, seed, kernels=KERNELS, tile_nnz=2048, tile_rows=512, set_kernel=vx.set_param,
                  fails=()):
    """Every kernel and op against csr_kernel_ref; kernels of one family also against each other."""
    n = row.size - 1
    rng = np.random.default_rng(seed)
    X = (rng.random(m) - 0.5).astype(dtype)
    Y0 = (rng.random(n) - 0.5).astype(dtype)
    refs = Refs(row, col, val, X, dtype, tile_nnz, tile_rows)
    seen = {}
    for k in kernels:
        set_kernel("spmv.kernel", k)
        if k in fails:
            with pytest.raises(L.VexbError):
                run_ops(ctx, A, X, Y0)
            continue
        got = run_ops(ctx, A, X, Y0)
        s = refs(k)
        for op, (alpha, append) in OPS.items():
            assert_same(got[op], store_ref(Y0, s, alpha, append, dtype), f"kernel {k}, {op}")
        f = "cta" if k in CTA_KERNELS else "warp" if k in WARP_KERNELS else None
        if f:
            if f in seen:
                for op in OPS:
                    assert np.array_equal(got[op], seen[f][op]), (k, op)
            seen.setdefault(f, got)
    set_kernel("spmv.kernel", -1)
    return X, refs


def spmat(ctx, row, col, val, m, fmt=vx.FMT_CSR):
    return vx.SpMat(ctx, row.size - 1, m, row, col, val, fmt)


# ------------------------------------------------------------------------------------------------ 1. shapes

SHAPE_CASES = [(c, np.float64, np.int64) for c in CASES] + [(c, np.float32, np.int64) for c in CASES] \
    + [("long_rows", np.float64, np.int32), ("warp_modes", np.float32, np.int32), ("tile_cut", np.float64, np.int32)]


@pytest.mark.gpu
@pytest.mark.parametrize("name, dtype, idx", SHAPE_CASES, ids=[f"{c}-{np.dtype(d).name}-{np.dtype(i).name}" for c, d, i in SHAPE_CASES])
def test_shapes(ctx1, params, name, dtype, idx):
    row, col, val, m = case_matrix(name, dtype, idx)
    A = spmat(ctx1, row, col, val, m)
    info = A.info().loc
    assert info.fmt == vx.FMT_CSR
    assert info.n_tiles == len(csr_tiles(row)) - 1
    X, refs = check_kernels(ctx1, A, row, col, val, m, dtype, seed=len(name), set_kernel=params)
    # the generated row function of y = z + A*x: one launch, storage order
    n = row.size - 1
    Z = (np.random.default_rng(7).random(n) - 0.5).astype(dtype)
    x, z, y = vx.vector(ctx1, X), vx.vector(ctx1, Z), vx.vector(ctx1, n, dtype)
    n0 = vx.launch_count()
    y.assign(z + A * x)
    assert vx.launch_count() - n0 == 1
    assert_same(y.read(), (Z + refs(3)).astype(dtype), "y = z + A*x")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_direct_kernel_long_rows_below_2048(ctx1, params, dtype):
    """csr_direct_kernel at spmv.tile_nnz < 2048: rows of tile_nnz + 1 .. 2048 entries take the long-row branch (they
    used to take the normal one and write their products past the kernel's shared memory)."""
    lengths = ([SEP_CTA, 1500, 3, 1025, 1024, 7, 2048, 2049, 1023, 0, 1500] + [5] * 300) * 3
    row, col, val, m = from_lengths(lengths, 5000, seed=21, dtype=dtype)
    for tn in (64, 1024, 1500):
        params("spmv.tile_nnz", tn)
        A = spmat(ctx1, row, col, val, m)
        params("spmv.tile_nnz", 2048)
        assert A.info().loc.tile_nnz == tn & ~3
        check_kernels(ctx1, A, row, col, val, m, dtype, seed=tn, kernels=(2, 0), tile_nnz=tn, set_kernel=params)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_nothing_past_y(ctx1, params, dtype):
    """vexb_spmv on a strip made by vexb_csr_create, y longer than n: the entries past n keep their sentinel."""
    row, col, val, m = from_lengths(mixed_lengths(5000, 31, long_every=700), seed=32, dtype=dtype)
    n, tail = row.size - 1, 77
    rng = np.random.default_rng(33)
    X = (rng.random(m) - 0.5).astype(dtype)
    sentinel = np.full(n + tail, 12345.5, dtype)
    lib, k = L.lib(), ctx1.local[0]
    h = C.c_void_p()
    L.check(lib.vexb_csr_create(ctx1.devs[k], ctx1.streams[k], n, m, row.ctypes.data, 8, col.ctypes.data, 8, val.ctypes.data,
                                L.F64 if dtype == np.float64 else L.F32, L.FMT_CSR, C.byref(h)))
    try:
        refs = Refs(row, col, val, X, dtype)
        x = vx.vector(ctx1, X)
        for kern in KERNELS:
            params("spmv.kernel", kern)
            y = vx.vector(ctx1, sentinel)
            want = sentinel[:n]
            for alpha, append in OPS.values():
                L.check(lib.vexb_spmv(ctx1.devs[k], ctx1.streams[k], h, x.bufs[k], y.bufs[k], alpha, int(append)))
                want = store_ref(want, refs(kern), alpha, append, dtype)
            got = y.read()
            assert np.all(got[n:] == 12345.5), kern
            assert_same(got[:n], want, f"kernel {kern}")
    finally:
        L.check(lib.vexb_spmat_destroy(h))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_misaligned_x_falls_back_to_warp_tiles(ctx1, params, dtype):
    """x one element past a 16-byte boundary: the window kernel cannot bulk-copy its slice and runs the warp tiles."""
    row, col, val, m = from_lengths(mixed_lengths(6000, 41, long_every=900), seed=42, dtype=dtype)
    n = row.size - 1
    rng = np.random.default_rng(43)
    X = (rng.random(m) - 0.5).astype(dtype)
    refs = Refs(row, col, val, X, dtype)
    assert not np.array_equal(refs(0), refs(4))                   # the two orders give different bits here
    lib, k = L.lib(), ctx1.local[0]
    h = C.c_void_p()
    L.check(lib.vexb_csr_create(ctx1.devs[k], ctx1.streams[k], n, m, row.ctypes.data, 8, col.ctypes.data, 8, val.ctypes.data,
                                L.F64 if dtype == np.float64 else L.F32, L.FMT_CSR, C.byref(h)))
    try:
        xs = vx.vector(ctx1, np.concatenate([np.zeros(1, dtype), X]))
        shifted = C.c_void_p(xs.bufs[k].value + np.dtype(dtype).itemsize)
        aligned = vx.vector(ctx1, X)
        for kern, xp, want in ((6, shifted, refs(4)), (4, shifted, refs(4)), (6, aligned.bufs[k], refs(0))):
            params("spmv.kernel", kern)
            y = vx.vector(ctx1, n, dtype)
            L.check(lib.vexb_spmv(ctx1.devs[k], ctx1.streams[k], h, xp, y.bufs[k], 1.0, 0))
            assert_same(y.read(), want, f"kernel {kern}")
    finally:
        L.check(lib.vexb_spmat_destroy(h))


# ------------------------------------------------------------------------------------------------ 2. parameters

_sweep = {}


def sweep_matrix(dtype):
    key = np.dtype(dtype).name
    if key not in _sweep:
        w = mixed_lengths(30000, 51, long_every=2500, long_len=(8193, 9500), runs=2, run_len=4100)
        w[[100, 5000, 15000]] = [1500, 70, 65]
        _sweep[key] = from_lengths(w, seed=52, dtype=dtype)
    return _sweep[key]


def pipe_fits(dtype, tn, tr):
    """csr_pipe_kernel's launch: two stages at least, within the 224 KB it asks for."""
    stage = ((tn + 8) * np.dtype(dtype).itemsize + (tn + 8) * 4 + (tr + 12) * 4 + 127) & ~127
    return 2 * stage + 32 * 2 + 16 <= 224 * 1024


SWEEP = [(np.float64, tn, tr, xw) for tn in (64, 1024, 2048, 8192) for tr in (32, 512, 4096) for xw in (64, 2048)] \
    + [(np.float32, 64, 32, 64), (np.float32, 1024, 512, 2048), (np.float32, 8192, 4096, 2048), (np.float32, 2048, 4096, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype, tn, tr, xw", SWEEP, ids=[f"{np.dtype(d).name}-{a}-{b}-{c}" for d, a, b, c in SWEEP])
def test_tile_parameters(ctx1, params, dtype, tn, tr, xw):
    row, col, val, m = sweep_matrix(dtype)
    params("spmv.tile_nnz", tn); params("spmv.tile_rows", tr); params("spmv.xwin", xw)
    A = spmat(ctx1, row, col, val, m)
    for k in ("spmv.tile_nnz", "spmv.tile_rows", "spmv.xwin"):
        params(k, DEFAULTS[k])
    info = A.info().loc
    assert info.tile_nnz == tn and info.n_tiles == len(csr_tiles(row, tn, tr)) - 1
    fails = () if pipe_fits(dtype, tn, tr) else (1,)
    check_kernels(ctx1, A, row, col, val, m, dtype, seed=tn + tr + xw, tile_nnz=tn, tile_rows=tr, set_kernel=params, fails=fails)


# ------------------------------------------------------------------------------------------------ 3. persistent laps

_laps = {}
LAP_TILES = (256, 64)                  # CTA tiles of the pipe kernel's laps: ~12 k tiles, ~90 per CTA at one CTA per SM


def lap_case(ctx, dtype, tiles):
    """~200 k rows and ~3 M entries: short and medium rows, long rows, runs of empty rows.  The matrix, the strip (CTA
    tiles of `tiles` = (tile_nnz, tile_rows)) and its references are built once."""
    key = np.dtype(dtype).name
    if key not in _laps:
        w = mixed_lengths(200000, 61, long_every=1500, runs=40)
        row, col, val, m = from_lengths(w, seed=62, dtype=dtype)
        _laps[key] = (row, col, val, m, (np.random.default_rng(63).random(m) - 0.5).astype(dtype))
    row, col, val, m, X = _laps[key]
    if (key, tiles) not in _laps:
        vx.set_param("spmv.tile_nnz", tiles[0]); vx.set_param("spmv.tile_rows", tiles[1])
        try:
            A = spmat(ctx, row, col, val, m)
        finally:
            vx.set_param("spmv.tile_nnz", DEFAULTS["spmv.tile_nnz"]); vx.set_param("spmv.tile_rows", DEFAULTS["spmv.tile_rows"])
        assert A.info().loc.n_tiles == len(csr_tiles(row, *tiles)) - 1
        _laps[key, tiles] = (A, Refs(row, col, val, X, dtype, *tiles))
    return (row, m, X) + _laps[key, tiles]


LAPS = [(1, {"spmv.stages": 2}), (1, {"spmv.stages": 16}), (1, {}), (1, {"tiles": False}), (4, {}),
        (5, {"spmv.ring_stages": 2, "spmv.ring_warps": 1}), (5, {"spmv.ring_stages": 2, "spmv.ring_warps": 8}),
        (5, {"spmv.ring_stages": 8, "spmv.ring_warps": 1}), (5, {"spmv.ring_stages": 8, "spmv.ring_warps": 8}), (5, {})]
LAP_CASES = [(d, k, s, cap) for d in (np.float64, np.float32) for k, s in LAPS for cap in (1, 0)
             if cap == 1 or set(s) <= {"tiles"}]


def _lap_id(d, k, s, cap):
    sets = "-".join(f"{a.split('.')[-1]}{b}" for a, b in s.items()) or "default"
    return f"{np.dtype(d).name}-k{k}-{sets}-cap{cap}"


def ring_fits(dtype, stages, warps):
    """csr_ring_kernel's launch: warps x stages slots of 264 values, 264 columns and 264 row pointers, 128-byte aligned."""
    slot = (264 * np.dtype(dtype).itemsize + 264 * 4 + 264 * 4 + 127) & ~127
    return warps * stages * (slot + 8) <= 224 * 1024


@pytest.mark.gpu
@pytest.mark.parametrize("dtype, kernel, setting, cap", LAP_CASES, ids=[_lap_id(*c) for c in LAP_CASES])
def test_persistent_laps(ctx1, params, dtype, kernel, setting, cap):
    """spmv.ctas_per_sm = 1: every persistent CTA (kernel 1, on 256-entry tiles) takes ~90 tiles and every warp of
    kernels 4 and 5 ~10 (8 warps per CTA) or ~80 (one), so loops turn and rings wrap many times; cap 0 is the default
    grid, and kernel 1 also runs on the default tiles."""
    row, m, X, A, refs = lap_case(ctx1, dtype, LAP_TILES if kernel == 1 and setting.get("tiles", True) else (2048, 512))
    setting = {k: v for k, v in setting.items() if k != "tiles"}
    n = row.size - 1
    Y0 = (np.random.default_rng(64).random(n) - 0.5).astype(dtype)
    params("spmv.ctas_per_sm", cap)
    for k, v in setting.items():
        params(k, v)
    params("spmv.kernel", kernel)
    if kernel == 5 and not ring_fits(dtype, setting.get("spmv.ring_stages", 3), setting.get("spmv.ring_warps", 8)):
        with pytest.raises(L.VexbError, match="shared memory"):
            run_ops(ctx1, A, X, Y0)
        return
    got = run_ops(ctx1, A, X, Y0)
    for op, (alpha, append) in OPS.items():
        assert_same(got[op], store_ref(Y0, refs(kernel), alpha, append, dtype), f"kernel {kernel} {setting} {op}")


# ------------------------------------------------------------------------------------------------ 4. several parts

def parts_matrix(kind, dtype):
    w = mixed_lengths(6000, 71, long_every=800, runs=3, run_len=100)
    return from_lengths(w, seed=72, dtype=dtype, band=None if kind == "scattered" else 60)


def compress(ptr, rows):
    """Row pointers and entry indices of the strip made of `rows` (sorted) of a CSR with pointers `ptr`."""
    cnt = ptr[rows + 1] - ptr[rows]
    p = np.zeros(rows.size + 1, np.int64)
    np.cumsum(cnt, out=p[1:])
    return p, np.repeat(ptr[rows] - p[:-1], cnt) + np.arange(int(p[-1]), dtype=np.int64)


def part_ref(A, k, kernel, X, Y0, alpha, append, dtype):
    """y of part k as vexb_dspmat_apply composes it without the peer-memory halo: interior (or all) rows from the local
    strip, boundary rows from the boundary strip, then y += alpha * (ghost entries) for rows that have any.  The
    interior is the longest ghost-free run of rows if it covers >= 80 % of them, else every ghost-free row."""
    info = A.info(k)
    n = int(info.nrows)
    lp, lc, lv = np.empty(n + 1, np.int64), np.empty(info.loc_nnz, np.int64), np.empty(info.loc_nnz, dtype)
    rp, rc, rv = np.empty(n + 1, np.int64), np.empty(info.rem_nnz, np.int64), np.empty(info.rem_nnz, dtype)
    L.check(L.lib().vexb_dspmat_download_split(A.parts[k], lp.ctypes.data, lc.ctypes.data, lv.ctypes.data,
                                               rp.ctypes.data, rc.ctypes.data, rv.ctypes.data))
    xl = X[int(A.col_part[k]):int(A.col_part[k + 1])]
    xg = X[np.asarray(A.ghosts[k], np.int64)]

    def strip(ptr, col, val, x, rows):
        p, j = compress(ptr, rows)
        return csr_kernel_ref(kernel, p, col[j], val[j], x, dtype)

    if rc.size == 0:
        return store_ref(Y0, strip(lp, lc, lv, xl, np.arange(n)), alpha, append, dtype)
    has = np.diff(rp) > 0
    best_lo = best_hi = run_lo = 0
    for i in range(n + 1):
        if i == n or has[i]:
            if i - run_lo > best_hi - best_lo:
                best_lo, best_hi = run_lo, i
            run_lo = i + 1
    interior = np.zeros(n, bool)
    if (best_hi - best_lo) * 5 >= n * 4:
        interior[best_lo:best_hi] = True
    else:
        interior = ~has
    y = Y0.copy()
    for rows in (np.nonzero(interior)[0], np.nonzero(~interior)[0]):
        if rows.size:
            y[rows] = store_ref(Y0[rows], strip(lp, lc, lv, xl, rows), alpha, append, dtype)
    rows = np.nonzero(has)[0]
    y[rows] = store_ref(y[rows], strip(rp, rc, rv, xg, rows), alpha, True, dtype)
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kind", ["scattered", "banded"])
@pytest.mark.parametrize("nparts", [2, 3])
def test_parts(ctx2, ctx3, params, nparts, kind, dtype):
    """Boundary and ghost strips are CSR strips with a row map: every kernel, with = and with append."""
    ctx = {2: ctx2, 3: ctx3}[nparts]
    row, col, val, m = parts_matrix(kind, dtype)
    n = row.size - 1
    A = spmat(ctx, row, col, val, m)
    assert not A.peer_halo
    rng = np.random.default_rng(nparts)
    X = (rng.random(m) - 0.5).astype(dtype)
    Y0 = (rng.random(n) - 0.5).astype(dtype)
    contiguous = []
    for kern in KERNELS:
        params("spmv.kernel", kern)
        got = run_ops(ctx, A, X, Y0)
        for op in ("set", "half_append"):
            alpha, append = OPS[op]
            want = np.concatenate([part_ref(A, k, kern, X, Y0[int(A.part[k]):int(A.part[k + 1])], alpha, append, dtype)
                                   for k in range(nparts)])
            assert_same(got[op], want, f"kernel {kern}, {op}")
    for k in range(nparts):
        info = A.info(k)
        contiguous.append(info.loc.nrows < info.nrows or info.rem_nnz == 0)
    # the banded matrix keeps a contiguous interior (a strip with a row offset), the scattered one a row-mapped one
    assert all(contiguous) == (kind == "banded")
