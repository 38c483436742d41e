"""CPU self-checks of tests/reduce_order.py, the restatement the GPU reduction suite compares the kernels with: its
shuffle tree, Kahan step and grids against cases worked by hand, its sums against exact and compensated sums, and its
CG simulation against oracle.cg.  No GPU needed."""
import math

import numpy as np
import pytest

import oracle
import reduce_order as ro

SMS = [132, 7]
DTYPES = [np.float64, np.float32]


def test_warp_tree_by_hand():
    v = oracle.uniform_real(1, 32) - 0.5
    a = list(v)
    for off in (16, 8, 4, 2, 1):
        a = [a[l] + a[l + off] for l in range(off)]
    assert ro.warp_tree(v) == a[0]
    w =np.stack([v, v[::-1]])
    assert list(ro.warp_tree(w)) == [ro.warp_tree(v), ro.warp_tree(v[::-1].copy())]


@pytest.mark.parametrize("dtype, p", [(np.float64, 53), (np.float32, 24)])
def test_kahan_step_by_hand(dtype, p):
    """[1, 2^-p, 2^-p]: each 2^-p is half an ulp of 1, so a plain sum stays at 1 (ties to even) while the compensated
    one reaches 1 + 2^(1-p)."""
    typ = np.dtype(dtype).type
    terms = [typ(1), typ(2.0 ** -p), typ(2.0 ** -p)]
    s = c = typ(0)
    plain = typ(0)
    for t in terms:
        s, c = ro.kahan_take(s, c, t)
        plain = plain + t
    assert plain == typ(1)
    assert s == typ(1 + 2.0 ** (1 - p)) and s.dtype == dtype
    # through the kernels' geometry: element 0's accumulator takes the three terms, everything else is +0
    n, sms, bps = 3 * 512 * 4 * ro.lanes(dtype) + 1, 1, 1
    for path in ("sweep", "interp", "multi"):
        idx = ro.first_takes(n, dtype, path, sms, bps)[:3]
        assert len(idx) == 3 and idx[0] == 0
        v = np.zeros(n, dtype)
        v[idx] = terms
        assert ro.reduce_sum(v, False, path, sms, bps) == typ(1)
        assert ro.reduce_sum(v, True, path, sms, bps) == typ(1 + 2.0 ** (1 - p))


def test_second_term_compensation_is_dropped():
    """Two terms per accumulator: the compensation of the second term is never used, so SUM_KAHAN gives SUM's bits."""
    n, sms, bps = 2 * 132 * 2 * 256 * 4, 132, 1
    rng = np.random.default_rng(3)
    v = rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)
    assert len(ro.first_takes(n, np.float64, "sweep", sms, bps)) == 2
    assert ro.reduce_sum(v, True, "sweep", sms, bps) == ro.reduce_sum(v, False, "sweep", sms, bps)


def test_grids_by_hand():
    # sweep: ceil(floor(n / E) / 512) blocks, at least 1, at most SMs * bps
    assert ro.sweep_blocks(0, np.float64, 132, 8) == 0
    assert ro.sweep_blocks(1, np.float64, 132, 8) == 1                 # n < E: no vector, one block for the tail
    assert ro.sweep_blocks(7, np.float32, 132, 8) == 1
    assert ro.sweep_blocks(2048, np.float64, 132, 8) == 1              # 512 vectors of 4
    assert ro.sweep_blocks(2052, np.float64, 132, 8) == 2
    assert ro.sweep_blocks(2051, np.float64, 132, 8) == 1              # 512 vectors + a tail of 3
    assert ro.sweep_blocks(4096, np.float32, 132, 8) == 1
    assert ro.sweep_blocks(4104, np.float32, 132, 8) == 2
    assert ro.sweep_blocks(10 ** 8, np.float64, 132, 8) == 1056
    assert ro.sweep_blocks(10 ** 8, np.float64, 7, 8) == 56
    assert ro.sweep_blocks(10 ** 8, np.float64, 7, 0) == 7             # bps clamped to [1, 16]
    assert ro.sweep_blocks(10 ** 8, np.float64, 7, 99) == 112
    # interpreter: ceil(n / 1024), at most SMs * bps
    assert ro.interp_blocks(0, 132, 8) == 0
    assert ro.interp_blocks(1, 132, 8) == 1
    assert ro.interp_blocks(1024, 132, 8) == 1
    assert ro.interp_blocks(1025, 132, 8) == 2
    assert ro.interp_blocks(132 * 1024 + 1, 132, 1) == 132
    assert ro.interp_blocks(10 ** 6, 7, 16) == 112
    # the kernel vexb_reduce_all picks
    assert ro.reduce_path(np.float64, "mul") == "sweep"
    assert ro.reduce_path(np.float32, "absdiff") == "sweep"
    assert ro.reduce_path(np.float64, "mul", force_interp=True) == "interp"
    assert ro.reduce_path(np.float64, None) == "interp"
    assert ro.reduce_path(np.int64, "copy") == "interp"


def test_first_takes_by_hand():
    # sweep, float64, 7 SMs at 1 block per SM: 7 * 512 vectors per turn
    n = 2 * 7 * 512 * 4 + 8 + 3
    assert ro.first_takes(n, np.float64, "sweep", 7, 1) == [0, 7 * 512 * 4, 2 * 7 * 512 * 4, n - 3]   # 3 turns, the tail
    n = 7 * 512 * 4 + 2
    assert ro.first_takes(n, np.float64, "sweep", 7, 1) == [0, n - 2]           # one turn, then the tail
    assert ro.first_takes(5, np.float32, "sweep", 7, 1) == [0]                  # n < E: the tail alone
    assert ro.first_takes(3 * 7 * 1024, np.float64, "interp", 7, 1) == [0, 7 * 1024, 14 * 1024]
    assert ro.first_takes(600, np.float64, "multi", 7, 1) == [0, 256, 512]


def _mixed(seed, n, dtype):
    rng = np.random.default_rng(seed)
    return (rng.choice([-1.0, 1.0], n) * rng.uniform(1, 2, n) * 2.0 ** rng.integers(-40, 41, n)).astype(dtype)


def _lengths(dtype, sms, bps):
    E = ro.lanes(dtype)
    cap = sms * bps
    return [1, E - 1, E + 1, 512 * E + 1, 1025, cap * 1024 + 1, (2 * cap * 512 + cap * 256 + 37) * E + E - 1]


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_integer_data_sums_exactly(dtype, sms):
    for bps in (1, 8):
        for n in _lengths(dtype, sms, bps):
            v = np.random.default_rng(n).integers(-8, 9, n).astype(dtype)
            want = int(v.astype(np.int64).sum())
            for path in ("sweep", "interp", "multi"):
                for kahan in (False, True):
                    got = ro.reduce_sum(v, kahan, path, sms, bps)
                    assert got.dtype == dtype and got == want, (n, bps, path, kahan)
    assert ro.reduce_sum(np.zeros(0, dtype)) == 0


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_real_data_within_the_tree_bound(dtype, sms):
    for bps in (1, 8):
        for n in _lengths(dtype, sms, bps):
            v = _mixed(n, n, dtype)
            exact = math.fsum(v.astype(np.float64))
            for path in ("sweep", "interp", "multi"):
                bound = ro.error_bound(v, ro.sum_depth(n, dtype, path, sms, bps))
                for kahan in (False, True):
                    got = float(ro.reduce_sum(v, kahan, path, sms, bps))
                    assert abs(got - exact) <= bound, (n, bps, path, kahan, got, exact, bound)


@pytest.mark.parametrize("dtype", DTYPES)
def test_negative_zeros_sum_to_positive_zero(dtype):
    """Every fold starts from +0, and +0 + -0 = +0."""
    for n in (1, 7, 4096 + 5, 3 * 7 * 1024 + 9):
        v = np.full(n, -0.0, dtype)
        for path in ("sweep", "interp", "multi"):
            for kahan in (False, True):
                assert not np.signbit(ro.reduce_sum(v, kahan, path, 7, 1))
    assert not np.signbit(ro.fused_dot(np.full(300, -0.0, dtype), np.ones(300, dtype)))


def test_slots_fold_in_slot_order():
    v = np.array([2.0 ** 53, 1.0, 1.0], np.float64)
    assert ro.slots_sum(v, [0, 1, 2, 3]) == 2.0 ** 53                    # (2^53 + 1) + 1, each rounding to even
    assert ro.slots_sum(v, [0, 0, 1, 3]) == 2.0 ** 53 + 2                # 0 + 2^53 + (1 + 1)


def test_fused_dot_by_hand():
    """dot_fold with 2049 partials: thread 0 adds p0, p1024, p2048; threads 1..1023 two partials; then the trees."""
    rng = np.random.default_rng(7)
    parts = rng.standard_normal(2049)
    g = [0.0] * 1024
    for k, p in enumerate(parts):
        g[k % 1024] = g[k % 1024] + p
    warps = [ro.warp_tree(np.array(g[32 * w:32 * w + 32])) for w in range(32)]
    assert ro.dot_fold(parts) == ro.warp_tree(np.array(warps))
    # dist_apply_kernel partials: 300 rows -> 2 blocks, rows past n add +0
    w, y = rng.standard_normal(300), rng.standard_normal(300)
    t = np.zeros(512)
    t[:300] = w * y
    want = []
    for b in range(2):
        ws = [ro.warp_tree(t[256 * b + 32 * k:256 * b + 32 * k + 32]) for k in range(8)]
        tot = ws[0]
        for s in ws[1:]:
            tot = tot + s
        want.append(tot)
    assert list(ro.dot_partials(w, y)) == want
    assert abs(ro.fused_dot(w, y) - math.fsum(w * y)) <= 20 * 2.0 ** -53 * np.sum(np.abs(w * y))


def test_laplacian_is_the_spd_stencil():
    row, col, val, N = ro.laplacian(4)
    assert N == 64 and row[-1] == 64 * 7 - 6 * 16
    A = np.zeros((N, N))
    for i in range(N):
        A[i, col[row[i]:row[i + 1]]] = val[row[i]:row[i + 1]]
        assert np.all(np.diff(col[row[i]:row[i + 1]]) > 0)
    assert np.array_equal(A, A.T) and np.all(np.linalg.eigvalsh(A) > 0)
    assert A[0, 0] == 6 and A[0, 1] == -1 and A[3, 4] == 0 and A[0, 16] == -1


@pytest.mark.parametrize("sms", SMS)
def test_cg_simulation_tracks_the_oracle(sms):
    row, col, val, N = ro.laplacian(17)
    b = oracle.uniform_real(3, N)
    xo, hist_o = oracle.cg(row, col, val, b, np.zeros(N), 20)
    x, hist = ro.cg_fused(row, col, val, b, 20, sms)
    assert hist[-1] < 1e-3 * hist[0]
    assert np.allclose(hist, hist_o, rtol=1e-12, atol=0)
    assert np.allclose(x, xo, rtol=1e-12, atol=1e-14)
