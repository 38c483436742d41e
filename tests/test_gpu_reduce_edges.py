"""Reductions, the fused dot and the fused CG iteration, bit for bit against a restatement of their order of additions.

tests/reduce_order.py restates the grids and the folds of reduce_sweep_kernel, reduce_interp_kernel,
reduce_multi_kernel, block_finish, cg_update_r_kernel, dist_apply_kernel's dot partials and dot_fold_kernel, every
operation rounded in the result dtype.  Every value here is compared with it on its bits (uint64 / uint32 views, so
-0.0 and +0.0 differ), in float64 and float32, with reduce.blocks_per_sm 1, 8 and 16 and the SM count of device 0:
  * SUM and SUM_KAHAN through the five reduce shapes on the sweep kernel, the same expressions with
    eval.force_interp = 1, and x + y, which the interpreter takes without forcing; at lengths around the vector width
    E, one block's 512 E, the interpreter's 1024, the capped grid (SMs * bps * 512 E, SMs * bps * 1024) and a length
    whose grid-stride loop turns three times with a partial last turn and a tail.  Data: mixed magnitudes and signs,
    heavy cancellation, all -0.0 (the fold starts from +0, so the sum is +0.0), and data on which the restatements of
    SUM and SUM_KAHAN differ (so losing the compensation fails);
  * vex::CombineReductors [SUM, SUM_KAHAN, MAX, MIN, SUM], several slots of one device (each slot folds its slice,
    the host adds the slots in order), vexb_cg_update_r's r and rho', SpMat.apply_dot's dot in every encoding with a
    dist_apply_kernel (1 to 16 385 partials for dot_fold_kernel), and 20 CGFused iterations, stream-launched and
    replayed as CUDA graphs.
Expressions have at most one rounding operation per element, so whether the interpreter would contract a multiply-add
never decides a result.  MIN, MAX and MINMAX are exact on the same data."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import reduce_order as ro
import vexcl_b200 as vx
from test_gpu_ell_edges import ENCODINGS, STENCIL, band, spmat
from vexcl_b200 import _lib as L
from vexcl_b200.api import DeviceScalar
from vexcl_b200.solvers import CGFused

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
DEFAULTS = {"reduce.blocks_per_sm": 8, "eval.force_interp": 0}
LONG = 1 << 20                       # past this length only "mul" runs every data set on both paths; the other
                                     # expressions run the mixed data on their own path


@contextlib.contextmanager
def param(name, value):
    """Set a library parameter for the with-block, then put back the value it had (its default if never set)."""
    old = C.c_long()
    prev = old.value if L.lib().vexb_get_param(name.encode(), C.byref(old)) == L.OK else DEFAULTS[name]
    vx.set_param(name, value)
    try:
        yield
    finally:
        vx.set_param(name, prev)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(v, dtype):
    a = np.asarray(v, dtype)
    return a.view(np.uint64 if a.itemsize == 8 else np.uint32)


def assert_bits(got, want, dtype, what):
    g, w = bits(got, dtype), bits(want, dtype)
    assert np.array_equal(g, w), f"{what}: got {np.asarray(got, dtype)!r}, want {np.asarray(want, dtype)!r}"


# ------------------------------------------------------------------------------------------------ data

EXPRS = {                            # name: (expression of vectors x, y; the same terms in numpy)
    "copy": (lambda x, y: x, lambda X, Y: X),
    "mul": (lambda x, y: x * y, lambda X, Y: X * Y),
    "sqr": (lambda x, y: x * x, lambda X, Y: X * X),
    "sub": (lambda x, y: x - y, lambda X, Y: X - Y),
    "absdiff": (lambda x, y: vx.fabs(x - y), lambda X, Y: np.abs(X - Y)),
    "add": (lambda x, y: x + y, lambda X, Y: X + Y),
}


def paths(name, n):
    """(eval.force_interp, path) pairs an expression runs on."""
    if name not in ro.SWEEP_SHAPES:
        return [(0, "interp")]
    if n > LONG and name != "mul":
        return [(0, "sweep")]
    return [(0, "sweep"), (1, "interp")]


def mixed(seed, n, dtype):
    """sign * U[1, 2) * 2^k, k uniform in [-40, 40]."""
    rng = np.random.default_rng(seed)
    m = np.ldexp(1 + rng.random(n, dtype=dtype), rng.integers(-40, 41, n, dtype=np.int32))
    return np.where(rng.random(n, dtype=dtype) < 0.5, -m, m)


def cancelling(seed, n, dtype):
    """x in the first half and -x (1 + eps) at the same place in the second half, eps a few ulps of 1: the sum is a
    small remainder of large terms."""
    h = n // 2
    A = mixed(seed, h, dtype).astype(np.float64)
    eps = np.random.default_rng(seed + 1).integers(1, 16, h) * float(np.finfo(dtype).eps)
    X = np.empty(n, dtype)
    X[:h] = A
    X[h:2 * h] = -A * (1 + eps)
    if n % 2:
        X[-1] = 1.5
    return X


class Data:
    """The data sets of one length, generated once: data(kind, name) gives X, Y for expression `name`."""

    def __init__(self, n, dtype, seed):
        self.n, self.dtype, self.seed, self.memo = n, dtype, seed, {}

    def _get(self, key, make):
        if key not in self.memo:
            self.memo[key] = make()
        return self.memo[key]

    def __call__(self, kind, name):
        n, dtype, seed = self.n, self.dtype, self.seed
        if kind == "mixed":
            return self._get("m1", lambda: mixed(seed, n, dtype)), self._get("m2", lambda: mixed(seed + 1, n, dtype))
        if kind == "cancel":
            X = self._get("c", lambda: cancelling(seed + 2, n, dtype))
            if name == "mul":                                 # y = 1 + a few ulps: x*y rounds, the halves still cancel
                eps = float(np.finfo(dtype).eps)
                return X, self._get("c1", lambda: (1 + np.random.default_rng(seed + 3).integers(0, 4, n) * eps).astype(dtype))
            return X, self._get("cs", lambda: (self("mixed", name)[1].astype(np.float64) * 2.0 ** -50).astype(dtype))
        assert kind == "negzero"                              # terms of -0.0 where the expression allows one
        return np.full(n, -0.0, dtype), np.full(n, {"mul": 1.0, "add": -0.0}.get(name, 0.0), dtype)


KAHAN_ROOT = {np.float64: 1.0625 * 2.0 ** -27, np.float32: 1.5 * 2.0 ** -13}


def kahan_data(name, n, dtype, idx):
    """Element 0's accumulator takes 1, s, s (at idx), everything else is +0; s = r^2 lies between a quarter and a half
    ulp of 1, so SUM stays at 1 and SUM_KAHAN carries 2 s to 1 + ulp."""
    typ = np.dtype(dtype).type
    r = typ(KAHAN_ROOT[dtype])
    s = r * r
    X, Y = np.zeros(n, dtype), np.zeros(n, dtype)
    X[idx] = [1, r, r] if name == "sqr" else [1, s, s]
    if name == "mul":
        Y[:] = 1
    return X, Y


def three_turns(dtype, bps):
    """floor(n / E) = 2 full turns of the capped sweep grid + half a turn + 37 vectors (the last turn ends inside
    u = 0 of one block), then a tail of E - 1."""
    E, cap = ro.lanes(dtype), sms() * bps
    return (2 * cap * 512 + cap * 256 + 37) * E + E - 1


def reduce_lengths(dtype, bps):
    E, cap = ro.lanes(dtype), sms() * bps
    return sorted({1, E - 1, E, E + 1, 512 * E - 1, 512 * E, 512 * E + 1, 1023, 1024, 1025,
                   cap * 512 * E, cap * 512 * E + E, cap * 1024 - 1, cap * 1024 + 1, three_turns(dtype, bps)})


# ------------------------------------------------------------------------------------------------ 1. single reductions

def load(x, y, X, Y):
    x.write(X)
    y.write(Y)


def check_sums(ctx, x, y, name, X, Y, dtype, bps, runs, what, device=False):
    """SUM and SUM_KAHAN of expression `name` (x, y hold X, Y) on each (force_interp, path) of runs against the
    restatement."""
    expr, ref = EXPRS[name]
    T = ref(X, Y)
    assert T.dtype == dtype
    ds = DeviceScalar(ctx, dtype) if device else None
    for force, path in runs:
        with param("eval.force_interp", force):
            for op in (L.SUM, L.SUM_KAHAN):
                got = vx.Reductor(ctx, dtype, op)(expr(x, y))
                want = ro.reduce_sum(T, op == L.SUM_KAHAN, path, sms(), bps)
                assert_bits(got, want, dtype, (what, name, path, op))
                if device:
                    vx.Reductor(ctx, dtype, op).device(expr(x, y), ds)
                    assert_bits(ds.get(), got, dtype, (what, name, path, op, "device"))
    return T


@pytest.mark.parametrize("bps", [1, 8, 16])
@pytest.mark.parametrize("dtype", DTYPES)
def test_single_reductions(ctx1, dtype, bps):
    S = sms()
    with param("reduce.blocks_per_sm", bps):
        for n in reduce_lengths(dtype, bps):
            x, y = vx.vector(ctx1, n, dtype), vx.vector(ctx1, n, dtype)
            data = Data(n, dtype, seed=n % 1000)
            # mixed magnitudes: sums, the device-resident result, and MIN / MAX / MINMAX exact
            X, Y = data("mixed", None)
            load(x, y, X, Y)
            for name, (expr, ref) in EXPRS.items():
                runs = paths(name, n)
                T = check_sums(ctx1, x, y, name, X, Y, dtype, bps, runs, (n, "mixed"), device=True)
                for force, path in runs:
                    with param("eval.force_interp", force):
                        assert vx.Reductor(ctx1, dtype, L.MAX)(expr(x, y)) == T.max(), (n, name, path)
                        assert vx.Reductor(ctx1, dtype, L.MIN)(expr(x, y)) == T.min(), (n, name, path)
                        assert vx.Reductor(ctx1, dtype, L.MINMAX)(expr(x, y)) == (T.min(), T.max()), (n, name, path)
            for name, (expr, ref) in EXPRS.items():
                if n > LONG and name != "mul":
                    continue
                runs = paths(name, n)
                # -0.0 everywhere: +0.0
                load(x, y, *data("negzero", name))
                for force, path in runs:
                    with param("eval.force_interp", force):
                        for op in (L.SUM, L.SUM_KAHAN):
                            assert_bits(vx.Reductor(ctx1, dtype, op)(expr(x, y)), 0.0, dtype, (n, name, path, op, "-0"))
                # heavy cancellation
                X, Y = data("cancel", name)
                load(x, y, X, Y)
                check_sums(ctx1, x, y, name, X, Y, dtype, bps, runs, (n, "cancel"))
                # an accumulator that takes 1, s, s: the compensation decides the sum
                for force, path in runs:
                    idx = ro.first_takes(n, dtype, path, S, bps)[:3]
                    if len(idx) < 3:
                        continue                  # a compensation is first used by an accumulator's third term
                    X, Y = kahan_data(name, n, dtype, idx)
                    T = ref(X, Y)
                    want = {op: ro.reduce_sum(T, op == L.SUM_KAHAN, path, S, bps) for op in (L.SUM, L.SUM_KAHAN)}
                    assert bits(want[L.SUM], dtype) != bits(want[L.SUM_KAHAN], dtype), (n, name, path)
                    load(x, y, X, Y)
                    with param("eval.force_interp", force):
                        for op in (L.SUM, L.SUM_KAHAN):
                            assert_bits(vx.Reductor(ctx1, dtype, op)(expr(x, y)), want[op], dtype, (n, name, path, op, "kahan"))
    assert ro.first_takes(three_turns(dtype, bps), dtype, "sweep", S, bps)[3] == three_turns(dtype, bps) - (ro.lanes(dtype) - 1)


# ------------------------------------------------------------------------------------------------ 2. CombineReductors

KINDS = [L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.SUM]


def combined_want(T, sum_of):
    s, k = sum_of(T, False), sum_of(T, True)
    return [s, k, T.max(), T.min(), s]


def check_combined(ctx, x, y, name, X, Y, dtype, sum_of, what):
    expr, ref = EXPRS[name]
    T = ref(X, Y)
    load(x, y, X, Y)
    got = vx.Reductor(ctx, dtype, KINDS)(expr(x, y))
    want = combined_want(T, sum_of)
    for j in range(len(KINDS)):
        assert_bits(got[j], want[j], dtype, (what, name, j))
    return T


@pytest.mark.parametrize("bps", [1, 8, 16])
@pytest.mark.parametrize("dtype", DTYPES)
def test_combined_reductors(ctx1, dtype, bps):
    S, cap = sms(), sms() * bps
    sum_of = lambda T, kahan: ro.reduce_sum(T, kahan, "multi", S, bps)
    with param("reduce.blocks_per_sm", bps):
        for n in (1, 1023, 1024, 1025, cap * 1024 - 1, cap * 1024 + 1, 3 * cap * 1024 + 700):
            x, y = vx.vector(ctx1, n, dtype), vx.vector(ctx1, n, dtype)
            data = Data(n, dtype, seed=n % 1000 + 3)
            for name in ("copy", "mul"):
                for kind in ("mixed", "cancel") if n <= LONG else ("mixed",):
                    check_combined(ctx1, x, y, name, *data(kind, name), dtype, sum_of, (n, kind))
                idx = ro.first_takes(n, dtype, "multi", S, bps)[:3]
                if len(idx) == 3:
                    X, Y = kahan_data(name, n, dtype, idx)
                    T = check_combined(ctx1, x, y, name, X, Y, dtype, sum_of, (n, "kahan"))
                    assert bits(sum_of(T, False), dtype) != bits(sum_of(T, True), dtype)


# ------------------------------------------------------------------------------------------------ 3. several slots

@pytest.mark.parametrize("nparts", [2, 3])
@pytest.mark.parametrize("dtype", DTYPES)
def test_slots(ctx2, ctx3, nparts, dtype):
    ctx = {2: ctx2, 3: ctx3}[nparts]
    E, S = ro.lanes(dtype), sms()
    lo, hi = np.finfo(dtype).min, np.finfo(dtype).max
    for n in (0, 19, 1025, 3 * 512 * E + E - 1, 1_000_003):
        part = ctx.partition(n)
        sizes = np.diff(part)
        if n == 19:
            assert any(0 < s < E for s in sizes), sizes           # a slot that holds only a tail
        x, y = vx.vector(ctx, n, dtype), vx.vector(ctx, n, dtype)
        if n == 0:
            for name, (expr, _) in EXPRS.items():
                for op in (L.SUM, L.SUM_KAHAN):
                    assert_bits(vx.Reductor(ctx, dtype, op)(expr(x, y)), 0.0, dtype, (nparts, name, op))
                assert vx.Reductor(ctx, dtype, L.MAX)(expr(x, y)) == lo and vx.Reductor(ctx, dtype, L.MIN)(expr(x, y)) == hi
                assert vx.Reductor(ctx, dtype, L.MINMAX)(expr(x, y)) == (hi, lo)
                got = vx.Reductor(ctx, dtype, KINDS)(expr(x, y))
                assert_bits(got, [0.0, 0.0, lo, hi, 0.0], dtype, (nparts, name, "combined"))
            continue
        data = Data(n, dtype, seed=n % 1000 + 11)
        for name, (expr, ref) in EXPRS.items():
            X, Y = data("mixed", name)
            T = ref(X, Y)
            load(x, y, X, Y)
            for force, path in paths(name, n):
                with param("eval.force_interp", force):
                    for op in (L.SUM, L.SUM_KAHAN):
                        want = ro.slots_sum(T, part, op == L.SUM_KAHAN, path, S, 8)
                        assert_bits(vx.Reductor(ctx, dtype, op)(expr(x, y)), want, dtype, (nparts, n, name, path, op))
            if name in ("copy", "mul"):
                sum_of = lambda V, kahan: ro.slots_sum(V, part, kahan, "multi", S, 8)
                check_combined(ctx, x, y, name, X, Y, dtype, sum_of, (nparts, n))


# ------------------------------------------------------------------------------------------------ 4. cg_update_r

@pytest.mark.parametrize("bps", [1, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_cg_update_r(ctx1, dtype, bps):
    """alpha = rho / pq is not a power of two, so r - alpha q and its squares round.  Nothing past n changes."""
    typ = np.dtype(dtype).type
    lib, vt = L.lib(), (L.F64 if dtype == np.float64 else L.F32)
    ws, _ = ctx1.workspace(0)
    E, S = ro.lanes(dtype), sms()
    pad = 11
    rho, pq = typ(2.718281828459045), typ(0.3183098861837907)
    with param("reduce.blocks_per_sm", bps):
        for n in (1, E - 1, E, E + 1, 512 * E - 1, 512 * E, 512 * E + 1, 3 * 512 * E + E - 1, S * bps * 512 * E + 3 * E + 3,
                  three_turns(dtype, bps)):
            R = ((oracle.uniform_real(n % 1000, n + pad) - 0.5) * 8).astype(dtype)
            Q = ((oracle.uniform_real(n % 1000 + 1, n + pad) - 0.5) * 3).astype(dtype)
            r, q = vx.vector(ctx1, R), vx.vector(ctx1, Q)
            d_rho, d_pq, d_new = DeviceScalar(ctx1, dtype, rho), DeviceScalar(ctx1, dtype, pq), DeviceScalar(ctx1, dtype, 0.0)
            L.check(lib.vexb_cg_update_r(0, ctx1.streams[0], vt, n, r.bufs[0], q.bufs[0], d_rho.bufs[0], d_pq.bufs[0],
                                         d_new.bufs[0], ws, None))
            want_r, want_rho = ro.cg_update_r(R[:n], Q[:n], rho, pq, S, bps)
            got = r.read()
            assert_bits(got[:n], want_r, dtype, (n, "r"))
            assert_bits(got[n:], R[n:], dtype, (n, "padding"))
            assert_bits(d_new.get(), want_rho, dtype, (n, "rho'"))


# ------------------------------------------------------------------------------------------------ 5. fused dot

def check_dot(ctx, A, n, dtype, seed, what):
    """apply_dot with dot_with = None (the dot of x and y), then with a w vector at alpha = -0.5 with append.  w is
    chosen from the y that product gives, so that the terms w[r] y[r] cancel in pairs (t, then -t (1 + eps) half a
    vector later): the dot is a small remainder of large partials, and any other order of additions shows in its bits."""
    X, Y0 = (((oracle.uniform_real(seed + k, n) - 0.5) * 4).astype(dtype) for k in range(2))
    x, y = vx.vector(ctx, X), vx.vector(ctx, Y0)
    d = DeviceScalar(ctx, dtype)
    assert A.apply_dot(x, y, d), what
    assert_bits(d.get(), ro.fused_dot(X, y.read()), dtype, (what, "x"))
    y.write(Y0)
    A.apply(x, y, -0.5, True)
    Yp = y.read().astype(np.float64)
    T = cancelling(seed, n, dtype).astype(np.float64)
    W = np.where(Yp != 0, T / np.where(Yp != 0, Yp, 1), 0).astype(dtype)
    w = vx.vector(ctx, W)
    y.write(Y0)
    assert A.apply_dot(x, y, d, dot_with=w, alpha=-0.5, append=True), what
    assert_bits(d.get(), ro.fused_dot(W, y.read()), dtype, (what, "w"))


@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("w", [3, 5, 7])
@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_dot(ctx1, dtype, w, enc):
    """1, 2 and 1023 / 1025 partials: dot_fold_kernel's threads take one partial, or thread 0 takes two."""
    offsets, vals = STENCIL[w]
    for n in (1, 255, 256, 257, 256 * 1024 - 256, 256 * 1024 + 256):
        row, col, val = band(n, n, offsets, np.array(vals, dtype))
        A = spmat(ctx1, n, n, row, col, val, enc)
        check_dot(ctx1, A, n, dtype, n % 1000, (n, w, enc))


@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_dot_long_batch(ctx1, dtype):
    """16 383 and 16 385 partials: each thread of dot_fold_kernel adds a batch of 16 (or 15), and at 16 385 thread 0
    starts a second batch."""
    offsets, vals = STENCIL[5]
    for n in (256 * 16384 - 256, 256 * 16384 + 256):
        row, col, val = band(n, n, offsets, np.array(vals, dtype))
        A = vx.SpMat(ctx1, n, n, row, col, val, vx.FMT_HELL)
        check_dot(ctx1, A, n, dtype, 5, n)


# ------------------------------------------------------------------------------------------------ 6. CGFused

@pytest.mark.parametrize("grid", [17, 131])
def test_fused_cg(ctx1, grid):
    """17^3 = 4913 rows (N mod 8 = 1); 131^3 = 2 248 091 rows, where cg_update_r's grid is capped at SMs * 8 blocks and
    its loop turns twice.  Every rho' and the final x equal the CPU simulation bit for bit, stream-launched and replayed
    as two alternating CUDA graphs."""
    iters, S = 20, sms()
    row, col, val, N = ro.laplacian(grid)
    if grid == 131:
        assert ro.sweep_blocks(N, np.float64, S, 8) == S * 8 and N // 4 > S * 8 * 512
    b = oracle.uniform_real(3, N)
    x_sim, hist_sim = ro.cg_fused(row, col, val, b, iters, S)
    A = vx.SpMat(ctx1, N, N, row, col, val)
    runs = {}
    for use_graph in (False, True):
        bv, xv = vx.vector(ctx1, b), vx.vector(ctx1, N)
        xv.assign(0.0)
        cg = CGFused(A, bv, xv)
        assert_bits(cg.r.read(), b, np.float64, "r = b - A*0")
        hist = []
        if use_graph:
            cg.capture()                                   # iterations 1 and 2 run while warming up
            hist = [cg.rho2[1].get(), cg.rho2[0].get()]    # rho' of iteration k lands in rho2[k & 1]
        while len(hist) < iters:
            cg.run(1)
            hist.append(cg.residual2())
        ctx1.finish()
        assert cg.fused_product
        assert_bits(hist, hist_sim, np.float64, ("history", use_graph))
        runs[use_graph] = xv.read()
        assert_bits(runs[use_graph], x_sim, np.float64, ("x", use_graph))
    assert_bits(runs[True], runs[False], np.float64, "graph against stream")
