"""Sliced ELL (VEXB_FMT_SELL) where hybrid ELL already serves: K right-hand sides in one pass over the strip
(sell_multi_kernel behind SpMat.apply_multi) and the product as a terminal of a generated assignment kernel that sweeps in
the strip's storage order (vexb_dspmat_sweep_strip, VEXB_TERM_SPMV in vexb_eval).

Everything is compared on bits (integer views), in float64 and float32:
  * component k of apply_multi against A.apply(x_k, y_k);
  * an inlined product against the composition: t = A*x by the product kernel, then the same elementwise expression with
    the vector t in place of the product (products and sums are separate roundings on both sides).
Launches are counted with vx.launch_count().

Aliasing: the inline paths (hybrid ELL and CSR before, sliced ELL now) make no check.  The target may be an elementwise
operand, since element r is read and written by the one thread that owns row r; the target must not be the x of an inlined
product, on any format, because rows gather x while other rows are being written."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import vexcl_b200 as vx
from vexcl_b200 import _lib as L
from vexcl_b200 import build
from vexcl_b200.api import _Lowering, wrap

pytestmark = pytest.mark.gpu

DEFAULTS = {"spmv.sell_sigma": 1024, "spmv.no_multi": 0, "spmv.sell_inline": 1, "spmv.no_inline": 0}
DTYPES = [np.float64, np.float32]


@pytest.fixture
def params(built):
    try:
        yield vx.set_param
    finally:
        for k, v in DEFAULTS.items():
            vx.set_param(k, v)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def assert_same(got, want, what=""):
    g, w = bits(got), bits(want)
    assert np.array_equal(g, w), f"{what}: {np.count_nonzero(g != w)} of {g.size} differ, first at {np.nonzero(g != w)[0][:8]}"


def values(rng, size, dtype):
    return ((rng.random(size) + 0.5) * np.where(rng.random(size) < 0.5, -1.0, 1.0)).astype(dtype)


def matrix(rng, n, m, dtype, wmax=40, spread=None, idx=np.int64, lo=None, hi=None, empty=False):
    """Rows of U[0, wmax) entries (none with empty=True) at distinct sorted columns: anywhere in [0, m), within `spread`
    of the diagonal, or -- lo/hi given per row -- inside [lo[i], hi[i])."""
    w = np.zeros(n, np.int64) if empty else rng.integers(0, wmax, n)
    cols = []
    for i in range(n):
        a, b = (0, m) if spread is None else (max(0, i - spread), min(m, i + spread + 1))
        if lo is not None:
            a, b = int(lo[i]), int(hi[i])
        w[i] = min(w[i], b - a)
        cols.append(a + np.sort(rng.choice(b - a, size=w[i], replace=False)))
    row = np.concatenate([[0], np.cumsum(w)]).astype(idx)
    col = (np.concatenate(cols) if n else np.empty(0)).astype(idx)
    return row, col, values(rng, col.size, dtype)


def sell(ctx, n, m, mat):
    A = vx.SpMat(ctx, n, m, *mat, vx.FMT_SELL)
    assert all(A.info(k).loc.fmt == L.FMT_SELL for k in ctx.local if A.info(k).nrows)
    return A


def sweep_strip(A, k=0):
    h = C.c_void_p()
    L.check(L.lib().vexb_dspmat_sweep_strip(A.parts[k], C.byref(h)))
    return h.value


SIGMA = 1024
SIZES = [1, 31, 32, 33, SIGMA - 1, SIGMA, SIGMA + 1, 8 * SIGMA + 17]


# ------------------------------------------------------------------------------------------------ multivector

def groups(K):
    """Launches of vexb_spmv_multi for K vectors: groups of 4, then 3 / 2 / 1."""
    return K // 4 + (1 if K % 4 else 0)


def check_multi(ctx, A, n, m, dtype, K, rng, launches=None):
    X = [values(rng, m, dtype) for _ in range(K)]
    Y0 = [values(rng, n, dtype) for _ in range(K)]
    xs = [vx.vector(ctx, x) for x in X]
    ya, yr = [vx.vector(ctx, y) for y in Y0], [vx.vector(ctx, y) for y in Y0]
    for name, (alpha, append) in {"=": (1.0, False), "+=": (1.0, True), "-=": (-1.0, True), "0.5+=": (0.5, True)}.items():
        ctx.finish()
        l0 = vx.launch_count()
        A.apply_multi(xs, ya, alpha, append)
        if launches is not None:
            assert vx.launch_count() - l0 == launches * len(ctx.local), name
        for k in range(K):
            A.apply(xs[k], yr[k], alpha, append)
            assert_same(ya[k].read(), yr[k].read(), f"{name} component {k} of {K}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize("cols", ["col16", "col32"])
def test_multivector_in_one_pass(ctx1, params, dtype, K, cols):
    rng = np.random.default_rng(100 + K)
    n = 2 * SIGMA + 77
    A = sell(ctx1, n, n, matrix(rng, n, n, dtype, spread=300 if cols == "col16" else None))
    assert groups(K) == {1: 1, 2: 1, 3: 1, 4: 1, 5: 2, 6: 2}[K]
    check_multi(ctx1, A, n, n, dtype, K, rng, launches=groups(K))
    params("spmv.no_multi", 1)
    check_multi(ctx1, A, n, n, dtype, K, rng, launches=K)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_multivector_sizes(ctx1, params, dtype, n):
    rng = np.random.default_rng(n)
    for sigma, idx in ((256, np.int32), (1024, np.int64)):
        params("spmv.sell_sigma", sigma)
        m = n + 13                                              # rectangular, the last row touching the last column
        row, col, val = matrix(rng, n, m, dtype, idx=idx)
        if row[n] > row[n - 1]:
            col[-1] = m - 1
        check_multi(ctx1, sell(ctx1, n, m, (row, col, val)), n, m, dtype, 4, rng, launches=1)
        check_multi(ctx1, sell(ctx1, n, m, (row, col, val)), n, m, dtype, 3, rng, launches=1)


def test_multivector_empty_rows_and_float_values(ctx1, params):
    rng = np.random.default_rng(5)
    n = 100
    A = vx.SpMat(ctx1, n, n, *matrix(rng, n, n, np.float64, empty=True), vx.FMT_SELL)
    check_multi(ctx1, A, n, n, np.float64, 4, rng)               # no entry at all: y is zeroed or kept, vector by vector
    n = SIGMA + 5
    F = vx.SpMat(ctx1, n, n, *matrix(rng, n, n, np.float64), vx.FMT_SELL | vx.FMT_VALUES_F32)
    assert F.info().loc.fmt == L.FMT_SELL and sweep_strip(F) is None
    check_multi(ctx1, F, n, n, np.float64, 4, rng, launches=4)   # float-valued strips: one vector at a time


def block_diagonal(rng, ctx, n, dtype, coupled):
    part = ctx.partition(n)
    lo, hi = np.zeros(n, np.int64), np.full(n, n, np.int64)
    if not coupled:
        for k in range(len(part) - 1):
            lo[part[k]:part[k + 1]], hi[part[k]:part[k + 1]] = part[k], part[k + 1]
    return matrix(rng, n, n, dtype, lo=lo, hi=hi)


@pytest.mark.parametrize("coupled", [False, True])
@pytest.mark.parametrize("which", ["ctx2", "ctx3"])
def test_multivector_on_several_parts(request, params, which, coupled):
    ctx = request.getfixturevalue(which)
    rng = np.random.default_rng(17)
    n = 3 * SIGMA + 50
    A = sell(ctx, n, n, block_diagonal(rng, ctx, n, np.float64, coupled))
    check_multi(ctx, A, n, n, np.float64, 4, rng, launches=None if coupled else 1)


# ------------------------------------------------------------------------------------------------ inlined products

def check_inline(ctx, n, dtype, rng, build_expr, mats, op="=", launches=1, alias=False):
    """build_expr(P, z, w_products...) with P = the products: inlined (vx.make_inline(A * x) or A * x terms) against the
    vectors t_k = A_k * x_k."""
    Z, Y0 = values(rng, n, dtype), values(rng, n, dtype)
    xs = [vx.vector(ctx, values(rng, A.m, dtype)) for A in mats]
    z = vx.vector(ctx, Z)
    yf, yr = vx.vector(ctx, Y0), vx.vector(ctx, Y0)
    ts = [vx.vector(ctx, n, dtype) for _ in mats]
    for A, x, t in zip(mats, xs, ts):
        A.apply(x, t)
    assign = {"=": lambda y, e: y.assign(e), "+=": lambda y, e: y.__iadd__(e), "-=": lambda y, e: y.__isub__(e)}[op]
    assign(yr, build_expr(ts, yr if alias else z, False))
    assign(yf, build_expr([A * x for A, x in zip(mats, xs)], yf if alias else z, True))       # warm: generates the kernel
    yf2 = vx.vector(ctx, Y0)
    ctx.finish()
    l0 = vx.launch_count()
    assign(yf2, build_expr([A * x for A, x in zip(mats, xs)], yf2 if alias else z, True))
    if launches is not None:
        assert vx.launch_count() - l0 == launches * len(ctx.local)
    assert_same(yf2.read(), yr.read(), op)
    assert_same(yf.read(), yr.read(), op + " (first use)")


def e_add(P, z, inl):         # y = z + A*x
    return z + P[0]


def e_sub2(P, z, inl):        # y = z - 2*(A*x); the additive term is scaled by -2, which rounds nothing
    return z - 2 * P[0] if inl else z + wrap(-2.0 if z.np_dtype == np.float64 else np.float32(-2.0)) * P[0]


def e_twice(P, z, inl):       # y += A*x + A*w: the same strip twice
    return P[0] + P[1] if inl else wrap(P[0]) + P[1]


def e_index(P, z, inl):       # y = z * make_inline(A*x) + element_index
    return z * (vx.make_inline(P[0]) if inl else P[0]) + vx.ElementIndex()


def e_two(P, z, inl):         # two matrices in one expression
    return z * (vx.make_inline(P[0]) if inl else P[0]) - (vx.make_inline(P[1]) if inl else P[1])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", SIZES)
def test_inline_sizes(ctx1, params, dtype, n):
    rng = np.random.default_rng(1000 + n)
    for sigma, idx, spread in ((256, np.int32, 200), (1024, np.int64, None)):
        params("spmv.sell_sigma", sigma)
        A = sell(ctx1, n, n, matrix(rng, n, n, dtype, idx=idx, spread=spread))
        assert sweep_strip(A) is not None
        check_inline(ctx1, n, dtype, rng, e_add, [A])
        check_inline(ctx1, n, dtype, rng, e_sub2, [A])
        check_inline(ctx1, n, dtype, rng, e_index, [A])
        check_inline(ctx1, n, dtype, rng, e_twice, [A, A], op="+=")
        check_inline(ctx1, n, dtype, rng, e_add, [A], alias=True)          # y = y + A*x: the target as an elementwise operand


@pytest.mark.parametrize("dtype", DTYPES)
def test_inline_rectangular_and_empty(ctx1, params, dtype):
    rng = np.random.default_rng(3)
    n, m = SIGMA + 9, 2 * SIGMA
    row, col, val = matrix(rng, n, m, dtype)
    col[-1] = m - 1
    check_inline(ctx1, n, dtype, rng, e_add, [sell(ctx1, n, m, (row, col, val))])
    row, col, val = matrix(rng, n, n, dtype)
    keep = np.ones(n, bool); keep[5:200] = False; keep[n - 3:] = False     # runs of empty rows
    w = np.diff(row) * keep
    sel = np.repeat(keep, np.diff(row))
    row2 = np.concatenate([[0], np.cumsum(w)]).astype(np.int64)
    check_inline(ctx1, n, dtype, rng, e_add, [sell(ctx1, n, n, (row2, col[sel], val[sel]))])


@pytest.mark.parametrize("dtype", DTYPES)
def test_inline_with_other_matrices(ctx1, params, dtype):
    rng = np.random.default_rng(4)
    n = 2 * SIGMA + 3
    A = sell(ctx1, n, n, matrix(rng, n, n, dtype))
    B = sell(ctx1, n, n, matrix(rng, n, n, dtype, spread=100))
    H = vx.SpMat(ctx1, n, n, *matrix(rng, n, n, dtype, wmax=2, lo=np.maximum(np.arange(n) - 1, 0), hi=np.minimum(np.arange(n) + 2, n)),
                 vx.FMT_HELL)
    assert H.info().loc.fmt == L.FMT_HELL
    check_inline(ctx1, n, dtype, rng, e_two, [A, H])                        # sliced ELL swept, hybrid ELL by row: one launch
    check_inline(ctx1, n, dtype, rng, e_two, [H, A])
    # two distinct sliced-ELL matrices: the second takes its temporary, the bits are those of the composition
    check_inline(ctx1, n, dtype, rng, e_two, [A, B], launches=None)
    check_inline(ctx1, n, dtype, rng, e_twice, [A, B], op="+=", launches=None)
    # the library itself refuses a second strip
    low = _Lowering(0, 0)
    low.size = n
    x, z = vx.vector(ctx1, values(rng, n, dtype)), vx.vector(ctx1, n, dtype)
    xa = low.term(L.TERM_VEC, x.dtype, ptr=x.bufs[0].value)
    low.emit("TERM", x.dtype, low.term(L.TERM_SPMV, x.dtype, pad0=xa, ptr=sweep_strip(A)))
    low.emit("TERM", x.dtype, low.term(L.TERM_SPMV, x.dtype, pad0=xa, ptr=sweep_strip(B)))
    low.emit("ADD", x.dtype)
    code = L.lib().vexb_eval(ctx1.devs[0], ctx1.streams[0], z.bufs[0], z.dtype, L.SET, C.byref(low.e), n, 0)
    assert code == L.ERR_UNSUPPORTED
    # ... and reductions and multi-expressions refuse any
    red = _Lowering(0, 0)
    red.size = n
    xa = red.term(L.TERM_VEC, x.dtype, ptr=x.bufs[0].value)
    red.emit("TERM", x.dtype, red.term(L.TERM_SPMV, x.dtype, pad0=xa, ptr=sweep_strip(A)))
    ws, r = ctx1.workspace(0)
    assert L.lib().vexb_reduce_all(ctx1.devs[0], ctx1.streams[0], C.byref(red.e), x.dtype, n, 0, L.SUM, r, ws, None) != L.OK
    s = vx.Reductor(ctx1, dtype, L.SUM)(z - vx.make_inline(A * x))          # the front end keeps the temporary
    t = vx.vector(ctx1, n, dtype)
    A.apply(x, t)
    assert s == pytest.approx(vx.Reductor(ctx1, dtype, L.SUM)(z - t), rel=1e-5 if dtype == np.float32 else 1e-12)


def test_inline_switches(ctx1, params):
    rng = np.random.default_rng(6)
    n = SIGMA + 1
    A = sell(ctx1, n, n, matrix(rng, n, n, np.float64))
    params("spmv.sell_inline", 0)
    assert sweep_strip(A) is None
    check_inline(ctx1, n, np.float64, rng, e_add, [A], launches=2)          # the sweep of z, then the product appended
    params("spmv.sell_inline", 1)
    params("spmv.no_inline", 1)
    assert sweep_strip(A) is None
    check_inline(ctx1, n, np.float64, rng, e_add, [A], launches=2)


@pytest.mark.parametrize("coupled", [False, True])
@pytest.mark.parametrize("which", ["ctx2", "ctx3"])
def test_inline_on_several_parts(request, params, which, coupled):
    ctx = request.getfixturevalue(which)
    rng = np.random.default_rng(18)
    n = 3 * SIGMA + 50
    A = sell(ctx, n, n, block_diagonal(rng, ctx, n, np.float64, coupled))
    assert all((sweep_strip(A, k) is None) == coupled for k in ctx.local)
    check_inline(ctx, n, np.float64, rng, e_index, [A], launches=None if coupled else 1)
    if not coupled:
        check_inline(ctx, n, np.float64, rng, e_add, [A])
        return
    # a coupled matrix falls back: `y = z + A*x` keeps the unfused path, which appends the local and the remote strip to z
    # one after the other -- the bits it has with the sweep switched off
    x, z = vx.vector(ctx, values(rng, n, np.float64)), vx.vector(ctx, values(rng, n, np.float64))
    y1, y0 = vx.vector(ctx, n), vx.vector(ctx, n)
    y1.assign(z + A * x)
    params("spmv.sell_inline", 0)
    y0.assign(z + A * x)
    assert_same(y1.read(), y0.read())


@pytest.mark.parametrize("dtype", DTYPES)
def test_nothing_is_written_past_n(ctx1, params, dtype):
    """Vectors 64 elements longer than the strip, the tail holding a sentinel."""
    rng = np.random.default_rng(8)
    n, G = SIGMA + 7, 64
    A = sell(ctx1, n, n, matrix(rng, n, n, dtype))
    x = vx.vector(ctx1, values(rng, n, dtype))
    sentinel = dtype(-12345.5)
    Y0 = np.concatenate([values(rng, n, dtype), np.full(G, sentinel, dtype)])
    z = vx.vector(ctx1, Y0)
    # one kernel: y[0, n) = z + A*x
    y = vx.vector(ctx1, Y0)
    low = _Lowering(0, 0)
    low.size, low.sweep = n + G, None
    low.lower(wrap(z) + vx.make_inline(A * x))
    L.check(L.lib().vexb_eval(ctx1.devs[0], ctx1.streams[0], y.bufs[0], y.dtype, L.SET, C.byref(low.e), n, 0))
    t = vx.vector(ctx1, n, dtype)
    A.apply(x, t)
    assert_same(y.read()[:n], Y0[:n] + t.read())
    assert_same(y.read()[n:], Y0[n:])
    # three vectors in one pass
    ys = [vx.vector(ctx1, Y0) for _ in range(3)]
    xs = [vx.vector(ctx1, values(rng, n, dtype)) for _ in range(3)]
    xa = (C.c_void_p * 3)(*[v.bufs[0] for v in xs])
    ya = (C.c_void_p * 3)(*[v.bufs[0] for v in ys])
    L.check(L.lib().vexb_spmv_multi(ctx1.devs[0], ctx1.streams[0], sweep_strip(A), 3, xa, ya, 1.0, 0))
    for k in range(3):
        A.apply(xs[k], t)
        assert_same(ys[k].read()[:n], t.read())
        assert_same(ys[k].read()[n:], Y0[n:])


def test_cpp_front_end(built):
    """tests/cpp/test_sell_fused.cpp on two partition slots and on one."""
    build.build_cpp_tests()
    exe = build.ROOT / "tests" / "cpp" / "bin" / "test_sell_fused"
    for parts in ("2", "1"):
        r = subprocess.run([str(exe), "42"], capture_output=True, text=True, env={**os.environ, "VEXCL_TEST_PARTS": parts})
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
