"""vex::make_temp on the GPU.  The contract: an expression with make_temp(tag, e, T) has the bits of the same expression with
T(e) written out at every use, on every path -- the interpreter (eval.force_interp = 1), the NVRTC kernel (eval.jit = 1), the
default mode once its background compilation is done, the generated reductions, the multi-expression kernel and the
kernels with inlined sparse products.  The written-out twin is the same tree lowered with every temporary expanded in
place (`expanded` below).  Reference closed forms: tests/temporary.cpp."""
import ctypes as C
import time

import numpy as np
import pytest

import vexcl_b200 as vx
from vexcl_b200 import api, _lib as L

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 1023, 1024, 1025]
FLOAT = [np.float64, np.float32]
ALL = [np.float64, np.float32, np.int32, np.uint64]
CTXS = ["ctx1", "ctx2"]


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({8: np.uint64, 4: np.uint32}[a.dtype.itemsize])


def same(got, want, what=""):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape and np.array_equal(g, w), f"{what}: {np.count_nonzero(g != w)} of {g.size} differ"


def wait_jit():
    p = C.c_int(1)
    while p.value:
        L.check(L.lib().vexb_jit_pending(C.byref(p)))
        time.sleep(0.01)


def _expand(self, n):
    self.lower(n.a)
    self.cvt(n.a.dtype, n.dtype)


class expanded:
    """Within the block every temporary is lowered as T(e) written out at its use."""
    def __enter__(self):
        self.saved = api._Lowering.temp
        api._Lowering.temp = _expand
    def __exit__(self, *a):
        api._Lowering.temp = self.saved


MODES = {"interp": {"eval.force_interp": 1, "eval.jit": 0}, "jit": {"eval.jit": 1}, "background": {}}


@pytest.fixture
def mode(request, built):
    name = request.param
    for k, v in MODES[name].items():
        vx.set_param(k, v)
    try:
        yield name
    finally:
        vx.set_param("eval.force_interp", 0)
        vx.set_param("eval.jit", 2)


def values(rng, n, dt):
    if np.dtype(dt).kind == "f":
        return (rng.random(n) + 0.25).astype(dt)
    return rng.integers(1, 100, n).astype(dt)


def exprs(dt, x, y):
    """Temporaries read several times, nested, and one read in one if_else branch only."""
    # small enough that the written-out twin stays within 16 terminals
    if np.dtype(dt).kind == "f":
        t1 = vx.make_temp(1, vx.sin(x) + y)
        t2 = vx.make_temp(2, t1 * x)
        s = vx.make_temp(3, vx.sqrt(y))
        return (t1 - t2) * (t1 + t2) + vx.if_else(x > 0.75, s, x)
    t1 = vx.make_temp(1, x * y)
    t2 = vx.make_temp(2, t1 ^ x)
    s = vx.make_temp(3, y * y)
    return t1 * t2 + (t2 - t1) + vx.if_else(x > 50, s, x)


def run(ctx, dt, n, op, mk, y0):
    rng = np.random.default_rng(n + 7)
    vec = lambda a: vx.vector(ctx, a) if a.size else vx.vector(ctx, 0, dt)
    x, y = vec(values(rng, n, dt)), vec(values(rng, n, dt))
    got, want = vec(y0), vec(y0)
    got._assign(op, mk(dt, x, y))
    with expanded():
        want._assign(op, mk(dt, x, y))
    wait_jit()
    got2, want2 = vec(y0), vec(y0)                         # the default mode's second use: the specialised kernel
    got2._assign(op, mk(dt, x, y))
    with expanded():
        want2._assign(op, mk(dt, x, y))
    return got.read(), want.read(), got2.read(), want2.read()


OPS_F = [L.SET, L.ADD, L.SUB, L.MUL, L.DIV]
OPS_I = OPS_F + [L.MOD, L.AND, L.OR, L.XOR, L.LSH, L.RSH]


@pytest.mark.parametrize("mode", list(MODES), indirect=True)
@pytest.mark.parametrize("dt", ALL, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("cx", CTXS)
def test_every_assignment_operator_has_the_written_out_bits(request, mode, dt, cx):
    ctx = request.getfixturevalue(cx)
    n = 10007
    y0 = values(np.random.default_rng(1), n, dt)
    for op in (OPS_F if np.dtype(dt).kind == "f" else OPS_I):
        g, w, g2, w2 = run(ctx, dt, n, op, exprs, y0)
        same(g, w, f"{mode} op {op}")
        same(g2, w2, f"{mode} op {op}, second use")


def _grid_sizes():
    p = L.DevProps()
    L.check(L.lib().vexb_device_props(0, C.byref(p)))
    interp = p.sm_count * 4 * 1024                      # interpreter: interp.blocks_per_sm x 1024 elements per block
    jit = p.sm_count * 64 * 1024                        # generated kernel: 64 blocks per SM x 1024
    return [interp - 1, interp, interp + 1, 2 * interp + 1, jit + 1]


@pytest.mark.parametrize("mode", list(MODES), indirect=True)
@pytest.mark.parametrize("cx", CTXS)
def test_sizes_and_the_grid_stride_loop(request, mode, cx):
    ctx = request.getfixturevalue(cx)
    for dt in (np.float64, np.int32):
        for n in SIZES + _grid_sizes():
            y0 = values(np.random.default_rng(2), n, dt)
            g, w, g2, w2 = run(ctx, dt, n, L.SET, exprs, y0)
            same(g, w, f"{mode} n={n}")
            same(g2, w2, f"{mode} n={n}, second use")


@pytest.mark.parametrize("mode", list(MODES), indirect=True)
@pytest.mark.parametrize("cx", CTXS)
def test_an_explicit_float_temporary_of_double_operands(request, mode, cx):
    ctx = request.getfixturevalue(cx)
    n = 4099
    X = values(np.random.default_rng(3), n, np.float64)
    x, y = vx.vector(ctx, X), vx.vector(ctx, n)
    t = vx.make_temp(1, x * 3.0 + 1.0, np.float32)
    y.assign(t * x)
    wait_jit()
    y.assign(t * x)
    same(y.read(), (X * 3.0 + 1.0).astype(np.float32).astype(np.float64) * X, mode)


def udf():
    return api.UserFunction(np.float64, "tsq", [(np.float64, "v")], "return v * v + 0.5;")


@pytest.mark.parametrize("mode", list(MODES), indirect=True)
@pytest.mark.parametrize("cx", CTXS)
@pytest.mark.parametrize("call", [False, True])
def test_reductions_have_the_written_out_bits(request, mode, cx, call):
    ctx = request.getfixturevalue(cx)
    f = udf()
    for dt in (np.float64, np.float32, np.int32):
        rng = np.random.default_rng(4)
        n = 30007
        x, y = vx.vector(ctx, values(rng, n, dt)), vx.vector(ctx, values(rng, n, dt))
        def mk():
            if np.dtype(dt).kind == "f":
                t = vx.make_temp(1, f(x) if call else vx.cos(x) * y)
                return t * t - t / y
            t = vx.make_temp(1, x * 7 + y)
            return t * (t % 13) - y
        for kind in (L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.MINMAX, [L.SUM, L.MAX, L.MIN, L.SUM_KAHAN]):
            R = vx.Reductor(ctx, dt, kind)
            got = R(mk())
            wait_jit()
            got2 = R(mk())
            with expanded():
                want = R(mk())
            assert np.array_equal(np.asarray(got, dtype=dt), np.asarray(want, dtype=dt)), (dt, kind)
            assert np.array_equal(np.asarray(got2, dtype=dt), np.asarray(want, dtype=dt)), (dt, kind)


@pytest.mark.parametrize("cx", CTXS)
def test_reference_reduce_temporary(request, cx):
    ctx = request.getfixturevalue(cx)
    n = 1024
    x = vx.vector(ctx, np.random.default_rng(5).random(n))
    t1 = vx.make_temp(1, vx.pow_(vx.sin(x), 2.0))
    t2 = vx.make_temp(2, vx.pow_(vx.cos(x), 2.0))
    s = vx.Reductor(ctx, np.float64, L.SUM)(10 * (t1 + t2))
    assert abs(s - 10.0 * n) <= 1e-8 * 10.0 * n                     # BOOST_CHECK_CLOSE(..., 1e-6) is in percent


def fused_multi(ctx, lhs, rhs):
    """assign_multi once the kernel exists, in one launch per slot."""
    vx.assign_multi(lhs, rhs)
    wait_jit()
    ctx.finish()
    l0 = vx.launch_count()
    assert vx.assign_multi(lhs, rhs), "the multi-expression kernel did not serve the request"
    ctx.finish()
    assert vx.launch_count() - l0 == len(ctx.local)


@pytest.mark.parametrize("cx", CTXS)
@pytest.mark.parametrize("dt", FLOAT, ids=lambda d: np.dtype(d).name)
def test_tie_and_multivector_temporaries_in_one_launch(request, cx, dt):
    ctx = request.getfixturevalue(cx)
    n = 100003
    rng = np.random.default_rng(6)
    X = rng.random(n).astype(dt)
    x = vx.vector(ctx, X)
    a, b, ra, rb = (vx.vector(ctx, n, dt) for _ in range(4))
    t = vx.make_temp(1, vx.sin(x))
    fused_multi(ctx, [a, b], [t, vx.sqrt(1.0 - t * t)])             # y = std::tie(tmp, sqrt(1 - tmp * tmp))
    ra.assign(t)
    rb.assign(vx.sqrt(1.0 - t * t))
    same(a.read(), ra.read(), "tie component 0")
    same(b.read(), rb.read(), "tie component 1")
    tol = 1e-10 if dt == np.float64 else 1e-6
    assert np.allclose(a.read(), np.sin(X.astype(np.float64)), rtol=tol)
    assert np.allclose(b.read(), np.cos(X.astype(np.float64)), rtol=tol)
    # a multivector temporary (make_temp<1, double>(tan(x)), y = tmp * tmp): each component its own
    x0, x1 = vx.vector(ctx, rng.random(n).astype(dt)), vx.vector(ctx, rng.random(n).astype(dt))
    t0, t1 = vx.make_temp(1, vx.tan(x0)), vx.make_temp(1, vx.tan(x1))
    fused_multi(ctx, [a, b], [t0 * t0, t1 * t1])
    ra.assign(t0 * t0)
    rb.assign(t1 * t1)
    same(a.read(), ra.read(), "multivector component 0")
    same(b.read(), rb.read(), "multivector component 1")
    X0 = x0.read().astype(np.float64)
    assert np.allclose(a.read(), np.tan(X0) ** 2, rtol=tol * 10)


# ------------------------------------------------------------------------------------------------ sparse products

def values_pm(rng, size, dtype):
    return ((rng.random(size) + 0.5) * np.where(rng.random(size) < 0.5, -1.0, 1.0)).astype(dtype)


def banded(rng, n, dtype, w=9):
    cols, rows = [], [0]
    for i in range(n):
        c = np.arange(max(0, i - w // 2), min(n, i + w // 2 + 1))
        cols.append(c)
        rows.append(rows[-1] + c.size)
    col = np.concatenate(cols).astype(np.int64)
    return np.array(rows, np.int64), col, values_pm(rng, col.size, dtype)


def irregular(rng, n, dtype):
    w = rng.integers(0, 40, n)
    w[rng.random(n) < 0.01] = 300
    cols = [np.sort(rng.choice(n, size=min(k, n), replace=False)) for k in w]
    row = np.concatenate([[0], np.cumsum([c.size for c in cols])]).astype(np.int64)
    return row, np.concatenate(cols).astype(np.int64), values_pm(rng, int(row[-1]), dtype)


def product_case(ctx, A, x, n, dtype, what):
    p = vx.vector(ctx, n, dtype)
    p.assign(vx.make_inline(A * x))                                    # the product into a vector, by the same row code
    want = vx.vector(ctx, n, dtype)
    want.assign(p * p + p - vx.sin(p))
    got = vx.vector(ctx, n, dtype)
    t = vx.make_temp(1, vx.make_inline(A * x))
    got.assign(t * t + t - vx.sin(t))                                  # first use: compiles
    ctx.finish()
    l0 = vx.launch_count()
    got.assign(t * t + t - vx.sin(t))
    ctx.finish()
    assert vx.launch_count() - l0 == len(ctx.local), what
    same(got.read(), want.read(), what)
    s = vx.Reductor(ctx, dtype, L.SUM)
    with expanded():
        r_want = s(t * t + t)
    assert np.array_equal(np.asarray(s(t * t + t), dtype), np.asarray(r_want, dtype)), what


@pytest.mark.parametrize("dt", FLOAT, ids=lambda d: np.dtype(d).name)
def test_temporaries_of_inlined_products(ctx1, dt):
    rng = np.random.default_rng(8)
    n = 20000
    X = values_pm(rng, n, dt)
    x = vx.vector(ctx1, X)
    for fmt, mat, name in ((vx.FMT_CSR, irregular(rng, n, dt), "csr"), (vx.FMT_HELL, banded(rng, n, dt), "hybrid ELL"),
                           (vx.FMT_SELL, irregular(rng, n, dt), "sliced ELL")):
        A = vx.SpMat(ctx1, n, n, *mat, fmt)
        product_case(ctx1, A, x, n, dt, name)
    # SpMatCCSR: the 1-D Laplacian's unique rows
    idx = np.ones(n, np.uint64); idx[0] = idx[-1] = 0
    C_ = vx.SpMatCCSR(ctx1, n, idx, np.array([0, 1, 4], np.uint64), np.array([0, -1, 0, 1], np.int64),
                      np.array([1, -1, 2, -1], dt))
    p = vx.vector(ctx1, n, dt)
    C_.apply(x, p)
    want, got = vx.vector(ctx1, n, dt), vx.vector(ctx1, n, dt)
    want.assign(p * x + vx.sin(p))
    t = vx.make_temp(2, vx.make_inline(C_ * x))
    got.assign(t * x + vx.sin(t))
    ctx1.finish()
    l0 = vx.launch_count()
    got.assign(t * x + vx.sin(t))
    ctx1.finish()
    assert vx.launch_count() - l0 == 1
    same(got.read(), want.read(), "ccsr")


def test_temporaries_of_inlined_products_on_two_slots(ctx2):
    """Two slots on one device: strips with a halo cannot be inlined and take a product temporary; the bits stay."""
    rng = np.random.default_rng(9)
    n = 20000
    x = vx.vector(ctx2, values_pm(rng, n, np.float64))
    A = vx.SpMat(ctx2, n, n, *banded(rng, n, np.float64), vx.FMT_HELL)
    p = vx.vector(ctx2, n)
    A.apply(x, p)
    want, got = vx.vector(ctx2, n), vx.vector(ctx2, n)
    want.assign(p * p + p)
    t = vx.make_temp(1, vx.make_inline(A * x))
    got.assign(t * t + t)
    same(got.read(), want.read(), "two slots")


def test_refusals_on_the_device_entry_points(ctx1):
    lib = L.lib()
    n = 1024
    x, y = vx.vector(ctx1, n), vx.vector(ctx1, n)
    e = L.Expr()
    e.term[0].kind, e.term[0].dtype, e.term[0].v.ptr = L.TERM_VEC, L.F64, x.bufs[0].value
    e.n_terms = 1
    for k, (op, typ, arg) in enumerate([("TERM", L.F64, 0), ("TDEF", L.F32, 0), ("TREF", L.F32, 0)]):
        e.code[k].op, e.code[k].type, e.code[k].arg = L.OP[op], typ, arg
    e.n_code = 3
    dev, st = ctx1.devs[0], ctx1.streams[0]
    assert lib.vexb_eval(dev, st, y.bufs[0], L.F64, L.SET, C.byref(e), n, 0) == L.ERR_INVALID
    ws_bytes = C.c_size_t(0)
    L.check(lib.vexb_reduce_workspace_bytes(dev, C.byref(ws_bytes)))
    ws, res = vx.vector(ctx1, ws_bytes.value // 8 + 8), vx.vector(ctx1, 16)
    assert lib.vexb_reduce(dev, st, C.byref(e), L.F64, n, 0, L.SUM, res.bufs[0], ws.bufs[0]) == L.ERR_INVALID
    ops = (C.c_int * 2)(L.SUM, L.MAX)
    assert lib.vexb_reduce_multi(dev, st, C.byref(e), L.F64, n, 0, 2, ops, res.bufs[0], ws.bufs[0], None) == L.ERR_INVALID
    es = (C.POINTER(L.Expr) * 2)(C.pointer(e), C.pointer(e))
    out = (C.c_void_p * 2)(y.bufs[0], x.bufs[0])
    h = C.c_int(0)
    assert lib.vexb_eval_multi(dev, st, 2, out, L.F64, L.SET, es, n, 0, C.byref(h)) == L.ERR_INVALID
    ctx1.finish()
