"""vex::SpMatCCSR products as expression terminals (VEXB_TERM_CCSR) on the GPU, every value compared on its bits in
float64 and float32.  The reference of each case is the same expression with the product replaced by a device temporary
from A.apply; the terminal alone must also equal oracle.ccsr.ccsr_spmv.  Covers: builtins, products, the same terminal
twice, two CCSR matrices, a CCSR terminal beside an inlined SpMat product (CSR and hybrid ELL), a VEX_FUNCTION, a device
scalar, if_else; =, +=, -=, *=, /=; SUM, SUM_KAHAN, MIN, MAX, MIN_MAX and combined reductions at reduce.blocks_per_sm 1,
8 and 16; sizes around the block and the grid-stride loop, idx widths 1, 2 and 4, an empty unique row, the reference's
32^3 Poisson matrix, 32- and 64-bit input index types; one launch per call, guard elements past n, aliasing, refusals,
vexb_eval_multi; and tests/cpp/test_ccsr_terms.cpp."""
import contextlib
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
from oracle import ccsr
import vexcl_b200 as vx
from vexcl_b200 import _lib as L
from vexcl_b200 import api, gen

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
DEFAULTS = {"reduce.blocks_per_sm": 8}
BIN = Path(__file__).resolve().parent / "cpp" / "bin"


@contextlib.contextmanager
def param(name, value):
    old = C.c_long()
    prev = old.value if L.lib().vexb_get_param(name.encode(), C.byref(old)) == L.OK else DEFAULTS[name]
    vx.set_param(name, value)
    try:
        yield
    finally:
        vx.set_param(name, prev)


def bits(v, dtype):
    a = np.asarray(v, dtype)
    return a.view({8: np.uint64, 4: np.uint32}[a.itemsize])


def same(got, want, dtype, what=""):
    g, w = bits(got, dtype), bits(want, dtype)
    bad = np.nonzero(g != w)[0] if g.ndim else ([0] if g != w else [])
    assert len(bad) == 0, f"{what}: {len(bad)} elements differ, first at {bad[:5]}: {np.asarray(got).ravel()[bad[:3]]} vs {np.asarray(want).ravel()[bad[:3]]}"


def mixed(rng, n, dtype):
    """sign * U[1, 2) * 2^k: sums of these depend on the order of additions."""
    v = rng.uniform(1, 2, n) * np.exp2(rng.integers(-12, 13, n)) * rng.choice([-1.0, 1.0], n)
    return v.astype(dtype)


def random_ccsr(n, m, seed, dtype, reach=40, index_dtype=np.uint64, col_dtype=np.int64):
    """n rows over m unique rows: unique row 0 is the diagonal (rows within `reach` of an end use it), unique row 1 has
    no entries, the others 1..9 entries at offsets in [-reach, reach]."""
    rng = np.random.default_rng(seed)
    widths = rng.integers(1, 10, m)
    widths[0] = 1
    if m > 1:
        widths[1] = 0
    row = np.concatenate([[0], np.cumsum(widths)]).astype(index_dtype)
    col = rng.integers(-reach, reach + 1, int(row[-1])).astype(col_dtype)
    col[0] = 0
    val = mixed(rng, int(row[-1]), dtype)
    idx = rng.integers(0, m, n) if m > 1 else np.zeros(n, np.int64)
    i = np.arange(n)
    idx[(i < reach) | (i >= n - reach)] = 0
    idx[(i < reach) & (i % 3 == 1) & (m > 1)] = 1             # empty rows near the ends too
    return idx.astype(index_dtype), row, col, val


def ccsr_by_entry(n, idx, row, col, val, x):
    """oracle.ccsr.ccsr_spmv restated entry by entry instead of unique row by unique row (same operations on every row, in
    the same order): for matrices with many unique rows, where the oracle's loop over them is too slow."""
    idx, row, col = idx.astype(np.int64), row.astype(np.int64), col.astype(np.int64)
    start, width = row[idx], row[idx + 1] - row[idx]
    i = np.arange(n)
    s = np.zeros(n, dtype=val.dtype)
    for j in range(int(width.max()) if n else 0):
        on = np.nonzero(width > j)[0]
        e = start[on] + j
        s[on] = s[on] + val[e] * x[i[on] + col[e]]
    return s


class Case:
    """A CCSR matrix, x, and the temporary t = A*x from A.apply."""

    def __init__(self, ctx, n, m, seed, dtype, **kw):
        self.ctx, self.n, self.dtype = ctx, n, dtype
        self.idx, self.row, self.col, self.val = random_ccsr(n, m, seed, dtype, **kw)
        self.A = vx.SpMatCCSR(ctx, n, self.idx, self.row, self.col, self.val)
        rng = np.random.default_rng(seed + 1)
        self.xh = mixed(rng, n, dtype)
        self.x = vx.vector(ctx, self.xh)
        self.t = vx.vector(ctx, n, dtype)
        self.A.apply(self.x, self.t)
        spmv = ccsr.ccsr_spmv if m <= 300 or n <= 200_000 else ccsr_by_entry
        self.want = spmv(n, self.idx, self.row, self.col, self.val, self.xh)


def poisson_case(ctx, dtype, n=32):
    c = Case.__new__(Case)
    N = n ** 3
    c.ctx, c.n, c.dtype = ctx, N, dtype
    c.idx, c.row, c.col, c.val = gen.poisson_ccsr(n)
    c.val = c.val.astype(dtype)
    c.A = vx.SpMatCCSR(ctx, N, c.idx, c.row, c.col, c.val)
    c.xh = oracle.uniform_real(3, N).astype(dtype)
    c.x = vx.vector(ctx, c.xh)
    c.t = vx.vector(ctx, N, dtype)
    c.A.apply(c.x, c.t)
    c.want = ccsr.ccsr_spmv(N, c.idx, c.row, c.col, c.val, c.xh)
    return c


def one_launch(fn):
    fn()                                                       # warm: the kernel is generated at first use
    n0 = vx.launch_count()
    r = fn()
    assert vx.launch_count() - n0 == 1
    return r


def assign_pair(c, mk, op=L.SET, y0=None):
    """y op= mk(A*x) and y op= mk(t): (fused result, reference result)."""
    y0 = np.zeros(c.n, c.dtype) if y0 is None else y0
    out = []
    for p in (c.A * c.x, c.t):
        y = vx.vector(c.ctx, y0)
        y._assign(op, mk(p))
        out.append(y.read())
    return out


# ---- the terminal alone --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,width", [(3, 1), (300, 2), (70_000, 4)])
def test_terminal_equals_the_product(ctx1, dtype, m, width):
    c = Case(ctx1, 100_003, m, 11, dtype)
    assert c.A.info().idx_bytes == width
    same(c.t.read(), c.want, dtype, "A.apply vs oracle")
    y = vx.vector(ctx1, c.n, dtype)
    one_launch(lambda: y.assign(vx.make_inline(c.A * c.x)))
    same(y.read(), c.want, dtype, "make_inline(A*x)")
    y.assign(vx.make_inline(c.A * c.x) + dtype(0) * c.x)       # an expression around it, not an additive spelling
    same(y.read(), c.want + dtype(0) * c.xh, dtype, "make_inline(A*x) + 0*x")
    if m == 300:
        same(ccsr_by_entry(c.n, c.idx, c.row, c.col, c.val, c.xh), c.want, dtype, "restatement vs oracle")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("index_dtype,col_dtype", [(np.uint32, np.int32), (np.uint64, np.int64)])
def test_poisson_32_rows_reach_n_squared(ctx1, dtype, index_dtype, col_dtype):
    n = 32
    c = poisson_case(ctx1, dtype, n)
    idx, row, col, val = gen.poisson_ccsr(n, index_dtype=index_dtype, col_dtype=col_dtype)
    A = vx.SpMatCCSR(ctx1, n ** 3, idx, row, col, val.astype(dtype))
    assert int(np.abs(col).max()) == n * n
    y = vx.vector(ctx1, c.n, dtype)
    y.assign(vx.sin(A * c.x))
    same(y.read(), assign_pair(c, lambda p: vx.sin(p))[1], dtype, "sin(A*x)")
    y.assign(c.x * (A * c.x))
    same(y.read(), c.xh * c.want, dtype, "x * (A*x)")


# ---- expressions ---------------------------------------------------------------------------------------------------
def spmat(ctx, c, fmt):
    """A SpMat (CSR or hybrid ELL) of the same size, to inline beside the CCSR terminal."""
    row, col, val = oracle.tridiagonal(c.n)
    return vx.SpMat(ctx, c.n, c.n, row, col, val.astype(c.dtype), fmt)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["sin", "x_times", "twice", "two_matrices", "csr_beside", "hell_beside", "user_function",
                                  "device_scalar", "if_else", "scaled"])
def test_expressions(ctx1, dtype, name):
    c = Case(ctx1, 50_001, 300, 21, dtype)
    B = Case(ctx1, 50_001, 3, 22, dtype)
    B.A.apply(c.x, B.t)                                        # B's product of c's x
    sq = api.UserFunction(dtype, "sq_" + np.dtype(dtype).name, [(dtype, "a")], "return a * a;")
    ds = api.DeviceScalar(ctx1, dtype, 0.75)
    S = {"csr_beside": vx.FMT_CSR, "hell_beside": vx.FMT_HELL}.get(name)
    S = spmat(ctx1, c, S) if S is not None else None
    x = c.x
    exprs = {
        "sin": lambda p, q: vx.sin(p),
        "x_times": lambda p, q: x * p,
        "twice": lambda p, q: p * p + x,
        "two_matrices": lambda p, q: p * q - x,
        "csr_beside": lambda p, q: p * vx.make_inline(S * x),
        "hell_beside": lambda p, q: vx.make_inline(S * x) + p * x,
        "user_function": lambda p, q: sq(p) + x,
        "device_scalar": lambda p, q: ds * p + x,
        "if_else": lambda p, q: vx.if_else(p > 0, x, p * dtype(0.5)),
        "scaled": lambda p, q: x * (dtype(2) * p) + (p / dtype(4)) * x,
    }
    mk = exprs[name]
    y, ref = vx.vector(ctx1, c.n, dtype), vx.vector(ctx1, c.n, dtype)
    one_launch(lambda: y.assign(mk(c.A * x, B.A * x)))
    ref.assign(mk(c.t, B.t))
    same(y.read(), ref.read(), dtype, name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("op", [L.SET, L.ADD, L.SUB, L.MUL, L.DIV])
def test_assignment_operators(ctx1, dtype, op):
    c = Case(ctx1, 40_000, 300, 31, dtype)
    y0 = mixed(np.random.default_rng(3), c.n, dtype)
    for mk in (lambda p: c.x * p, lambda p: vx.sin(p)):
        got, want = assign_pair(c, mk, op, y0)
        same(got, want, dtype, f"op {op}")
    if op in (L.MUL, L.DIV):                                   # y *= A*x: the product itself as the right-hand side
        got, want = assign_pair(c, lambda p: p, op, y0)
        same(got, want, dtype, f"op {op}, bare product")


# ---- reductions ----------------------------------------------------------------------------------------------------
KINDS = [L.SUM, L.SUM_KAHAN, L.MIN, L.MAX, L.MINMAX, (L.SUM, L.MAX, L.MIN, L.SUM_KAHAN)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bps", [1, 8, 16])
def test_reductions(ctx1, dtype, bps):
    with param("reduce.blocks_per_sm", bps):
        for n in (1, 257, 1025, 300_001):
            c = Case(ctx1, n, 300 if n > 1000 else 3, 41 + n, dtype)
            for kind in KINDS:
                red = vx.Reductor(ctx1, dtype, list(kind) if isinstance(kind, tuple) else kind)
                for mk in (lambda p: c.x * p, lambda p: p):
                    got = one_launch(lambda: red(mk(c.A * c.x)))
                    want = red(mk(c.t))
                    same(np.asarray(got), np.asarray(want), dtype, f"n={n} kind={kind} bps={bps}")


def test_energy_norm_poisson(ctx1):
    c = poisson_case(ctx1, np.float64)
    red = vx.Reductor(ctx1, np.float64, L.SUM)
    same(red(c.x * (c.A * c.x)), red(c.x * c.t), np.float64, "sum(x * (A*x))")


# ---- edges ---------------------------------------------------------------------------------------------------------
def grid_sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    turn = sms * 64 * 256                                      # elements of one turn of the capped grid
    return [1, 255, 256, 257, 1023, 1024, 1025, turn + 1000, 2 * turn - 1]


@pytest.mark.parametrize("dtype", DTYPES)
def test_sizes_widths_and_guards(ctx1, dtype):
    lib = L.lib()
    for n in grid_sizes():
        for m in ((3, 300, 70_000) if n > 100_000 else (3, 300)):
            c = Case(ctx1, n, m, 51 + n % 97, dtype)
            same(c.t.read(), c.want, dtype, f"n={n} m={m} A.apply vs oracle")
            guard = 64
            big = vx.vector(ctx1, np.full(n + guard, -7.0, dtype))
            low = api._Lowering(0, 0)
            low.size = n
            low.lower(vx.sin(c.A * c.x) * c.x)

            def run():
                L.check(lib.vexb_eval(ctx1.devs[0], ctx1.streams[0], big.bufs[0], api._vdt(dtype), L.SET, C.byref(low.e), n, 0))
            one_launch(run)
            ref = vx.vector(ctx1, n, dtype)
            ref.assign(vx.sin(c.t) * c.x)
            out = big.read()
            same(out[:n], ref.read(), dtype, f"n={n} m={m}")
            same(out[n:], np.full(guard, -7.0, dtype), dtype, f"n={n} m={m}: guard elements")


# ---- aliasing, refusals, multi-expressions -------------------------------------------------------------------------
def raw_ccsr_expr(c, x_ptr, dtype=None, width=None, x_kind=L.TERM_VEC):
    """x * (A*x) by hand: terminal 0 = x, 1 = the CCSR product."""
    dt = api._vdt(c.dtype) if dtype is None else dtype
    e = L.Expr()
    e.n_terms = 2
    e.term[0].kind, e.term[0].dtype, e.term[0].v.ptr = x_kind, dt, x_ptr
    e.term[1].kind, e.term[1].dtype, e.term[1].v.ptr = L.TERM_CCSR, dt, c.A.h.value
    e.term[1].pad[0], e.term[1].pad[1] = 0, c.A.idx_bytes if width is None else width
    for k, (op, arg) in enumerate((("TERM", 0), ("TERM", 1), ("MUL", 0))):
        e.code[k].op, e.code[k].type, e.code[k].arg = L.OP[op], dt, arg
    e.n_code = 3
    return e


@pytest.mark.parametrize("dtype", DTYPES)
def test_aliasing(ctx1, dtype):
    c = Case(ctx1, 30_000, 300, 61, dtype)
    x2 = vx.vector(ctx1, c.xh)
    x2.assign(vx.sin(c.A * x2))                                # x = sin(A*x): the product goes to a temporary first
    same(x2.read(), np.asarray(assign_pair(c, lambda p: vx.sin(p))[1]), dtype, "x = sin(A*x)")
    x3 = vx.vector(ctx1, c.xh)
    x3 *= c.A * x3
    same(x3.read(), c.xh * c.want, dtype, "x *= A*x")
    e = raw_ccsr_expr(c, c.x.bufs[0].value)
    st = L.lib().vexb_eval(ctx1.devs[0], ctx1.streams[0], c.x.bufs[0], api._vdt(dtype), L.SET, C.byref(e), c.n, 0)
    assert st == L.ERR_UNSUPPORTED
    same(c.x.read(), c.xh, dtype, "x untouched by the refused call")


def test_refusals(ctx1):
    c = Case(ctx1, 20_000, 300, 71, np.float64)
    y = vx.vector(ctx1, c.n)
    lib, dev, st = L.lib(), ctx1.devs[0], ctx1.streams[0]
    xf = vx.vector(ctx1, c.xh.astype(np.float32))
    yf = vx.vector(ctx1, c.n, np.float32)
    ev = lambda e, n=c.n, off=0, lhs=y, dt=L.F64: lib.vexb_eval(dev, st, lhs.bufs[0], dt, L.SET, C.byref(e), n, off)
    assert ev(raw_ccsr_expr(c, c.x.bufs[0].value)) == L.OK
    assert ev(raw_ccsr_expr(c, xf.bufs[0].value, dtype=L.F32), lhs=yf, dt=L.F32) == L.ERR_INVALID     # value type
    assert ev(raw_ccsr_expr(c, c.x.bufs[0].value), n=c.n - 1) == L.ERR_INVALID                        # part of the matrix
    assert ev(raw_ccsr_expr(c, c.x.bufs[0].value), n=c.n - 16, off=16) == L.ERR_INVALID
    assert ev(raw_ccsr_expr(c, c.x.bufs[0].value, width=4)) == L.ERR_INVALID                          # idx width
    assert ev(raw_ccsr_expr(c, c.x.bufs[0].value, x_kind=L.TERM_SCALAR)) == L.ERR_INVALID             # x not a vector
    e = raw_ccsr_expr(c, c.x.bufs[0].value)
    ws, r = ctx1.workspace(0)
    assert lib.vexb_reduce_all(dev, st, C.byref(e), L.F64, c.n - 1, 0, L.SUM, r, ws, None) == L.ERR_INVALID
    ops = (C.c_int * 2)(L.SUM, L.MAX)
    ws2, r2 = ctx1.workspace(0, 2)
    assert lib.vexb_reduce_multi(dev, st, C.byref(e), L.F64, c.n, 8, 2, ops, r2, ws2, None) == L.ERR_INVALID
    same(y.read(), c.xh * c.want, np.float64, "only the accepted call wrote y")


@pytest.mark.parametrize("dtype", DTYPES)
def test_eval_multi_not_handled(ctx1, dtype):
    c = Case(ctx1, 30_000, 3, 81, dtype)
    e0, e1 = api._Lowering(0, 0), api._Lowering(0, 0)
    e0.size = e1.size = c.n
    e0.lower(api.wrap(c.x * (c.A * c.x)))
    e1.lower(api.wrap(vx.sin(c.A * c.x)))
    a, b = vx.vector(ctx1, c.n, dtype), vx.vector(ctx1, c.n, dtype)
    es = (C.POINTER(L.Expr) * 2)(C.pointer(e0.e), C.pointer(e1.e))
    out = (C.c_void_p * 2)(a.bufs[0], b.bufs[0])
    handled = C.c_int(1)
    L.check(L.lib().vexb_eval_multi(ctx1.devs[0], ctx1.streams[0], 2, out, api._vdt(dtype), L.SET, es, c.n, 0, C.byref(handled)))
    assert handled.value == 0
    assert api.assign_multi([a, b], [c.x * (c.A * c.x), vx.sin(c.A * c.x)]) is False
    same(a.read(), c.xh * c.want, dtype, "component 0")
    ref = vx.vector(ctx1, c.n, dtype)
    ref.assign(vx.sin(c.t))
    same(b.read(), ref.read(), dtype, "component 1")


def test_cpp_front_end(built):
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = BIN / "test_ccsr_terms"
    assert exe.exists(), f"{exe} was not built"
    for parts in ("1", "2"):
        r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts), timeout=300)
        print(r.stdout[-3000:])
        print(r.stderr[-3000:])
        assert r.returncode == 0 and " 0 failures" in r.stdout, f"parts={parts}: status {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
