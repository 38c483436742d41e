"""Reductions of expressions with inlined sparse products and user functions, in one generated kernel per slot.

Every check compares Reductor(expr) on its bits (uint views, so -0.0 and +0.0 differ) with the explicit temporary
path, tmp.assign(expr); Reductor(tmp), which is what the front ends did before: the generated kernel rounds element i
to the expression's type as the temporary stores it, converts it as the pre-compiled reduction reads it, and folds it
with the same skeleton, grid and fold code (fold.cuh).  Each fused call must be one launch per slot.

Covered: f - A*x, (f - A*x)^2, fabs(f - A*x), make_inline(A*x) * z and A*x + B*z on CSR and on hybrid ELL with 32-bit
columns, 16-bit columns, slot masks, row classes and a CSR tail, over Poisson 2-D / 3-D, random, tridiagonal and band
matrices; float64 and float32; SUM, SUM_KAHAN, MAX, MIN, MINMAX and [SUM, SUM_KAHAN, MAX, MIN, SUM] combined; lengths
around the sweep's vector width E, the interpreter's 1024 and three turns of a capped grid; reduce.blocks_per_sm 1, 8
and 16; the interpreter skeleton through eval.force_interp; a float expression reduced in double; the reference's
counting sums and integer results of user functions; two and three slots on one device with block-diagonal matrices;
a peer group when two GPUs are present."""
import contextlib
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle
import vexcl_b200 as vx
from test_gpu_ell_edges import ENCODINGS, band, spmat, with_long_rows
from vexcl_b200 import _lib as L
from vexcl_b200.api import DeviceScalar, UserFunction

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
DEFAULTS = {"reduce.blocks_per_sm": 8, "eval.force_interp": 0}
SINGLE = [L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.MINMAX]
FIVE = [L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.SUM]


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
    return a.view({8: np.uint64, 4: np.uint32}[a.itemsize])


def mixed(seed, n, dtype):
    """sign * U[1, 2) * 2^k, k uniform in [-20, 20]: sums of these depend on the order of additions."""
    rng = np.random.default_rng(seed)
    v = rng.uniform(1, 2, n) * np.exp2(rng.integers(-20, 21, n)) * rng.choice([-1.0, 1.0], n)
    return v.astype(dtype)


def check(ctx, kind, dtype, mk, n, vdtype, what):
    """Reductor(mk()) against tmp.assign(mk()); Reductor(tmp): same bits, one launch per slot."""
    red = vx.Reductor(ctx, dtype, kind)
    n0 = vx.launch_count()
    got = red(mk())
    launches = vx.launch_count() - n0
    tmp = vx.vector(ctx, n, vdtype)
    tmp.assign(mk())
    want = red(tmp)
    assert np.array_equal(bits(got, dtype), bits(want, dtype)), f"{what}: got {got!r}, want {want!r}"
    assert launches == len(ctx.local), f"{what}: {launches} launches"
    return got


def run_kinds(ctx, kinds, dtype, mk, n, vdtype, what):
    for kind in kinds:
        check(ctx, kind, dtype, mk, n, vdtype, f"{what} kind={kind}")


# ------------------------------------------------------------------------------------------------ sparse terms

def block_diagonal(row, col, val, part):
    """The entries of (row, col, val) whose column lies in the slot of their row: strips without a halo."""
    n = row.size - 1
    rows = np.repeat(np.arange(n), np.diff(row))
    owner = np.searchsorted(part, np.arange(n), side="right") - 1
    keep = (col >= part[owner[rows]]) & (col < part[owner[rows] + 1])
    r = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(rows[keep], minlength=n), out=r[1:])
    return r, col[keep], val[keep]


MATRICES = {                          # name: builder of (row, col, val)
    "poisson2d": lambda: oracle.poisson(2, 71),
    "poisson3d": lambda: oracle.poisson(3, 17),
    "random": lambda: oracle.random_matrix(5003, 5003, 9, 7),
    "tridiagonal": lambda: oracle.tridiagonal(4099),
    "band5": lambda: band(6007, 6007, (-300, -1, 0, 1, 300), np.array([-0.5, -1.0, 4.25, -1.5, -0.75])),
    "tail": lambda: with_long_rows(*band(3001, 3001, (-70, -1, 0, 1, 70), np.array([-0.5, -1.0, 4.25, -1.5, -0.75])),
                                   long_rows={5, 600, 2999 - 60}),
}

FORMATS = {                           # name: (matrix, construction)
    "csr": ("tridiagonal", "csr"),
    "col32": ("random", "col32"),
    "col16": ("poisson3d", "col16"),
    "masks": ("band5", "masks"),
    "classes": ("poisson2d", "classes"),
    "tail": ("tail", "col32"),
}


def make_matrix(ctx, name, enc, dtype, part=None):
    row, col, val = MATRICES[name]()
    row, col, val = np.asarray(row, np.int64), np.asarray(col, np.int64), np.asarray(val, np.float64)
    if part is not None:
        row, col, val = block_diagonal(row, col, val, part)
    n = row.size - 1
    val = val.astype(dtype)
    if enc == "csr":
        A = vx.SpMat(ctx, n, n, row, col, val, vx.FMT_CSR)
    else:
        A = spmat(ctx, n, n, row, col, val, enc)
    return A, n


EXPRS = {                             # name: expression of (A, B, x, z, f)
    "residual": lambda A, B, x, z, f: f - vx.make_inline(A * x),
    "square": lambda A, B, x, z, f: (f - vx.make_inline(A * x)) * (f - vx.make_inline(A * x)),
    "fabs": lambda A, B, x, z, f: vx.fabs(f - vx.make_inline(A * x)),
    "times_z": lambda A, B, x, z, f: vx.make_inline(A * x) * z,
    "two_products": lambda A, B, x, z, f: vx.make_inline(A * x) + vx.make_inline(B * z),
}


def sparse_operands(ctx, n, dtype, seed):
    return [vx.vector(ctx, mixed(seed + k, n, dtype)) for k in range(3)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_sparse_expressions(ctx1, fmt, dtype):
    name, enc = FORMATS[fmt]
    A, n = make_matrix(ctx1, name, enc, dtype)
    B = A                             # A*x + B*z: two row loops over one strip, with different vectors
    info = A.info().loc
    if enc == "csr":
        assert info.fmt == vx.FMT_CSR
    else:
        assert info.fmt == vx.FMT_HELL
        if fmt == "tail":
            assert info.csr_tail_nnz > 0
        if enc == "classes":
            assert info.ell_classes > 0
    x, z, f = sparse_operands(ctx1, n, dtype, 10)
    for ename, mk in EXPRS.items():
        kinds = SINGLE + [FIVE] if ename == "residual" else [L.SUM]
        run_kinds(ctx1, kinds, dtype, lambda: mk(A, B, x, z, f), n, dtype, f"{fmt} {ename}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_two_different_products(ctx1, dtype):
    """A*x + B*z with strips of two formats in one kernel."""
    A, n = make_matrix(ctx1, "poisson2d", "classes", dtype)
    B, m = make_matrix(ctx1, "poisson2d", "csr", dtype)
    x, z, f = sparse_operands(ctx1, n, dtype, 20)
    run_kinds(ctx1, [L.SUM, L.SUM_KAHAN, FIVE], dtype, lambda: EXPRS["two_products"](A, B, x, z, f), n, dtype, "A*x + B*z")


def lengths(dtype, bps):
    E = 4 if dtype == np.float64 else 8
    turn = sms() * bps * 512 * E                       # elements one turn of the capped sweep grid covers
    return [1, E - 1, E, E + 1, 1023, 1024, 1025, 2 * turn + turn // 2 + E + 1]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bps", [1, 8, 16])
def test_sparse_lengths(ctx1, dtype, bps):
    """f - A*x on slot masks at the vector, block and grid boundaries; the three-turn length at one block per SM."""
    with param("reduce.blocks_per_sm", bps):
        for n in lengths(dtype, bps)[:-1] + ([lengths(dtype, 1)[-1]] if bps == 1 else []):
            row, col, val = band(n, n, (-3, -1, 0, 1, 3), np.array([-0.5, -1.0, 4.25, -1.5, -0.75], dtype))
            A = spmat(ctx1, n, n, row, col, val, "masks" if n > 64 else "col32")
            x, z, f = sparse_operands(ctx1, n, dtype, 30)
            run_kinds(ctx1, [L.SUM, L.SUM_KAHAN, FIVE], dtype, lambda: f - vx.make_inline(A * x), n, dtype, f"n={n} bps={bps}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_interpreter_skeleton(ctx1, dtype):
    """eval.force_interp = 1: the temporary is folded by reduce_interp_kernel, and so is the fused request."""
    A, n = make_matrix(ctx1, "poisson3d", "col16", dtype)
    x, z, f = sparse_operands(ctx1, n, dtype, 40)
    times2 = UserFunction(dtype, "times2", [(dtype, "v")], "return v * 2;")
    with param("eval.force_interp", 1):
        for bps in (1, 16):
            with param("reduce.blocks_per_sm", bps):
                run_kinds(ctx1, [L.SUM, L.SUM_KAHAN, L.MINMAX], dtype, lambda: f - vx.make_inline(A * x), n, dtype, "interp sparse")
                run_kinds(ctx1, [L.SUM, L.SUM_KAHAN], dtype, lambda: times2(x) - z, n, dtype, "interp call")


def test_float_expression_reduced_in_double(ctx1):
    A, n = make_matrix(ctx1, "poisson2d", "classes", np.float32)
    x, z, f = sparse_operands(ctx1, n, np.float32, 50)
    run_kinds(ctx1, [L.SUM, L.SUM_KAHAN, L.MAX, FIVE], np.float64, lambda: f - vx.make_inline(A * x), n, np.float32, "float in double")
    half = UserFunction(np.float32, "half", [(np.float32, "v")], "return v * 0.5f;")
    run_kinds(ctx1, [L.SUM, L.SUM_KAHAN], np.float64, lambda: half(x) + z, n, np.float32, "float call in double")
    # and a double expression in float: rounded to double, then to float
    xd = vx.vector(ctx1, mixed(51, n, np.float64))
    twice = UserFunction(np.float64, "twice", [(np.float64, "v")], "return v + v;")
    run_kinds(ctx1, [L.SUM, FIVE], np.float32, lambda: twice(xd), n, np.float64, "double call in float")


# ------------------------------------------------------------------------------------------------ user functions

def test_reference_counting_sums(ctx):
    """vector_arithmetics.cpp:113-145: count(greater(x, y)) in uint64, sum(times2(x))."""
    N = 1 << 20
    X, Y = mixed(1, N, np.float64), mixed(2, N, np.float64)
    x, y = vx.vector(ctx, X), vx.vector(ctx, Y)
    greater = UserFunction(np.uint64, "greater", [(np.float64, "x"), (np.float64, "y")], "return x > y;")
    times2 = UserFunction(np.float64, "times2", [(np.float64, "x")], "return x * 2;")
    c = check(ctx, L.SUM, np.uint64, lambda: greater(x, y), N, np.uint64, "count greater")
    assert c == np.count_nonzero(X > Y)
    check(ctx, L.SUM, np.float64, lambda: times2(x), N, np.float64, "sum times2")
    run_kinds(ctx, [L.SUM_KAHAN, L.MAX, L.MIN, L.MINMAX, FIVE], np.float64, lambda: times2(x) - y, N, np.float64, "times2 - y")
    x.assign(1)
    y.assign(2)
    assert vx.Reductor(ctx, np.uint64, L.SUM)(greater(x, y)) == 0
    assert vx.Reductor(ctx, np.uint64, L.SUM)(greater(y, x)) == N
    assert vx.Reductor(ctx, np.float64, L.SUM)(times2(x)) == 2 * N


def test_integer_results(ctx1):
    N = 300007
    X, Y = mixed(3, N, np.float64), mixed(4, N, np.float64)
    x, y = vx.vector(ctx1, X), vx.vector(ctx1, Y)
    k = vx.vector(ctx1, (np.arange(N) % 1009 - 500).astype(np.int32))
    sgn = UserFunction(np.int32, "sgn", [(np.float64, "v")], "return (v > 0) - (v < 0);")
    scaled = UserFunction(np.int64, "scaled", [(np.float64, "v"), (np.int32, "j")], "return (long long)(v * 1e6) * j;")
    s = check(ctx1, L.SUM, np.int32, lambda: sgn(x), N, np.int32, "int32 sum")
    assert s == np.sign(X).astype(np.int64).sum()
    run_kinds(ctx1, [L.SUM_KAHAN, L.MAX, L.MIN, L.MINMAX, FIVE], np.int32, lambda: sgn(x) * k, N, np.int32, "int32")
    run_kinds(ctx1, [L.SUM, L.MAX, L.MIN, FIVE], np.int64, lambda: scaled(x, k), N, np.int64, "int64")
    run_kinds(ctx1, [L.SUM, L.MAX], np.float64, lambda: scaled(y, k), N, np.int64, "int64 in double")
    run_kinds(ctx1, [L.SUM, L.MIN], np.int32, lambda: scaled(y, k), N, np.int64, "int64 in int32")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bps", [1, 8, 16])
def test_user_function_lengths(ctx1, dtype, bps):
    plus = UserFunction(dtype, "plus", [(dtype, "a"), (dtype, "b")], "return a + b;")
    with param("reduce.blocks_per_sm", bps):
        for n in [0] + lengths(dtype, bps):
            x, y = vx.vector(ctx1, mixed(5, n, dtype)), vx.vector(ctx1, mixed(6, n, dtype))
            kinds = [L.SUM, L.SUM_KAHAN, L.MINMAX, FIVE] if n else [L.SUM, L.MAX, L.MINMAX]
            for kind in kinds:
                red = vx.Reductor(ctx1, dtype, kind)
                got = red(plus(x, y))
                tmp = vx.vector(ctx1, n, dtype)
                if n:
                    tmp.assign(plus(x, y))
                want = red(tmp)
                assert np.array_equal(bits(got, dtype), bits(want, dtype)), f"n={n} kind={kind}: {got!r} vs {want!r}"


def test_call_with_a_sparse_term(ctx1):
    A, n = make_matrix(ctx1, "poisson2d", "classes", np.float64)
    x, z, f = sparse_operands(ctx1, n, np.float64, 60)
    damp = UserFunction(np.float64, "damp", [(np.float64, "r"), (np.float64, "w")], "return r * w / (1.0 + fabs(r));")
    run_kinds(ctx1, SINGLE + [FIVE], np.float64, lambda: damp(f - vx.make_inline(A * x), z), n, np.float64, "call(sparse)")


def test_device_result(ctx1):
    """Reductor.device leaves the same bits in device memory."""
    A, n = make_matrix(ctx1, "band5", "masks", np.float64)
    x, z, f = sparse_operands(ctx1, n, np.float64, 70)
    red = vx.Reductor(ctx1, np.float64, L.SUM)
    out = DeviceScalar(ctx1, np.float64)
    n0 = vx.launch_count()
    red.device(f - vx.make_inline(A * x), out)
    assert vx.launch_count() - n0 == 1
    tmp = vx.vector(ctx1, n)
    tmp.assign(f - vx.make_inline(A * x))
    assert np.array_equal(bits(out.get(), np.float64), bits(red(tmp), np.float64))


# ------------------------------------------------------------------------------------------------ several slots

@pytest.mark.parametrize("nparts", [2, 3])
@pytest.mark.parametrize("dtype", DTYPES)
def test_slots(ctx2, ctx3, nparts, dtype):
    """Each slot folds its slice in one launch; the host adds the slots in order, as for the temporary."""
    ctx = ctx2 if nparts == 2 else ctx3
    for name, enc in (("poisson2d", "classes"), ("random", "csr"), ("band5", "col16")):
        n = MATRICES[name]()[0].size - 1
        A, n = make_matrix(ctx, name, enc, dtype, part=ctx.partition(n))
        x, z, f = sparse_operands(ctx, n, dtype, 80)
        run_kinds(ctx, [L.SUM, L.SUM_KAHAN, L.MINMAX, FIVE], dtype, lambda: f - vx.make_inline(A * x), n, dtype, f"{nparts} slots {name}")
    N = 200003
    x, y = vx.vector(ctx, mixed(7, N, dtype)), vx.vector(ctx, mixed(8, N, dtype))
    greater = UserFunction(np.uint64, "greater", [(dtype, "x"), (dtype, "y")], "return x > y;")
    check(ctx, L.SUM, np.uint64, lambda: greater(x, y), N, np.uint64, "count on slots")


def test_products_with_a_halo_keep_the_temporary(ctx2):
    """A strip that cannot be inlined (its rows reach into the other slot) is evaluated through the temporary, as before."""
    row, col, val = oracle.poisson(2, 40)
    n = row.size - 1
    A = vx.SpMat(ctx2, n, n, row, col, val, vx.FMT_HELL)
    x, z, f = sparse_operands(ctx2, n, np.float64, 90)
    red = vx.Reductor(ctx2, np.float64, L.SUM)
    tmp = vx.vector(ctx2, n)
    tmp.assign(f - vx.make_inline(A * x))
    assert np.array_equal(bits(red(f - vx.make_inline(A * x)), np.float64), bits(red(tmp), np.float64))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="a peer group needs two GPUs")
def test_peer_group():
    ctx = vx.Context([0, 1])
    N = 1 << 20
    x, y = vx.vector(ctx, mixed(9, N, np.float64)), vx.vector(ctx, mixed(10, N, np.float64))
    times2 = UserFunction(np.float64, "times2", [(np.float64, "x")], "return x * 2;")
    run_kinds(ctx, [L.SUM, L.SUM_KAHAN, L.MINMAX, FIVE], np.float64, lambda: times2(x) - y, N, np.float64, "peer group")


# ------------------------------------------------------------------------------------------------ C++ front end

@pytest.mark.parametrize("parts", ["1", "2"])
def test_cpp_fused_reductions(built, parts):
    """tests/cpp/test_fused_reductions.cpp: sum(f - A*x) through vex::sparse::matrix and make_inline(SpMat), the counting
    sums and a CombineReductors residual, each with the bits of the temporary and one launch per slice."""
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = Path(__file__).resolve().parent / "cpp" / "bin" / "test_fused_reductions"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts),
                       timeout=300)
    print(r.stdout[-3000:]); print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"status {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
