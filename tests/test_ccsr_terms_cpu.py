"""vex::SpMatCCSR products as expression terminals (VEXB_TERM_CCSR), checked without a GPU: the assignment and reduction
kernels generated for them compile for sm_90a from a request whose matrix handle is NULL (source generation never reads
it: the kernel depends on the value type and the idx width only), malformed requests are refused before any device is
touched, and the C++ front end accepts the terminal spellings beside the additive ones."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def L(built):
    from vexcl_b200 import _lib
    return _lib


def ccsr_expr(L, dt, width, code, x_dtype=None, x_kind=None):
    """Terminals: 0 = vector x, 1 = CCSR product of x (handle NULL, idx width `width`); `code` is a list of
    (op, type, arg) with "T" for the product and "X" for x."""
    e = L.Expr()
    e.n_terms = 2
    e.term[0].kind, e.term[0].dtype = (L.TERM_VEC if x_kind is None else x_kind), (dt if x_dtype is None else x_dtype)
    e.term[0].v.ptr = 0x1000
    e.term[1].kind, e.term[1].dtype = L.TERM_CCSR, dt
    e.term[1].pad[0], e.term[1].pad[1] = 0, width
    for k, (op, typ, arg) in enumerate(code):
        if op in ("T", "X"):
            op, arg = "TERM", (1 if op == "T" else 0)
        e.code[k].op, e.code[k].type, e.code[k].arg = L.OP[op], typ, arg
    e.n_code = len(code)
    return e


def x_times_sin(dt):
    return [("X", dt, 0), ("T", dt, 0), ("SIN", dt, 0), ("MUL", dt, 0)]


def x_times_t(dt):
    return [("X", dt, 0), ("T", dt, 0), ("MUL", dt, 0)]


def source(fn, *args, compile=True):
    n = C.c_size_t(0)
    st = fn(*args, None, C.byref(n), 0)
    if st:
        return st, None
    buf = C.create_string_buffer(n.value + 8192)
    cap = C.c_size_t(len(buf))
    st = fn(*args, buf, C.byref(cap), int(compile))
    return st, buf.value.decode()


IDX_TYPES = {1: "unsigned char", 2: "unsigned short", 4: "int"}


@pytest.mark.parametrize("width", [1, 2, 4])
@pytest.mark.parametrize("dt_name", ["F64", "F32"])
def test_assignment_source_compiles(L, width, dt_name):
    dt = getattr(L, dt_name)
    T = "double" if dt == L.F64 else "float"
    for aop in (L.SET, L.ADD, L.MUL):
        st, src = source(L.lib().vexb_jit_source, dt, aop, C.byref(ccsr_expr(L, dt, width, x_times_sin(dt))))
        assert st == L.OK, L.lib().vexb_last_error()
        assert "NVRTC: ok" in src
        assert f"__device__ __forceinline__ {T} ccsr_1(const ccsr_desc_j *__restrict__ m" in src
        assert f"__ldg((const {IDX_TYPES[width]} *)m->idx + i)" in src
        assert f"ccsr_1((const ccsr_desc_j *)tt.t[1].v.ptr, (const {T} *)tt.t[0].v.ptr, i)" in src
        # one element per thread per turn of the grid-stride loop, 256 threads per block
        assert "i += stride) lhs[i] = vexb_elem(tt, lhs, i, off);" in src


@pytest.mark.parametrize("width", [1, 2, 4])
@pytest.mark.parametrize("dt_name", ["F64", "F32"])
def test_reduction_sources_compile(L, width, dt_name):
    dt = getattr(L, dt_name)
    e = ccsr_expr(L, dt, width, x_times_t(dt))
    for ops in ([L.SUM], [L.SUM_KAHAN], [L.MIN], [L.MAX], [L.MINMAX], [L.SUM, L.MIN, L.MAX]):
        o = (C.c_int * len(ops))(*ops)
        st, src = source(L.lib().vexb_jit_source_reduce, dt, len(ops), o, C.byref(e))
        assert st == L.OK, L.lib().vexb_last_error()
        assert "NVRTC: ok" in src and "ccsr_1(" in src and "vexb_reduce_kernel" in src


def test_two_terminals_and_one_shared_x(L):
    """The same product twice is one terminal; two products of one x keep one vector terminal for x."""
    dt = L.F64
    e = ccsr_expr(L, dt, 1, [("T", dt, 0), ("T", dt, 0), ("MUL", dt, 0), ("X", dt, 0), ("ADD", dt, 0)])
    st, src = source(L.lib().vexb_jit_source, dt, L.SET, C.byref(e), compile=False)
    assert st == L.OK
    assert src.count("__device__ __forceinline__ double ccsr_") == 1
    e.n_terms = 3                                   # a second matrix (another idx width) on the same x
    e.term[2].kind, e.term[2].dtype, e.term[2].pad[0], e.term[2].pad[1] = L.TERM_CCSR, dt, 0, 2
    e.code[1].arg = 2
    st, src = source(L.lib().vexb_jit_source, dt, L.SET, C.byref(e))
    assert st == L.OK, L.lib().vexb_last_error()
    assert src.count("__device__ __forceinline__ double ccsr_") == 2 and "(const unsigned short *)m->idx" in src
    assert "NVRTC: ok" in src


def test_refusals_without_a_device(L):
    lib, dt = L.lib(), L.F64
    bad = {
        "idx width 3": ccsr_expr(L, dt, 3, x_times_t(dt)),
        "idx width 0": ccsr_expr(L, dt, 0, x_times_t(dt)),
        "integer values": ccsr_expr(L, L.I32, 1, x_times_t(L.I32)),
        "x of another type": ccsr_expr(L, dt, 1, [("T", dt, 0)], x_dtype=L.F32),
        "x not a vector": ccsr_expr(L, dt, 1, [("T", dt, 0)], x_kind=L.TERM_SCALAR),
    }
    for why, e in bad.items():
        n = C.c_size_t(0)
        assert lib.vexb_jit_source(dt, L.SET, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID, why
        one = (C.c_int * 1)(L.SUM)
        assert lib.vexb_jit_source_reduce(dt, 1, one, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID, why
    e = ccsr_expr(L, dt, 1, x_times_t(dt))
    e.term[1].pad[0] = 5                            # x slot out of range
    n = C.c_size_t(0)
    assert lib.vexb_jit_source(dt, L.SET, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID
    # a launch with a NULL handle is refused before any device is selected
    e = ccsr_expr(L, dt, 1, x_times_t(dt))
    assert lib.vexb_eval(0, None, C.c_void_p(0x2000), dt, L.SET, C.byref(e), 16, 0) == L.ERR_INVALID
    assert lib.vexb_reduce_all(0, None, C.byref(e), dt, 16, 0, L.SUM, C.c_void_p(0x3000), C.c_void_p(0x4000), None) == L.ERR_INVALID
    # not fused into multi-expression kernels
    es = (C.POINTER(L.Expr) * 2)(C.pointer(e), C.pointer(e))
    assert lib.vexb_jit_source_multi(dt, L.SET, 2, es, None, C.byref(n), 0) == L.ERR_INVALID


def test_eval_path_names_the_generated_kernel(L):
    e = ccsr_expr(L, L.F32, 2, x_times_sin(L.F32))
    buf = C.create_string_buffer(64)
    assert L.lib().vexb_eval_path(L.F32, L.SET, C.byref(e), buf, 64) == L.OK
    assert buf.value == b"jit"


# ---- C++ front end ------------------------------------------------------------------------------------------------
PRELUDE = """
#include <vexcl/vexcl.hpp>
#include <vexcl/spmat/ccsr.hpp>
VEX_FUNCTION(double, sq, (double, a), return a * a;);
int main() {
    vex::Context ctx(vex::Filter::Count(1));
    std::vector<size_t> idx(8, 0), row = {0, 1}; std::vector<ptrdiff_t> col = {0}; std::vector<double> val = {2};
    vex::SpMatCCSR<double> A(ctx.queue(0), 8, 1, idx.data(), row.data(), col.data(), val.data());
    vex::vector<double> X(ctx, 8), Y(ctx, 8);
    vex::multivector<double, 2> MX(ctx, 8), MY(ctx, 8);
    vex::Reductor<double, vex::SUM> sum(ctx);
    vex::Reductor<double, vex::MIN_MAX> minmax(ctx);
    vex::Reductor<double, vex::CombineReductors<vex::SUM, vex::MAX>> summax(ctx);
"""

SPELLINGS = {
    "sin": "Y = sin(A * X);",
    "x_times_product": "Y = X * (A * X);",
    "product_times_x": "Y = (A * X) * X;",
    "energy_norm": "double e = sum(X * (A * X)); (void)e;",
    "make_inline": "Y = vex::make_inline(A * X) * X;",
    "compound": "Y *= A * X; Y /= A * X;",
    "user_function": "Y = sq(A * X);",
    "if_else": "Y = vex::if_else(A * X > 0, X, A * X);",
    "scaled_operand": "Y = X * (2 * (A * X));",
    "reductions": "double s = sum(A * X); auto m = minmax(A * X); auto c = summax(vex::make_inline(A * X)); (void)s; (void)m; (void)c;",
    "additive": "Y = A * X; Y += A * X; Y -= A * X; Y = X + A * X; Y -= 0.5 * (A * X); Y = A * X - X; Y = 2 * (A * X) + A * X; Y = -(A * X);",
    "additive_multivector": "MY = A * MX; MY += A * MX;",
}

# The additive spellings keep their types, so they keep the hand-written CCSR kernels.
TYPES = """
    typedef vex::additive_operator<vex::SpMatCCSR<double>, vex::vector<double>> add_t;
    static_assert(std::is_same<decltype(A * X), add_t>::value, "A * X is the additive operator");
    static_assert(std::is_same<decltype(2 * (A * X)), add_t>::value, "a scaled product stays additive");
    static_assert(std::is_same<decltype(-(A * X)), add_t>::value, "a negated product stays additive");
    static_assert(std::is_same<decltype(X + A * X), vex::mixed_expression<const vex::vector<double>&, double>>::value, "x + A*x stays mixed");
    static_assert(std::is_same<decltype(A * X + A * X), vex::detail::additive_terms<double>>::value, "sums stay additive");
    static_assert(std::is_same<decltype(vex::make_inline(A * X)), const vex::ccsr_product<double, ptrdiff_t, size_t>>::value, "make_inline");
"""


def _syntax(body: str):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    src = PRELUDE + body + "\n}\n"
    return subprocess.run([gxx, "-std=c++17", "-fsyntax-only", "-Wall", "-I", str(ROOT / "include"), "-x", "c++", "-"],
                          input=src, capture_output=True, text=True)


@pytest.mark.parametrize("name", sorted(SPELLINGS))
def test_cpp_spelling_compiles(name):
    r = _syntax(SPELLINGS[name])
    assert r.returncode == 0, r.stderr[-3000:]


def test_cpp_additive_spellings_keep_their_types():
    r = _syntax(TYPES)
    assert r.returncode == 0, r.stderr[-3000:]
