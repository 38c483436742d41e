"""vex::raw_pointer without a GPU: malformed pointer programs are refused before anything runs, a `double` and a `double*`
parameter make two functions, the generated assignment, multi-expression and reduction sources of loads and of a user
function with a pointer parameter compile for sm_90a, the Python front end folds pointer arithmetic into one load, and
the C++ spellings compile while every misuse stops at its static_assert.  The numerical checks are in
tests/test_gpu_pointers.py and tests/cpp/test_vector_pointer.cpp."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def env(built):
    import vexcl_b200 as vx
    from vexcl_b200 import api, _lib as L

    class FakeCtx:
        nparts, local, devs, streams, weights = 1, [0], {0: 0}, {0: None}, None
        def partition(self, n): return vx.partition(n, 1)

    def fake_vec(n, dt, addr, nparts=1):
        v = api.vector.__new__(api.vector)
        ctx = FakeCtx()
        ctx.nparts = nparts
        v.ctx, v.n, v.np_dtype, v.dtype, v.part, v.bufs = ctx, n, np.dtype(dt), api._vdt(dt), vx.partition(n, 1), {0: C.c_void_p(addr)}
        return v
    return vx, api, L, fake_vec


def lowered(api, expr, n=1024):
    low = api._Lowering(0, 0)
    low.size = n
    low.lower(api.wrap(expr))
    return low


def _two_calls(fn, *args, compile=True):
    n = C.c_size_t(0)
    L_st = fn(*args, None, C.byref(n), 0)
    assert L_st == 0
    buf = C.create_string_buffer(n.value + 8192)
    cap = C.c_size_t(len(buf))
    return fn(*args, buf, C.byref(cap), int(compile)), buf.value.decode()


def source(L, lhs_dtype, op, e):
    st, src = _two_calls(L.lib().vexb_jit_source, lhs_dtype, op, C.byref(e))
    L.check(st)
    return src


def multi_source(L, lhs_dtype, op, exprs):
    es = (C.POINTER(L.Expr) * len(exprs))(*[C.pointer(e) for e in exprs])
    st, src = _two_calls(L.lib().vexb_jit_source_multi, lhs_dtype, op, len(exprs), es)
    L.check(st)
    return src


def reduce_source(L, dtype, ops, e):
    o = (C.c_int * len(ops))(*ops)
    st, src = _two_calls(L.lib().vexb_jit_source_reduce, dtype, len(ops), o, C.byref(e))
    L.check(st)
    return src


def _raw(L, code, terms):
    """A program over explicit terminals: terms = [(kind, dtype, pointer)]."""
    e = L.Expr()
    for k, (kind, dt, p) in enumerate(terms):
        e.term[k].kind, e.term[k].dtype, e.term[k].v.ptr = kind, dt, p
    e.n_terms = len(terms)
    for k, (op, typ, arg) in enumerate(code):
        e.code[k].op, e.code[k].type, e.code[k].arg = L.OP[op], typ, arg
    e.n_code = len(code)
    return e


def _register(L, name, ret, args, body):
    fid = C.c_int(-1)
    at = (C.c_int * max(len(args), 1))(*args)
    st = L.lib().vexb_function_register(name.encode(), ret, len(args), at, body.encode(), C.byref(fid))
    return st, fid.value


REFUSALS = ["load of a vector terminal", "index of type int", "index of type u64", "load of another type", "pointer plus one",
            "pointer converted", "pointer as a temporary", "pointer as a branch", "pointer as the result",
            "pointer to a value parameter", "value to a pointer parameter", "pointer of another type to a parameter"]


def _refusal(L, case):
    F, I, P, V, S = L.F64, L.I64, L.TERM_PTR, L.TERM_VEC, L.TERM_SCALAR
    ptr = [(P, F, 0x1000), (S, I, 0)]                                # slot 0: the pointer, slot 1: an I64 scalar 0
    if case == "load of a vector terminal":
        return _raw(L, [("TERM", I, 1), ("LOAD", F, 0)], [(V, F, 0x1000), (S, I, 0)])
    if case == "index of type int":
        return _raw(L, [("TERM", L.I32, 1), ("LOAD", F, 0)], [(P, F, 0x1000), (S, L.I32, 0)])
    if case == "index of type u64":
        return _raw(L, [("TERM", L.U64, 1), ("LOAD", F, 0)], [(P, F, 0x1000), (S, L.U64, 0)])
    if case == "load of another type":
        return _raw(L, [("TERM", I, 1), ("LOAD", L.F32, 0)], ptr)
    if case == "pointer plus one":
        return _raw(L, [("TERM", L.PTR(F), 0), ("TERM", I, 1), ("ADD", I, 0), ("TERM", I, 1), ("LOAD", F, 0), ("ADD", F, 0)], ptr)
    if case == "pointer converted":
        return _raw(L, [("TERM", L.PTR(F), 0), ("CVT", I, L.PTR(F))], ptr)
    if case == "pointer as a temporary":
        return _raw(L, [("TERM", L.PTR(F), 0), ("TDEF", L.PTR(F), 0), ("TERM", I, 1), ("LOAD", F, 0)], ptr)
    if case == "pointer as a branch":
        return _raw(L, [("TERM", I, 1), ("CVT", L.I32, I), ("TERM", L.PTR(F), 0), ("TERM", L.PTR(F), 0), ("SELECT", F, 0)], ptr)
    if case == "pointer as the result":
        return _raw(L, [("TERM", L.PTR(F), 0)], ptr)
    st, fval = _register(L, "ptr_refusal_value", F, [F], "return prm1;")
    L.check(st)
    st, fptr = _register(L, "ptr_refusal_ptr", F, [L.PTR(F)], "return prm1[0];")
    L.check(st)
    if case == "pointer to a value parameter":
        return _raw(L, [("TERM", L.PTR(F), 0), ("CALL", F, fval)], ptr)
    if case == "value to a pointer parameter":
        return _raw(L, [("TERM", I, 1), ("LOAD", F, 0), ("CALL", F, fptr)], ptr)
    return _raw(L, [("TERM", L.PTR(L.F32), 0), ("CALL", F, fptr)], [(P, L.F32, 0x1000)])


@pytest.mark.parametrize("case", REFUSALS)
def test_malformed_pointer_programs_are_refused_everywhere(env, case):
    vx, api, L, fake_vec = env
    lib = L.lib()
    e = _refusal(L, case)
    n = C.c_size_t(0)
    assert lib.vexb_jit_source(L.F64, L.SET, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID
    buf = C.create_string_buffer(64)
    assert lib.vexb_eval_path(L.F64, L.SET, C.byref(e), buf, 64) == L.ERR_INVALID
    good = lowered(api, fake_vec(1024, np.float64, 0x1000) * 2.0).e
    es = (C.POINTER(L.Expr) * 2)(C.pointer(good), C.pointer(e))
    assert lib.vexb_jit_source_multi(L.F64, L.SET, 2, es, None, C.byref(n), 0) == L.ERR_INVALID
    one = (C.c_int * 1)(L.SUM)
    assert lib.vexb_jit_source_reduce(L.F64, 1, one, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID
    assert lib.vexb_jit_precompile(L.F64, L.SET, C.byref(e), 0) == L.ERR_INVALID
    # the device entry points validate before they look for a device
    assert lib.vexb_eval(0, None, None, L.F64, L.SET, C.byref(e), 0, 0) == L.ERR_INVALID
    handled = C.c_int(0)
    out = (C.c_void_p * 2)(None, None)
    assert lib.vexb_eval_multi(0, None, 2, out, L.F64, L.SET, es, 0, 0, C.byref(handled)) == L.ERR_INVALID
    ws = C.c_void_p(0x3000)
    assert lib.vexb_reduce_all(0, None, C.byref(e), L.F64, 0, 0, L.SUM, ws, ws, None) == L.ERR_INVALID


def test_a_null_pointer_is_refused_except_by_the_source_printers(env):
    vx, api, L, fake_vec = env
    lib = L.lib()
    e = _raw(L, [("TERM", L.I64, 1), ("LOAD", L.F64, 0)], [(L.TERM_PTR, L.F64, 0), (L.TERM_SCALAR, L.I64, 0)])
    src = source(L, L.F64, L.SET, e)
    assert "NVRTC: ok" in src
    assert lib.vexb_eval(0, None, C.c_void_p(0x2000), L.F64, L.SET, C.byref(e), 16, 0) == L.ERR_INVALID
    assert "NULL" in lib.vexb_last_error().decode()


def test_registration_tells_a_value_from_a_pointer_parameter(env):
    vx, api, L, fake_vec = env
    st, a = _register(L, "same_name", L.F64, [L.F64], "return 1.0;")
    st2, b = _register(L, "same_name", L.F64, [L.PTR(L.F64)], "return 1.0;")
    st3, c = _register(L, "same_name", L.F64, [L.PTR(L.F64)], "return 1.0;")
    assert st == st2 == st3 == L.OK and a != b and b == c
    assert _register(L, "bad_ptr", L.F64, [L.PTR(L.F64) | 0x20], "return 1.0;")[0] == L.ERR_INVALID
    assert _register(L, "bad_ret", L.PTR(L.F64), [L.F64], "return prm1;")[0] == L.ERR_INVALID


@pytest.mark.parametrize("dt", [np.float64, np.float32, np.int32, np.uint32, np.int64, np.uint64], ids=lambda d: np.dtype(d).name)
def test_load_programs_compile_for_sm90a_in_all_three_kernel_kinds(env, dt):
    vx, api, L, fake_vec = env
    x, y = fake_vec(1024, dt, 0x1000), fake_vec(1024, dt, 0x2000)
    idx = fake_vec(1024, np.int32, 0x3000)
    p = vx.raw_pointer(x)
    i = vx.ElementIndex()
    stencil = 2 * p[i] - p[vx.if_else(i > 0, i - 1, i)] - p[vx.if_else(i + 1 < 1024, i + 1, i)]
    T = {np.float64: "double", np.float32: "float", np.int32: "int", np.uint32: "unsigned int", np.int64: "long long",
         np.uint64: "unsigned long long"}[dt]
    e = lowered(api, stencil).e
    src = source(L, y.dtype, L.SET, e)
    slots = re.findall(r"__ldg\(\(const " + re.escape(T) + r" \*\)tt\.t\[(\d+)\]", src)
    assert len(slots) == 3 and len(set(slots)) == 1 and "NVRTC: ok" in src         # one terminal serves the three loads
    assert src.count(f"< vexb_count(tt.t[{slots[0]}]) ? __ldg(") == 3                 # 0 outside the array
    src = multi_source(L, y.dtype, L.ADD, [lowered(api, stencil).e, lowered(api, p[idx] + y).e])
    assert src.count("__ldg(") == 4 and "NVRTC: ok" in src
    ops = [L.SUM, L.MAX] if dt in (np.float64, np.float32) else [L.MIN]
    rdt = y.dtype
    f = vx.UserFunction(dt, "twice_" + np.dtype(dt).name, [(dt, "a")], "return a + a;")
    src = reduce_source(L, rdt, ops, lowered(api, f(x * p[idx])).e)
    assert "__ldg(" in src and "NVRTC: ok" in src
    src = reduce_source(L, rdt, ops[:1], lowered(api, f(vx.deref(p + idx))).e)
    assert "NVRTC: ok" in src


def test_a_user_function_with_a_pointer_parameter_compiles_and_loads_plainly(env):
    vx, api, L, fake_vec = env
    x, y = fake_vec(1024, np.float64, 0x1000), fake_vec(1024, np.float64, 0x2000)
    nbody = vx.UserFunction(np.float64, "nbody_cpu", [(np.uint64, "n"), (np.uint64, "j"), (vx.ptr(np.float64), "x")],
                            "double sum = 0; for (size_t i = 0; i < n; ++i) if (i != j) sum += x[i]; return sum;")
    p = vx.raw_pointer(x)
    e = lowered(api, nbody(np.uint64(4096), vx.ElementIndex(), p) + p[vx.ElementIndex()]).e
    src = source(L, L.F64, L.SET, e)
    assert "double * prm3" in src and "double *x = prm3;" in src and "(double *)tt.t[" in src and "NVRTC: ok" in src
    assert "__ldg(" not in src.split("vexb_elem")[1] and "*((const double *)tt.t[" in src   # the body may write through x
    assert "NVRTC: ok" in multi_source(L, L.F64, L.SET, [e, lowered(api, y * 2.0).e])
    src = reduce_source(L, L.F64, [L.SUM, L.MIN], e)
    assert "NVRTC: ok" in src
    src = reduce_source(L, L.F64, [L.SUM_KAHAN], e)
    assert "NVRTC: ok" in src


def test_pointer_arithmetic_folds_into_one_load(env):
    vx, api, L, fake_vec = env
    x = fake_vec(1024, np.float64, 0x1000)
    a, b = fake_vec(1024, np.uint32, 0x2000), fake_vec(1024, np.int32, 0x3000)
    p = vx.raw_pointer(x)
    ops = lambda e: [(L._OPS[e.code[k].op], e.code[k].type, e.code[k].arg) for k in range(e.n_code)]
    # each offset widened on its own (u32 zero-extended, i32 sign-extended), then added in I64
    e = lowered(api, (p + a)[b]).e
    assert [o[0] for o in ops(e)] == ["TERM", "CVT", "TERM", "CVT", "ADD", "LOAD"]
    t = e.term[e.code[5].arg]                                   # the pointer carries x's element count in pad[0..5]
    assert t.kind == L.TERM_PTR and t.v.ptr == 0x1000 and sum(t.pad[k] << (8 * k) for k in range(6)) == 1024
    assert ops(e)[1] == ("CVT", L.I64, L.U32) and ops(e)[3] == ("CVT", L.I64, L.I32) and ops(e)[4][1] == L.I64
    e = lowered(api, vx.deref(p - a)).e
    assert [o[0] for o in ops(e)] == ["TERM", "CVT", "NEG", "LOAD"]
    e = lowered(api, vx.deref(p)).e
    assert [o[0] for o in ops(e)] == ["TERM", "LOAD"] and e.term[0].kind == L.TERM_SCALAR and e.term[0].dtype == L.I64
    assert [o[0] for o in ops(lowered(api, (b + p)[3]).e)] == ["TERM", "CVT", "TERM", "CVT", "ADD", "LOAD"]
    # a program with a load never takes a hand-written sweep
    buf = C.create_string_buffer(64)
    L.check(L.lib().vexb_eval_path(L.F64, L.SET, C.byref(lowered(api, p[vx.ElementIndex()]).e), buf, 64))
    assert buf.value.decode() in ("interp", "jit")


def test_the_python_front_end_refuses_other_uses_of_a_pointer(env):
    vx, api, L, fake_vec = env
    x = fake_vec(1024, np.float64, 0x1000)
    p = vx.raw_pointer(x)
    for bad in (lambda: p * 2, lambda: p + 1.5, lambda: x + (p - x), lambda: 2 - p, lambda: -p, lambda: x * p, lambda: p + p,
                lambda: vx.sin(p), lambda: vx.deref(x)):
        with pytest.raises(TypeError):
            bad()
    f = vx.UserFunction(np.float64, "takes_ptr", [(vx.ptr(np.float64), "x")], "return x[0];")
    with pytest.raises(TypeError):
        f(p + 1)
    with pytest.raises(TypeError):
        f(x)
    with pytest.raises(TypeError):
        f(vx.raw_pointer(fake_vec(1024, np.float32, 0x2000)))
    with pytest.raises(ValueError):
        vx.raw_pointer(fake_vec(1024, np.float64, 0x3000, nparts=2))
    with pytest.raises(ValueError):                          # a vector of two parts next to a pointer
        lowered(api, p[vx.ElementIndex()] + fake_vec(1024, np.float64, 0x3000, nparts=2))


CPP_SPELLINGS = r'''
#include <vexcl/vexcl.hpp>
VEX_FUNCTION(double, nbody, (size_t, n)(size_t, j)(double*, x), double s = 0; for (size_t i = 0; i < n; ++i) if (i != j) s += x[i]; return s;);
VEX_FUNCTION(float, first, (const float *, x)(int, k), return x[k];);
VEX_FUNCTION_V1(second, long long(const long long*, unsigned long long*), "return prm1[1] + (long long)prm2[0];");
void f(vex::vector<double> &y, const vex::vector<double> &x, const vex::vector<int> &idx, const vex::vector<float> &z,
       const vex::vector<long long> &l, const vex::vector<unsigned long long> &u) {
    auto p = vex::raw_pointer(x);
    vex::vector_pointer<double> q(x);
    auto i = vex::element_index();
    y = *(p + i) + *(p - 1) + p[idx] + (p + idx)[-1] + (idx + p)[2u] + *p + q[i];
    y = nbody(x.size(), i, p) + first(vex::raw_pointer(z), 3) + second(vex::raw_pointer(l), vex::raw_pointer(u));
    y += if_else(i > 0, (p + i)[-1], 0.0);
    vex::Reductor<double, vex::SUM> sum(y.queue_list());
    (void)sum(x * p[i % 4]);
}
'''

MISUSES = {
    "p * 2": ("y = p * 2;", "a raw_pointer is only indexed"),
    "2 * p": ("y = 2 * p;", "a raw_pointer is only indexed"),
    "p + 1.5": ("y = *(p + 1.5);", "pointer arithmetic takes an integral expression or scalar"),
    "p + x": ("y = *(p + x);", "pointer arithmetic takes an integral expression or scalar"),
    "p[x]": ("y = p[x];", "a raw_pointer is indexed by an integral expression or scalar"),
    "p - p": ("y = *(p - p);", "the difference of two raw pointers"),
    "x - p": ("y = *(1 - p);", "a raw_pointer is not subtracted from a value"),
    "p + p": ("y = *(p + p);", "two raw pointers are not added"),
    "-p": ("y = *(-p);", "a raw_pointer is not negated"),
    "p < x": ("y = (p < x);", "a raw_pointer is only indexed"),
    "p + 1 to a function": ("y = takes(p + 1);", "a user function takes a raw_pointer without arithmetic"),
}


def test_cpp_spellings_compile(tmp_path):
    (tmp_path / "spellings.cpp").write_text(CPP_SPELLINGS)
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wno-unused-function", "-fsyntax-only", "-I", str(ROOT / "include"),
                        str(tmp_path / "spellings.cpp")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wno-unused-function", "-fsyntax-only", "-I", str(ROOT / "include"),
                        str(ROOT / "tests" / "cpp" / "test_vector_pointer.cpp")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]


@pytest.mark.parametrize("case", sorted(MISUSES))
def test_cpp_misuse_stops_at_its_static_assert(tmp_path, case):
    stmt, msg = MISUSES[case]
    (tmp_path / "misuse.cpp").write_text(
        "#include <vexcl/vexcl.hpp>\nVEX_FUNCTION(double, takes, (double*, x), return x[0];);\n"
        "void f(vex::vector<double> &y, const vex::vector<double> &x) { auto p = vex::raw_pointer(x); " + stmt + " }\n")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", str(ROOT / "include"), str(tmp_path / "misuse.cpp")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "static assertion failed" in r.stderr and msg in r.stderr, r.stderr[-2000:]
