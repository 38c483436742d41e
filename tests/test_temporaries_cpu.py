"""vex::make_temp without a GPU: the generated sources (a temporary is defined once and read by every use; components of a
multi-expression share a temporary defined over the same terminals), NVRTC compiles them for sm_90a, malformed programs
are refused before anything runs, programs without temporaries print what they printed before, and the C++ spellings
compile.  The numerical checks are in tests/test_gpu_temporaries.py and tests/cpp/test_temporary.cpp."""
import ctypes as C
import json
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = Path(__file__).resolve().parent / "golden" / "jit_sources_without_temporaries.json"
DTYPES = [np.float64, np.float32, np.int32, np.uint64]


@pytest.fixture(scope="module")
def env(built):
    import vexcl_b200 as vx
    from vexcl_b200 import api, _lib as L

    class FakeCtx:
        nparts, local, devs, streams, weights = 1, [0], {0: 0}, {0: None}, None
        def partition(self, n): return vx.partition(n, 1)

    def fake_vec(n, dt, addr):
        v = api.vector.__new__(api.vector)
        v.ctx, v.n, v.np_dtype, v.dtype, v.part, v.bufs = FakeCtx(), n, np.dtype(dt), api._vdt(dt), vx.partition(n, 1), {0: C.c_void_p(addr)}
        return v
    return vx, api, L, fake_vec


def lowered(api, expr, n=1024):
    low = api._Lowering(0, 0)
    low.size = n
    low.lower(api.wrap(expr))
    return low


def _two_calls(fn, *args, compile=True):
    n = C.c_size_t(0)
    fn(*args, None, C.byref(n), 0)
    buf = C.create_string_buffer(n.value + 4096)
    cap = C.c_size_t(len(buf))
    return fn(*args, buf, C.byref(cap), int(compile)), buf.value.decode()


def source(api, L, lhs_dtype, op, expr, compile=True):
    st, src = _two_calls(L.lib().vexb_jit_source, lhs_dtype, op, C.byref(expr if isinstance(expr, L.Expr) else lowered(api, expr).e), compile=compile)
    L.check(st)
    return src


def multi_source(api, L, lhs_dtype, op, exprs, compile=True):
    lows = [lowered(api, e) for e in exprs]
    es = (C.POINTER(L.Expr) * len(lows))(*[C.pointer(low.e) for low in lows])
    st, src = _two_calls(L.lib().vexb_jit_source_multi, lhs_dtype, op, len(lows), es, compile=compile)
    L.check(st)
    return src


def reduce_source(api, L, dtype, ops, expr, compile=True):
    o = (C.c_int * len(ops))(*ops)
    e = expr if isinstance(expr, L.Expr) else lowered(api, expr).e
    st, src = _two_calls(L.lib().vexb_jit_source_reduce, dtype, len(ops), o, C.byref(e), compile=compile)
    L.check(st)
    return src


@pytest.mark.parametrize("dt", DTYPES, ids=lambda d: np.dtype(d).name)
def test_a_temporary_read_three_times_is_defined_once(env, dt):
    vx, api, L, fake_vec = env
    x, y = fake_vec(1024, dt, 0x1000), fake_vec(1024, dt, 0x2000)
    floating = np.dtype(dt).kind == "f"
    t = vx.make_temp(1, vx.sin(x) if floating else x * 3 + 1)
    src = source(api, L, y.dtype, L.SET, t * t + t)
    T = {np.float64: "double", np.float32: "float", np.int32: "int", np.uint64: "unsigned long long"}[dt]
    assert src.count(f"const {T} t0 = ") == 1 and "NVRTC: ok" in src
    assert src.count(f"__ldcs((const {T} *)tt.t[0].v.ptr + i)") == 1            # x is read once, by the definition
    if floating:
        assert src.count("sin") == 1
    red = reduce_source(api, L, y.dtype, [L.SUM], t * t + t)
    assert red.count(f"const {T} t0 = ") == 1 and "NVRTC: ok" in red
    red = reduce_source(api, L, y.dtype, [L.SUM, L.MAX], t * t + t)
    assert red.count(f"const {T} t0 = ") == 1 and "NVRTC: ok" in red


def test_nested_and_explicitly_typed_temporaries(env):
    vx, api, L, fake_vec = env
    x, y = fake_vec(1024, np.float64, 0x1000), fake_vec(1024, np.float64, 0x2000)
    t1 = vx.make_temp(1, vx.log(x))
    t2 = vx.make_temp(2, t1 + vx.sin(x))
    low = lowered(api, t1 * t2)
    ops = [L._OPS[low.e.code[k].op] for k in range(low.e.n_code)]
    assert ops == ["TERM", "LOG", "TDEF", "TREF", "TERM", "SIN", "ADD", "TDEF", "TREF", "TREF", "MUL"]   # dependencies first
    src = source(api, L, y.dtype, L.SET, t1 * t2)
    assert src.count("log(") == 1 and src.count("sin(") == 1 and "NVRTC: ok" in src
    f = vx.make_temp(1, x * 3.0 + 1.0, np.float32)                # T(e) written out: (double)(float)(x * 3 + 1)
    assert f.dtype == L.F32
    src = source(api, L, y.dtype, L.SET, f * x)
    assert "const float t0 = " in src and "NVRTC: ok" in src
    # an if_else branch that never reads the temporary does not stop its definition
    s = vx.make_temp(3, vx.sqrt(x))
    src = source(api, L, y.dtype, L.SET, vx.if_else(x > 0.5, s, x))
    assert src.count("const double t0 = ") == 1 and "NVRTC: ok" in src


def test_a_sparse_row_function_read_through_a_temporary_is_called_once(env):
    vx, api, L, fake_vec = env
    for dt in (L.F64, L.F32):
        low = api._Lowering(0, 0)
        xs = low.term(L.TERM_VEC, dt, ptr=0x1000)
        k = low.term(L.TERM_CCSR, dt, pad0=xs, ptr=0)          # a source query may pass no handle: the idx width says enough
        low.e.term[k].pad[1] = 2
        low.emit("TERM", dt, k); low.emit("TDEF", dt, 0)
        low.emit("TREF", dt, 0); low.emit("TREF", dt, 0); low.emit("MUL", dt); low.emit("TREF", dt, 0); low.emit("ADD", dt)
        src = source(api, L, dt, L.SET, low.e)
        assert src.count("(const ccsr_desc_j *)tt.t[") == 1 and "NVRTC: ok" in src
        red = reduce_source(api, L, dt, [L.SUM], low.e)
        assert red.count("(const ccsr_desc_j *)tt.t[") == 1 and "NVRTC: ok" in red


def test_tie_components_share_a_temporary_over_the_same_terminals(env):
    vx, api, L, fake_vec = env
    x, y = fake_vec(1024, np.float64, 0x1000), fake_vec(1024, np.float64, 0x2000)
    t = vx.make_temp(1, vx.sin(x))
    src = multi_source(api, L, x.dtype, L.SET, [t, vx.sqrt(1.0 - t * t)])
    assert src.count("sin(") == 1 and src.count("vexb_temp_0(mt.c[0], i, off)") == 1 and "NVRTC: ok" in src
    # a multivector temporary: every component defines its own over its own vector
    x0, x1 = fake_vec(1024, np.float64, 0x3000), fake_vec(1024, np.float64, 0x4000)
    t0, t1 = vx.make_temp(1, vx.tan(x0)), vx.make_temp(1, vx.tan(x1))
    src = multi_source(api, L, x.dtype, L.SET, [t0 * t0, t1 * t1])
    assert src.count("tan(") == 2 and "vexb_temp_1(mt.c[1], i, off)" in src and "NVRTC: ok" in src
    # one component with temporaries beside one without, nested and shared, every type
    for dt in DTYPES:
        a, b = fake_vec(1024, dt, 0x5000), fake_vec(1024, dt, 0x6000)
        u = vx.make_temp(1, a + b)
        w = vx.make_temp(2, u * a)
        src = multi_source(api, L, a.dtype, L.ADD, [w + u, a - b, u * 2])
        assert src.count("vexb_temp_") == 2 + 2 and "NVRTC: ok" in src, dt


def _raw(L, code, n_terms=1, dt=None):
    e = L.Expr()
    dt = L.F64 if dt is None else dt
    for k in range(n_terms):
        e.term[k].kind, e.term[k].dtype, e.term[k].v.ptr = L.TERM_VEC, dt, 0x1000 * (k + 1)
    e.n_terms = n_terms
    for k, (op, typ, arg) in enumerate(code):
        e.code[k].op, e.code[k].type, e.code[k].arg = L.OP[op], typ, arg
    e.n_code = len(code)
    return e


def _refusals(L):
    F, G = L.F64, L.F32
    return {
        "slot out of range": [("TERM", F, 0), ("TDEF", F, 8), ("TREF", F, 8)],
        "second definition": [("TERM", F, 0), ("TDEF", F, 0), ("TERM", F, 0), ("TDEF", F, 0), ("TREF", F, 0)],
        "read before definition": [("TREF", F, 0), ("TERM", F, 0), ("TDEF", F, 0)],
        "read as another type": [("TERM", F, 0), ("TDEF", F, 0), ("TREF", G, 0)],
        "defined as another type": [("TERM", F, 0), ("TDEF", G, 0), ("TREF", G, 0)],
        "defined at depth 2": [("TERM", F, 0), ("TERM", F, 0), ("TDEF", F, 0), ("TREF", F, 0), ("ADD", F, 0)],
        "defined on an empty stack": [("TDEF", F, 0), ("TERM", F, 0)],
    }


@pytest.mark.parametrize("case", ["slot out of range", "second definition", "read before definition", "read as another type",
                                  "defined as another type", "defined at depth 2", "defined on an empty stack"])
def test_malformed_temporaries_are_refused_everywhere(env, case):
    vx, api, L, fake_vec = env
    lib = L.lib()
    e = _raw(L, _refusals(L)[case])
    n = C.c_size_t(0)
    assert lib.vexb_jit_source(L.F64, L.SET, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID
    assert "temporar" in lib.vexb_last_error().decode() or "stack" in lib.vexb_last_error().decode()
    buf = C.create_string_buffer(64)
    assert lib.vexb_eval_path(L.F64, L.SET, C.byref(e), buf, 64) == L.ERR_INVALID
    good = lowered(api, fake_vec(1024, np.float64, 0x1000) * 2.0).e
    es = (C.POINTER(L.Expr) * 2)(C.pointer(good), C.pointer(e))
    assert lib.vexb_jit_source_multi(L.F64, L.SET, 2, es, None, C.byref(n), 0) == L.ERR_INVALID
    one = (C.c_int * 1)(L.SUM)
    assert lib.vexb_jit_source_reduce(L.F64, 1, one, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID
    assert lib.vexb_jit_precompile(L.F64, L.SET, C.byref(e), 0) == L.ERR_INVALID
    # the device entry points validate before they look for a device: an empty slice is enough to see the refusal
    assert lib.vexb_eval(0, None, None, L.F64, L.SET, C.byref(e), 0, 0) == L.ERR_INVALID
    handled = C.c_int(0)
    out = (C.c_void_p * 2)(None, None)
    assert lib.vexb_eval_multi(0, None, 2, out, L.F64, L.SET, es, 0, 0, C.byref(handled)) == L.ERR_INVALID


def test_the_front_end_refuses_a_clashing_tag_and_a_ninth_temporary(env):
    vx, api, L, fake_vec = env
    x = fake_vec(1024, np.float64, 0x1000)
    with pytest.raises(ValueError, match="one tag names two different expressions"):
        lowered(api, vx.make_temp(1, vx.sin(x)) + vx.make_temp(1, vx.cos(x)))
    same = lowered(api, vx.make_temp(1, vx.sin(x)) * vx.make_temp(1, vx.sin(x)))
    assert sum(same.e.code[k].op == L.OP["TDEF"] for k in range(same.e.n_code)) == 1
    e = vx.make_temp(0, x)
    for k in range(1, 8):
        e = e + vx.make_temp(k, x)
    lowered(api, e)                                                 # eight temporaries are fine
    with pytest.raises(ValueError, match="too many temporaries"):
        lowered(api, e + vx.make_temp(8, x))


def _programs_without_temporaries(vx, api, L, fake_vec):
    """Representative requests without temporaries: (name, kind, lhs / reduce dtype, op(s), lowered expressions)."""
    x, y, z = (fake_vec(1024, np.float64, 0x1000 * (k + 1)) for k in range(3))
    f, i = fake_vec(1024, np.float32, 0x5000), fake_vec(1024, np.int32, 0x6000)
    return [
        ("muladd", "eval", L.F64, L.SET, [x + y * z]),
        ("sin_mix", "eval", L.F64, L.ADD, [vx.sin(x) * y + z / 3.0 - vx.if_else(x > y, x, 2.0)]),
        ("float_int", "eval", L.F32, L.SET, [f * i + vx.ElementIndex(3) % 7]),
        ("int_shift", "eval", L.I32, L.RSH, [(i << 2) | 5]),
        ("tie", "multi", L.F64, L.SET, [x + y, y - x]),
        ("sum", "reduce", L.F64, [L.SUM], [vx.sin(x) * y]),
        ("combined", "reduce", L.F32, [L.SUM, L.MAX, L.MIN], [f * f]),
    ]


def _print_all(vx, api, L, fake_vec):
    out = {}
    for name, kind, dt, op, exprs in _programs_without_temporaries(vx, api, L, fake_vec):
        if kind == "eval":
            out[name] = source(api, L, dt, op, exprs[0], compile=False)
        elif kind == "multi":
            out[name] = multi_source(api, L, dt, op, exprs, compile=False)
        else:
            out[name] = reduce_source(api, L, dt, op, exprs[0], compile=False)
    return out


def test_programs_without_temporaries_print_what_they_printed_before(env):
    """tests/golden/jit_sources_without_temporaries.json holds these sources as the library printed them before
    temporaries existed."""
    vx, api, L, fake_vec = env
    want = json.loads(GOLDEN.read_text())
    got = _print_all(vx, api, L, fake_vec)
    assert got == want
    x, y, z = (fake_vec(1024, np.float64, 0x1000 * (k + 1)) for k in range(3))
    assert z.eval_path(L.SET, x + y * z) == "sweep:muladd"
    assert z.eval_path(L.SET, vx.sin(x) + y) == "interp"
    t = vx.make_temp(1, x + y)
    assert z.eval_path(L.SET, t * z) == "interp"                    # never a hand-written sweep, even for a sweep shape
    assert z.eval_path(L.SET, t) == "interp"


CPP_ADDITIVE = r"""
#include <vexcl/vexcl.hpp>
int main() {
    vex::Context ctx(vex::Filter::Any);
    std::vector<size_t> row{0, 1}, col{0}; std::vector<double> val{1};
    vex::SpMat<double> A(ctx, 1, 1, row.data(), col.data(), val.data());
    vex::vector<double> x(ctx, 1), y(ctx, 1);
    y = vex::make_temp<1>(A * x);
}
"""


def test_cpp_spellings_compile_and_an_additive_product_does_not(tmp_path):
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Wno-unused-function", "-fsyntax-only", "-I", str(ROOT / "include"),
                        str(ROOT / "tests" / "cpp" / "test_temporary.cpp")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    (tmp_path / "additive.cpp").write_text(CPP_ADDITIVE)
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", str(ROOT / "include"), str(tmp_path / "additive.cpp")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "vex::make_temp takes a vector expression" in r.stderr
