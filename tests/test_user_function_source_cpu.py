"""User functions with dependencies and preambles, and per-device program headers, as far as they can be checked without
a GPU: the printed source of the kernels (vexb_jit_source*_dev print what a device would compile, its header included)
and NVRTC, which compiles for sm_90a without a device.  Checks the closure order, single emission and plain names, where
the header goes and where it does not, where the preamble and its NVRTC option appear, the name-clash refusal,
registration identity, the validation of every new ABI argument, and that the C++ spellings register what they say.
The numerical checks are in tests/test_gpu_user_function_spellings.py and tests/cpp/test_user_functions.cpp."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
DEV = 5                 # a device ordinal for header tests: headers are host state, so no such device has to exist


@pytest.fixture(scope="module")
def env(built):
    import vexcl_b200 as vx
    from vexcl_b200 import api, _lib as L

    class FakeCtx:
        nparts, local, devs, streams, weights = 1, [0], {0: DEV}, {0: None}, None
        def partition(self, n): return vx.partition(n, 1)

    def fake_vec(n, dt, addr):
        v = api.vector.__new__(api.vector)
        v.ctx, v.n, v.np_dtype, v.dtype, v.part, v.bufs = FakeCtx(), n, np.dtype(dt), api._vdt(dt), vx.partition(n, 1), {0: C.c_void_p(addr)}
        return v
    return vx, api, L, fake_vec, FakeCtx()


def _lower(api, lhs, expr):
    low = api._Lowering(0, 0)
    low.size = lhs.n
    low.lower(api.wrap(expr))
    return low


def _text(fn, *args, compile=True):
    n = C.c_size_t(0)
    fn(*args, None, C.byref(n), 0)
    buf = C.create_string_buffer(n.value + 4096)
    cap = C.c_size_t(len(buf))
    return fn(*args, buf, C.byref(cap), int(compile)), buf.value.decode()


def source(L, lhs, expr_low, dev=-1, op=None, compile=True):
    api_op = 0 if op is None else op
    st, txt = _text(L.lib().vexb_jit_source_dev, dev, lhs.dtype, api_op, C.byref(expr_low.e), compile=compile)
    L.check(st)
    return txt


def reduce_source(L, low, dev=-1, ops=(0,), compile=True):
    arr = (C.c_int * len(ops))(*ops)
    st, txt = _text(L.lib().vexb_jit_source_reduce_dev, dev, L.F64, len(ops), arr, C.byref(low.e), compile=compile)
    L.check(st)
    return txt


def multi_source(L, lhs_dtype, lows, dev=-1, compile=True):
    arr = (C.POINTER(L.Expr) * len(lows))(*[C.pointer(lw.e) for lw in lows])
    st, txt = _text(L.lib().vexb_jit_source_multi_dev, dev, lhs_dtype, L.SET, len(lows), arr, compile=compile)
    L.check(st)
    return txt


def _defs(src):
    """Names of the user functions defined in a printed program, in order (reductions: after the embedded fold code)."""
    out = []
    for line in src.split("// end of fold.cuh")[-1].splitlines():
        if line.startswith("__device__ __forceinline__ ") and "(" in line and not line.split("(")[0].split()[-1].startswith(("vexb_", "spmv_", "ccsr_")):
            out.append(line.split("(")[0].split()[-1])
    return out


@pytest.fixture(autouse=True)
def no_header_left(env):
    vx = env[0]
    yield
    while vx.program_header(DEV):                     # a failed test must not leave a header to the next one
        vx.pop_program_header(env[4])


def test_closure_order_single_emission_and_plain_names(env):
    vx, api, L, fake_vec, _ = env
    x, y = fake_vec(1000, np.float64, 0x1000), fake_vec(1000, np.float64, 0x2000)
    a = api.UserFunction(np.float64, "cl_a", [(np.float64, "x")], "return x + 1;")
    b = api.UserFunction(np.float64, "cl_b", [(np.float64, "x")], "return cl_a(x) * 2;", deps=[a])
    c = api.UserFunction(np.float64, "cl_c", [(np.float64, "x")], "return cl_b(x) - cl_a(x);", deps=[b, a])
    d = api.UserFunction(np.float64, "cl_d", [(np.float64, "x")], "return cl_a(x) * x;", deps=[a])
    # three levels: post-order over the lists as written, each function once, the called one as name_<id>
    src = source(L, y, _lower(api, y, c(x)))
    assert _defs(src) == ["cl_a", "cl_b", f"cl_c_{c.id}"]
    assert "NVRTC: ok" in src
    # a dependency the expression also calls directly: under both names, the plain one once
    src = source(L, y, _lower(api, y, a(x) + c(x)))
    assert _defs(src) == [f"cl_a_{a.id}", "cl_a", "cl_b", f"cl_c_{c.id}"]
    assert "NVRTC: ok" in src
    # one dependency shared by two called functions
    src = source(L, y, _lower(api, y, d(x) * c(x) + d(y)))
    assert _defs(src) == ["cl_a", f"cl_d_{d.id}", "cl_b", f"cl_c_{c.id}"]
    assert src.count("cl_a(double prm1)") == 1 and "NVRTC: ok" in src
    # the argument prologue and the emission form are those of any user function
    assert "__device__ __forceinline__ double cl_a(double prm1) {\nconst double x = prm1; return x + 1;\n}\n" in src
    # reductions and multi-expressions hold the same closure
    rsrc = reduce_source(L, _lower(api, y, c(x) * y))
    assert _defs(rsrc) == ["cl_a", "cl_b", f"cl_c_{c.id}"] and "NVRTC: ok" in rsrc
    msrc = multi_source(L, L.F64, [_lower(api, y, c(x)), _lower(api, y, d(y) + x)])
    assert _defs(msrc) == ["cl_a", "cl_b", f"cl_c_{c.id}", f"cl_d_{d.id}"] and "NVRTC: ok" in msrc


def test_plain_name_clash_is_refused_before_nvrtc(env):
    vx, api, L, fake_vec, _ = env
    x, y = fake_vec(100, np.float64, 0x1000), fake_vec(100, np.float64, 0x2000)
    h1 = api.UserFunction(np.float64, "clash_h", [(np.float64, "x")], "return x + 1;")
    h2 = api.UserFunction(np.float64, "clash_h", [(np.float64, "x")], "return x + 2;")
    assert h1.id != h2.id
    f = api.UserFunction(np.float64, "clash_f", [(np.float64, "x")], "return clash_h(x);", deps=[h1])
    g = api.UserFunction(np.float64, "clash_g", [(np.float64, "x")], "return clash_h(x);", deps=[h2])
    source(L, y, _lower(api, y, f(x) + h2(x)))               # h2 called directly is h2_<id>: no clash
    low = _lower(api, y, f(x) + g(x))
    for fn, args in ((L.lib().vexb_jit_source_dev, (-1, y.dtype, 0, C.byref(low.e))),
                     (L.lib().vexb_jit_source_reduce_dev, (-1, L.F64, 1, (C.c_int * 1)(0), C.byref(low.e)))):
        st, _ = _text(fn, *args, compile=True)
        assert st == L.ERR_INVALID
        msg = L.lib().vexb_last_error().decode()
        assert f"{h1.id} and {h2.id}" in msg and "clash_h" in msg and "NVRTC" not in msg
    both = api.UserFunction(np.float64, "clash_both", [(np.float64, "x")], "return 0;", deps=[f, g])
    st, _ = _text(L.lib().vexb_jit_source_dev, -1, y.dtype, 0, C.byref(_lower(api, y, both(x)).e), compile=False)
    assert st == L.ERR_INVALID


def test_header_first_and_only_on_user_text(env):
    vx, api, L, fake_vec, ctx = env
    x, y = fake_vec(1000, np.float64, 0x1000), fake_vec(1000, np.float64, 0x2000)
    f = api.UserFunction(np.float64, "hdr_f", [(np.float64, "x")], "return x * HDR_SCALE;")
    plain = _lower(api, y, x * 2.0 + y)
    call = _lower(api, y, f(x) + y)
    before_plain = source(L, y, plain, dev=-1, compile=False)
    vx.push_program_header(ctx, "#define HDR_SCALE 3.0\n")
    assert vx.program_header(DEV) == "#define HDR_SCALE 3.0\n"
    src = source(L, y, call, dev=DEV)
    assert src.startswith("#define HDR_SCALE 3.0\n// generated by libvexb200") and "NVRTC: ok" in src
    assert source(L, y, call, dev=-1, compile=False).startswith("// generated")            # no device: no header
    assert source(L, y, plain, dev=DEV, compile=False) == before_plain                      # no user text: no header
    assert source(L, y, call, dev=DEV + 1, compile=False).startswith("// generated")       # another device's stack
    rsrc = reduce_source(L, _lower(api, y, f(x) * y), dev=DEV)
    assert rsrc.startswith("#define HDR_SCALE 3.0\n// generated by libvexb200 (csrc/jit.cu): reduction") and "NVRTC: ok" in rsrc
    assert not reduce_source(L, _lower(api, y, x * y), dev=DEV, compile=False).startswith("#define")
    msrc = multi_source(L, L.F64, [_lower(api, y, x + 1.0), _lower(api, y, f(y))], dev=DEV)
    assert msrc.startswith("#define HDR_SCALE 3.0\n") and "NVRTC: ok" in msrc
    # a push replaces the header, a pop restores it; a header without a final newline gets a line of its own
    vx.push_program_header(ctx, "#define HDR_SCALE 5.0")
    assert source(L, y, call, dev=DEV, compile=False).startswith("#define HDR_SCALE 5.0\n// generated")
    vx.pop_program_header(ctx)
    assert source(L, y, call, dev=DEV, compile=False).startswith("#define HDR_SCALE 3.0\n// generated")
    vx.pop_program_header(ctx)
    assert vx.program_header(DEV) == ""
    with pytest.raises(vx.VexbError):                      # HDR_SCALE is undefined without the header
        source(L, y, call, dev=DEV)


def test_push_and_pop_once_per_distinct_device(env):
    vx, api, L, _, _ = env

    class TwoSlotsOneDevice:
        local, devs = [0, 1, 2], {0: DEV, 1: DEV, 2: DEV + 1}
    c2 = TwoSlotsOneDevice()
    vx.push_program_header(c2, "A")
    vx.push_program_header(c2, "B")
    vx.pop_program_header(c2)
    assert vx.program_header(DEV) == "A" and vx.program_header(DEV + 1) == "A"
    vx.pop_program_header(c2)
    assert vx.program_header(DEV) == "" and vx.program_header(DEV + 1) == ""


def test_preamble_and_its_option_only_where_a_preamble_exists(env):
    vx, api, L, fake_vec, _ = env
    x, y = fake_vec(1000, np.float64, 0x1000), fake_vec(1000, np.float64, 0x2000)
    # the reference's example (vexcl/function.hpp:94-100): helpers without __device__
    pre = ("double sin2(double x) { return pow(sin(x), 2.0); }\n"
           "double cos2(double x) { return pow(cos(x), 2.0); }\n")
    one = api.UserFunction(np.float64, "pre_one", [(np.float64, "x")], "return sin2(prm1) + cos2(prm1);", preamble=pre)
    dep = api.UserFunction(np.float64, "pre_dep", [(np.float64, "x")], "return pre_one(x) * 2;", deps=[one])
    plain = api.UserFunction(np.float64, "pre_none", [(np.float64, "x")], "return x * 2;")
    src = source(L, y, _lower(api, y, one(x) + dep(x)))
    assert src.count(pre) == 1                              # once per function and program
    assert src.index(pre) < src.index(f"double pre_one_{one.id}(") < src.index("double pre_one(")
    assert "NVRTC: ok" in src
    assert "NVRTC: ok" in reduce_source(L, _lower(api, y, dep(x)))
    assert "double sin2" not in source(L, y, _lower(api, y, plain(x)), compile=False)
    # The option itself: a helper without __device__ in the program header is a host function, which device code can
    # call only under --device-as-default-execution-space.  A program without a preamble is compiled without it, so the
    # call fails; the same program with any preamble compiles.
    helper = "double hdr_helper(double x) { return x + 1; }\n"
    uses = api.UserFunction(np.float64, "pre_uses", [(np.float64, "x")], "return hdr_helper(x);")
    uses_pre = api.UserFunction(np.float64, "pre_uses", [(np.float64, "x")], "return hdr_helper(x);", preamble="// none\n")
    vx.push_program_header(env[4], helper)
    with pytest.raises(vx.VexbError):
        source(L, y, _lower(api, y, uses(x)), dev=DEV)
    assert "NVRTC: ok" in source(L, y, _lower(api, y, uses_pre(x)), dev=DEV)
    vx.pop_program_header(env[4])


def test_registration_identity(env):
    vx, api, L, _, _ = env
    args = [(np.float64, "x")]
    base = api.UserFunction(np.float64, "id_f", args, "return x;")
    dep = api.UserFunction(np.float64, "id_g", args, "return x;")
    assert api.UserFunction(np.float64, "id_f", args, "return x;").id == base.id
    variants = [api.UserFunction(np.float64, "id_f2", args, "return x;"),
                api.UserFunction(np.float32, "id_f", args, "return x;"),
                api.UserFunction(np.float64, "id_f", [(np.float32, "x")], "return x;"),
                api.UserFunction(np.float64, "id_f", args, "return x ;"),
                api.UserFunction(np.float64, "id_f", args, "return x;", deps=[dep]),
                api.UserFunction(np.float64, "id_f", args, "return x;", deps=[dep, dep]),
                api.UserFunction(np.float64, "id_f", args, "return x;", preamble="// p\n")]
    ids = [base.id] + [v.id for v in variants]
    assert len(set(ids)) == len(ids)
    assert api.UserFunction(np.float64, "id_f", args, "return x;", deps=[dep]).id == variants[4].id
    assert api.UserFunction(np.float64, "id_f", args, "return x;", preamble="// p\n").id == variants[6].id
    # vexb_function_register is register_ex without dependencies and preamble
    fid = C.c_int(-1)
    L.check(L.lib().vexb_function_register_ex(b"id_f", L.F64, 1, (C.c_int * 1)(L.F64), b"const double x = prm1; return x;",
                                              0, None, None, C.byref(fid)))
    assert fid.value == base.id


def test_abi_argument_validation(env):
    vx, api, L, fake_vec, _ = env
    lib = L.lib()
    fid = C.c_int(-1)
    one = (C.c_int * 1)(L.F64)
    ok = api.UserFunction(np.float64, "val_ok", [(np.float64, "x")], "return x;")

    def reg(name=b"val_f", nargs=1, at=one, body=b"return prm1;", ndeps=0, deps=None, pre=None, out=C.byref(fid)):
        return lib.vexb_function_register_ex(name, L.F64, nargs, at, body, ndeps, deps, pre, out)
    assert reg() == L.OK
    assert reg(ndeps=1, deps=(C.c_int * 1)(ok.id)) == L.OK
    for bad in (dict(name=None), dict(body=None), dict(out=None), dict(ndeps=-1), dict(ndeps=65, deps=(C.c_int * 65)()),
                dict(ndeps=1, deps=None), dict(ndeps=1, deps=(C.c_int * 1)(-1)), dict(ndeps=1, deps=(C.c_int * 1)(1 << 20)),
                dict(name=b"not a name"), dict(nargs=1, at=None)):
        assert reg(**bad) == L.ERR_INVALID, bad
    n = C.c_size_t(0)
    assert lib.vexb_program_header_push(-1, b"x") == L.ERR_INVALID
    assert lib.vexb_program_header_push(DEV, None) == L.ERR_INVALID
    assert lib.vexb_program_header_pop(-1) == L.ERR_INVALID
    assert lib.vexb_program_header_pop(DEV) == L.ERR_INVALID and "no program header" in lib.vexb_last_error().decode()
    assert lib.vexb_program_header_get(-1, None, C.byref(n)) == L.ERR_INVALID
    assert lib.vexb_program_header_get(DEV, None, None) == L.ERR_INVALID
    L.check(lib.vexb_program_header_push(DEV, b"#define V 1\n"))
    small = C.create_string_buffer(4)
    cap = C.c_size_t(4)
    assert lib.vexb_program_header_get(DEV, small, C.byref(cap)) == L.ERR_INVALID            # buffer too small
    L.check(lib.vexb_program_header_get(DEV, None, C.byref(n)))
    assert n.value == len("#define V 1\n") + 1
    L.check(lib.vexb_program_header_pop(DEV))
    x, y = fake_vec(10, np.float64, 0x1000), fake_vec(10, np.float64, 0x2000)
    low = _lower(api, y, ok(x))
    assert lib.vexb_jit_source_dev(-2, y.dtype, 0, C.byref(low.e), None, C.byref(n), 0) == L.ERR_INVALID
    assert lib.vexb_jit_source_reduce_dev(-2, L.F64, 1, (C.c_int * 1)(0), C.byref(low.e), None, C.byref(n), 0) == L.ERR_INVALID
    arr = (C.POINTER(L.Expr) * 2)(C.pointer(low.e), C.pointer(low.e))
    assert lib.vexb_jit_source_multi_dev(-2, y.dtype, 0, 2, arr, None, C.byref(n), 0) == L.ERR_INVALID


def test_header_less_printers_are_the_dev_minus_one_printers(env):
    vx, api, L, fake_vec, ctx = env
    x, y = fake_vec(1000, np.float64, 0x1000), fake_vec(1000, np.float64, 0x2000)
    f = api.UserFunction(np.float64, "old_f", [(np.float64, "x")], "return x * 2;")
    low = _lower(api, y, f(x) + y)
    vx.push_program_header(ctx, "#define UNUSED 1\n")
    st, old = _text(L.lib().vexb_jit_source, y.dtype, 0, C.byref(low.e), compile=False)
    L.check(st)
    assert old == source(L, y, low, dev=-1, compile=False)
    assert source(L, y, low, dev=DEV, compile=False) == "#define UNUSED 1\n" + old
    vx.pop_program_header(ctx)


CPP = r"""
#include <cstdio>
#include <vexcl/vexcl.hpp>
VEX_FUNCTION(double, sin2, (double, x), return pow(sin(x), 2.0););
VEX_FUNCTION_S(double, cos2, (double, x), "return pow(cos(x), 2.0);");
VEX_FUNCTION_D(double, one, (double, x), (sin2)(cos2), return sin2(x) + cos2(x););
VEX_FUNCTION_SD(double, two, (double, x), (one), "return one(x) + one(x);");
VEX_FUNCTION_DS(double, three, (double, x), (two)(sin2), VEX_STRINGIZE_SOURCE(return two(x) + sin2(x);));
VEX_FUNCTION_V1(v1, double(double), "return prm1;");
VEX_FUNCTION_V1_WITH_PREAMBLE(v1p, double(double), "double helper(double x) { return x; }\n", "return helper(prm1);");
VEX_FUNCTION_V1_TYPE(v1t, double(double, double), "", "return prm1 * prm2;");
int main() {
    const vex_function_v1t v1t;
    const int ids[] = {three.id(), v1.id(), v1p.id(), v1t.id()};
    for (int id : ids) {
        vexb_expr e = {};
        e.n_terms = 1; e.term[0].kind = VEXB_TERM_VEC; e.term[0].dtype = VEXB_F64; e.term[0].v.ptr = (void *)0x1000;
        int nargs = id == v1t.id() ? 2 : 1;
        for (int k = 0; k < nargs; ++k) { e.code[e.n_code].op = VEXB_OP_TERM; e.code[e.n_code].type = VEXB_F64; e.code[e.n_code++].arg = 0; }
        e.code[e.n_code].op = VEXB_OP_CALL; e.code[e.n_code].type = VEXB_F64; e.code[e.n_code++].arg = (uint16_t)id;
        size_t len = 0;
        if (vexb_jit_source(VEXB_F64, VEXB_SET, &e, nullptr, &len, 0) != VEXB_OK) { std::printf("error: %s\n", vexb_last_error()); return 1; }
        std::string s(len + 4096, '\0');
        len = s.size();
        if (vexb_jit_source(VEXB_F64, VEXB_SET, &e, &s[0], &len, 1) != VEXB_OK) { std::printf("error: %s\n", vexb_last_error()); return 1; }
        std::printf("=== %d\n%s", id, s.c_str());
    }
    return 0;
}
"""


def test_cpp_spellings_register_their_dependencies_and_compile(env, tmp_path):
    """The C++ macros without a device: every spelling registers, VEX_FUNCTION_D / _SD / _DS register their dependency
    sequences (walked by the preprocessor), and the programs they make compile with NVRTC."""
    (tmp_path / "spell.cpp").write_text(CPP)
    lib_dir = ROOT / "vexcl_b200"
    exe = tmp_path / "spell"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", str(ROOT / "include"), str(tmp_path / "spell.cpp"), "-o", str(exe),
                    "-L", str(lib_dir), "-lvexb200", f"-Wl,-rpath,{lib_dir}"], check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300, env=dict(os.environ))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    parts = r.stdout.split("=== ")[1:]
    assert len(parts) == 4 and all("NVRTC: ok" in p for p in parts)
    three = parts[0]
    assert _defs(three) == ["sin2", "cos2", "one", "two", three.split("\n")[0].join(["three_", ""])]
    assert "return two(x) + sin2(x);" in three
    v1p = parts[2]
    assert v1p.index("double helper(double x)") < v1p.index("double v1p_")
