"""The source printers of the run-time compiled kernels, without a GPU: with compile = 0 each prints exactly the text
pinned in tests/golden/jit_printers.json.  The same text reaches NVRTC when a device builds the kernel, so this pins the
programs themselves: the matrix-specialised CCSR kernel (three value / idx-width pairs), the user-defined stencil
operator, the product kernel of user value types, and the elementwise, multi-expression and reduction kernels of a
program that calls a user function with a dependency and a preamble, printed for a device with a pushed program
header.  User-function ids depend on what the process registered before, so they are printed as <id>."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

import usr_ops

GOLDEN = Path(__file__).resolve().parent / "golden" / "jit_printers.json"
DEV = 7                 # a device ordinal for the header: headers are host state, so no such device has to exist
HEADER = "#define JP_SCALE 3.0\n"


def _text(L, fn, *args):
    n = C.c_size_t(0)
    L.check(fn(*args, None, C.byref(n), 0))
    buf = C.create_string_buffer(n.value)
    L.check(fn(*args, buf, C.byref(n), 0))
    return buf.value.decode()


@pytest.fixture(scope="module")
def printed(built):
    import vexcl_b200 as vx
    from vexcl_b200 import api, gen, _lib as L
    lib = L.lib()
    out = {}

    # CCSR: the Poisson table in double with 1-byte idx, a random table in float with 2-byte idx, and in double with 4
    _, row, col, val = gen.poisson_ccsr(32)
    rng = np.random.default_rng(2)
    row2, col2 = np.array([0, 0, 11, 14], np.int32), rng.integers(-50, 50, 14).astype(np.int32)
    val2 = rng.random(14)
    for name, (r, c, v, idx) in {"ccsr_f64_idx1": (row, col, val, 1), "ccsr_f32_idx2": (row2, col2, val2.astype(np.float32), 2),
                                 "ccsr_f64_idx4": (row2, col2, val2, 4)}.items():
        r, c, v = np.ascontiguousarray(r, np.int32), np.ascontiguousarray(c, np.int32), np.ascontiguousarray(v)
        out[name] = _text(L, lib.vexb_ccsr_jit_source, r.size - 1, r.ctypes.data, c.ctypes.data, v.ctypes.data,
                          L.F64 if v.dtype == np.float64 else L.F32, idx)

    for name, (dt, width, center, body) in {"stencil_f64": (L.F64, 3, 1, "return sin(X[1] - X[0]) + sin(X[0] - X[-1]);"),
                                            "stencil_f32": (L.F32, 5, 0, "return X[0] + powf(X[1] + X[4], 3.0f);")}.items():
        k = C.c_int(-1)
        L.check(lib.vexb_stencil_operator_register(dt, width, center, body.encode(), C.byref(k)))
        out[name] = _text(L, lib.vexb_stencil_operator_source, k.value)

    for name, (d, val_bytes) in {"usr_triple": (usr_ops.TRIPLE, 24), "usr_block_f32": (usr_ops.block(np.float32), 16)}.items():
        keep = [d[k].encode() for k in ("val_type", "rhs_type", "decl", "product", "append")]
        ops = L.UsrOps(keep[0], keep[1], d["rhs_bytes"], keep[2], keep[3], keep[4])
        out[name] = _text(L, lib.vexb_jit_source_usr, C.byref(ops), val_bytes)

    class FakeCtx:
        nparts, local, devs, streams, weights = 1, [0], {0: DEV}, {0: None}, None
        def partition(self, n): return vx.partition(n, 1)

    def fake_vec(n, dt, addr):
        v = api.vector.__new__(api.vector)
        v.ctx, v.n, v.np_dtype, v.dtype, v.part, v.bufs = FakeCtx(), n, np.dtype(dt), api._vdt(dt), vx.partition(n, 1), {0: C.c_void_p(addr)}
        return v

    def lowered(expr):
        low = api._Lowering(0, 0)
        low.size = 1000
        low.lower(api.wrap(expr))
        return low

    x, y = fake_vec(1000, np.float64, 0x1000), fake_vec(1000, np.float64, 0x2000)
    half = api.UserFunction(np.float64, "jp_half", [(np.float64, "x")], "return jp_helper(x) * JP_SCALE;",
                            preamble="double jp_helper(double v) { return v / 2; }\n")
    top = api.UserFunction(np.float64, "jp_top", [(np.float64, "x")], "return jp_half(x) + x;", deps=[half])
    ids = {f"jp_half_{half.id}": "jp_half_<id>", f"jp_top_{top.id}": "jp_top_<id>"}
    L.check(lib.vexb_program_header_push(DEV, HEADER.encode()))
    try:
        out["eval_dev"] = _text(L, lib.vexb_jit_source_dev, DEV, L.F64, L.SET, C.byref(lowered(top(x) + y).e))
        lows = [lowered(top(x)), lowered(half(y) + x)]
        arr = (C.POINTER(L.Expr) * 2)(*[C.pointer(lw.e) for lw in lows])
        out["multi_dev"] = _text(L, lib.vexb_jit_source_multi_dev, DEV, L.F64, L.SET, 2, arr)
        red = lowered(top(x) * y)
        out["reduce_dev"] = _text(L, lib.vexb_jit_source_reduce_dev, DEV, L.F64, 1, (C.c_int * 1)(L.SUM), C.byref(red.e))
        out["reduce_multi_dev"] = _text(L, lib.vexb_jit_source_reduce_dev, DEV, L.F64, 2, (C.c_int * 2)(L.SUM, L.MAX), C.byref(red.e))
    finally:
        L.check(lib.vexb_program_header_pop(DEV))
    for name in ("eval_dev", "multi_dev", "reduce_dev", "reduce_multi_dev"):
        assert out[name].startswith(HEADER)
        for k, v in ids.items():
            out[name] = out[name].replace(k, v)
    return out


def test_printers_print_the_pinned_sources(printed):
    want = json.loads(GOLDEN.read_text())
    assert sorted(printed) == sorted(want)
    for name in want:
        assert printed[name] == want[name], name
