"""The reduction kernels NVRTC generates for expressions with user functions, checked without a GPU: the source of all
three skeletons compiles for sm_90a, malformed requests are refused before anything is generated, and the fold the
program embeds is csrc/fold.cuh byte for byte (the pre-compiled reductions include that file)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

FOLD = Path(__file__).resolve().parent.parent / "vexcl_b200" / "csrc" / "fold.cuh"


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


def reduce_source(L, dtype, ops, low, compile=True):
    o = (C.c_int * max(len(ops), 1))(*ops)
    n = C.c_size_t(0)
    L.check(L.lib().vexb_jit_source_reduce(dtype, len(ops), o, C.byref(low.e), None, C.byref(n), 0))
    buf = C.create_string_buffer(n.value + 4096)
    cap = C.c_size_t(len(buf))
    L.check(L.lib().vexb_jit_source_reduce(dtype, len(ops), o, C.byref(low.e), buf, C.byref(cap), int(compile)))
    return buf.value.decode()


def test_three_skeletons_compile(env):
    vx, api, L, fake_vec = env
    x, y = fake_vec(1024, np.float64, 0x1000), fake_vec(1024, np.float64, 0x2000)
    xf = fake_vec(1024, np.float32, 0x3000)
    greater = api.UserFunction(np.uint64, "greater", [(np.float64, "x"), (np.float64, "y")], "return x > y;")
    times2 = api.UserFunction(np.float64, "times2", [(np.float64, "x")], "return x * 2;")
    halfF = api.UserFunction(np.float32, "halfF", [(np.float32, "v")], "return v * 0.5f;")

    # (a) sweep: one op, dtype equal to the expression's floating type
    for dt, e, E in ((L.F64, times2(x) - y, 4), (L.F32, halfF(xf), 8)):
        for op in (L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.MINMAX):
            src = reduce_source(L, dt, [op], lowered(api, e))
            assert f"constexpr int U = 2, E = {E};" in src and "acc[0][0].take(vexb_red_val(tt, i, off));" in src
            assert "NVRTC: ok" in src
    # (b) interpreter: an integer result, a float expression in double, a forced interpreter
    src = reduce_source(L, L.U64, [L.SUM], lowered(api, greater(x, y)))
    assert "constexpr int U = 4;" in src and "Fold<VEXB_SUM, unsigned long long>" in src and "NVRTC: ok" in src
    src = reduce_source(L, L.U64, [L.SUM_KAHAN], lowered(api, greater(x, y)), compile=False)
    assert "Fold<VEXB_SUM, unsigned long long>" in src                    # no compensation on integers
    src = reduce_source(L, L.F64, [L.SUM_KAHAN], lowered(api, halfF(xf)))
    assert "const float v = vexb_elem" in src and "return (double)v;" in src and "NVRTC: ok" in src
    vx.set_param("eval.force_interp", 1)
    try:
        src = reduce_source(L, L.F64, [L.SUM], lowered(api, times2(x)), compile=False)
    finally:
        vx.set_param("eval.force_interp", 0)
    assert "constexpr int U = 4;" in src
    # (c) combined
    for dt in (L.F64, L.F32, L.I32, L.I64):
        src = reduce_source(L, dt, [L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.SUM], lowered(api, times2(x) * greater(y, x)))
        assert "constexpr int U = 4, NOPS = 5;" in src and "4ull * ws_stride, result + 4" in src and "NVRTC: ok" in src


def test_embedded_fold_is_the_shared_header(env):
    vx, api, L, fake_vec = env
    x = fake_vec(1024, np.float64, 0x1000)
    times2 = api.UserFunction(np.float64, "times2", [(np.float64, "x")], "return x * 2;")
    src = reduce_source(L, L.F64, [L.SUM], lowered(api, times2(x)), compile=False)
    text = FOLD.read_text()
    start = src.index("// The device side of every reduction")
    end = src.index("// end of fold.cuh\n")
    assert src[start:end] == text
    assert src.count("struct Fold") == 1 and src.count("block_finish(") == 1      # no second copy
    # the pre-compiled reductions take the same file and hold no fold of their own
    csrc = FOLD.parent
    assert '#include "fold.cuh"' in (csrc / "peer.cuh").read_text()
    for f in ("reduce.cu", "peer.cuh", "jit.cu"):
        body = (csrc / f).read_text()
        assert "struct Fold" not in body and "void block_finish" not in body and "struct RtFold" not in body, f


def test_malformed_requests_are_refused(env):
    vx, api, L, fake_vec = env
    x = fake_vec(1024, np.float64, 0x1000)
    times2 = api.UserFunction(np.float64, "times2", [(np.float64, "x")], "return x * 2;")
    low = lowered(api, times2(x))
    lib = L.lib()
    n = C.c_size_t(0)
    one = (C.c_int * 1)(L.SUM)
    five = (C.c_int * 17)(*([L.SUM] * 17))
    bad = [
        (L.F64, 1, one, C.byref(low.e), None),                             # len NULL
        (7, 1, one, C.byref(low.e), C.byref(n)),                           # dtype
        (-1, 1, one, C.byref(low.e), C.byref(n)),
        (L.F64, 0, one, C.byref(low.e), C.byref(n)),                       # nops
        (L.F64, 17, five, C.byref(low.e), C.byref(n)),
        (L.F64, 1, None, C.byref(low.e), C.byref(n)),                      # ops NULL
        (L.F64, 1, (C.c_int * 1)(5), C.byref(low.e), C.byref(n)),          # bad op
        (L.F64, 2, (C.c_int * 2)(L.SUM, L.MINMAX), C.byref(low.e), C.byref(n)),   # MINMAX does not combine
        (L.F64, 1, one, None, C.byref(n)),                                 # expr NULL
    ]
    for dtype, nops, ops, expr, length in bad:
        assert lib.vexb_jit_source_reduce(dtype, nops, ops, expr, None, length, 0) == L.ERR_INVALID, (dtype, nops)
    e = lowered(api, times2(x)).e
    e.n_code = 0
    assert lib.vexb_jit_source_reduce(L.F64, 1, one, C.byref(e), None, C.byref(n), 0) == L.ERR_INVALID
    small = C.create_string_buffer(16)
    cap = C.c_size_t(16)
    assert lib.vexb_jit_source_reduce(L.F64, 1, one, C.byref(low.e), small, C.byref(cap), 0) == L.ERR_INVALID
    # a body that does not compile is reported with the compiler's log
    broken = api.UserFunction(np.float64, "broken_r", [(np.float64, "x")], "return x +;")
    with pytest.raises(vx.VexbError) as ei:
        reduce_source(L, L.F64, [L.SUM], lowered(api, broken(x)))
    assert "NVRTC could not compile" in str(ei.value)
