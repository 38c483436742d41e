"""CPU checks of double matrices with float-stored values (VEXB_FMT_VALUES_F32): vexb_csr_create and vexb_dspmat_create
check the flag, the value type and every value before they touch a device, and the C++ spelling
`vex::SpMat<double>(..., VEXB_FMT_AUTO | VEXB_FMT_VALUES_F32)` compiles.  No device needed: a request that passes every
check goes on to select device NO_DEVICE, which no machine has."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
NO_DEVICE = 4096
F32_MAX = float(np.finfo(np.float32).max)


@pytest.fixture(scope="module")
def L(built):
    from vexcl_b200 import _lib
    _lib.lib()
    return _lib


def _matrix(val):
    n = len(val)
    ptr = np.arange(n + 1, dtype=np.int64)
    col = np.arange(n, dtype=np.int64)
    return n, ptr, col, np.ascontiguousarray(val)


def _csr_create(L, fmt, val, vdt=None):
    n, ptr, col, val = _matrix(val)
    vdt = (L.F64 if val.dtype == np.float64 else L.F32) if vdt is None else vdt
    h = C.c_void_p()
    code = L.lib().vexb_csr_create(NO_DEVICE, None, n, n, ptr.ctypes.data, 8, col.ctypes.data, 8, val.ctypes.data, vdt, fmt,
                                   C.byref(h))
    return code, L.lib().vexb_last_error().decode()


def _dspmat_create(L, fmt, val, vdt=None):
    n, ptr, col, val = _matrix(val)
    vdt = (L.F64 if val.dtype == np.float64 else L.F32) if vdt is None else vdt
    plan = C.c_void_p()
    cp = (C.c_size_t * 2)(0, n)
    off = (C.c_size_t * 2)(0, 0)
    L.check(L.lib().vexb_halo_plan_create(1, cp, None, off, C.byref(plan)))
    try:
        h = C.c_void_p()
        code = L.lib().vexb_dspmat_create(NO_DEVICE, None, 0, plan, n, ptr.ctypes.data, 8, col.ctypes.data, 8,
                                          val.ctypes.data, vdt, fmt, C.byref(h))
        return code, L.lib().vexb_last_error().decode()
    finally:
        L.lib().vexb_halo_plan_destroy(plan)


CREATE = {"csr": _csr_create, "dspmat": _dspmat_create}
VALUES = [0.1, -2.0 / 3.0, 1e-300, F32_MAX, -F32_MAX, np.inf, 1e300 * 0.0]


def test_flag_value(L):
    import vexcl_b200 as vx
    assert vx.FMT_VALUES_F32 == L.FMT_VALUES_F32 == 0x100
    assert "#define VEXB_FMT_VALUES_F32 0x100" in L.HEADER.read_text()
    assert [f for f, _ in L.SpmatInfo._fields_][-1] == "val_bytes"


@pytest.mark.parametrize("which", list(CREATE))
@pytest.mark.parametrize("base", [0, 1, 2, 3, 4])
def test_valid_requests_reach_the_device(L, which, base):
    """Every format with the flag, values that round to finite floats (and infinities, which stay infinite): all checks
    pass, and the call stops at the missing device."""
    code, msg = CREATE[which](L, base | L.FMT_VALUES_F32, np.array(VALUES))
    assert code == L.ERR_INVALID and "cannot select device" in msg, msg


@pytest.mark.parametrize("which", list(CREATE))
@pytest.mark.parametrize("case", ["f32_values", "unknown_bit", "unknown_bit_with_flag", "high_bit", "bad_base", "negative",
                                  "overflow", "overflow_negative", "overflow_rounding"])
def test_rejected_before_the_device(L, which, case):
    fmt, val, vdt = L.FMT_AUTO | L.FMT_VALUES_F32, np.array(VALUES), None
    if case == "f32_values":
        val = np.array(VALUES, np.float32)
    elif case == "unknown_bit":
        fmt = 0x200
    elif case == "unknown_bit_with_flag":
        fmt = L.FMT_VALUES_F32 | 0x80
    elif case == "high_bit":
        fmt = L.FMT_HELL | L.FMT_VALUES_F32 | (1 << 20)
    elif case == "bad_base":
        fmt = 5 | L.FMT_VALUES_F32
    elif case == "negative":
        fmt = -1
    elif case == "overflow":
        val = np.array([1.0, 1e39, 2.0])
    elif case == "overflow_negative":
        val = np.array([1.0, 2.0, -3.5e38])
    elif case == "overflow_rounding":
        # the smallest double that rounds to +inf in float: FLT_MAX + half an ulp (a tie, rounded to even = up)
        val = np.array([np.float64(F32_MAX) + 2.0 ** 103, 1.0])
        with np.errstate(over="ignore"):
            assert np.isinf(val.astype(np.float32)[0])
    code, msg = CREATE[which](L, fmt, val, vdt)
    assert code == L.ERR_INVALID, msg
    assert "cannot select device" not in msg, msg


def test_largest_values_below_overflow_pass(L):
    """FLT_MAX + half an ulp - one double ulp rounds down to FLT_MAX: accepted."""
    v = np.nextafter(np.float64(F32_MAX) + 2.0 ** 103, 0.0)
    assert np.isfinite(np.float32(v))
    for create in CREATE.values():
        code, msg = create(L, L.FMT_CSR | L.FMT_VALUES_F32, np.array([v, -v]))
        assert "cannot select device" in msg, msg


def test_flag_without_it_unchanged(L):
    """Without the flag, float and double values and every format reach the device as before."""
    for create in CREATE.values():
        for base in range(5):
            for val in (np.array([1.5, 1e39]), np.array([1.5, 2.5], np.float32)):
                code, msg = create(L, base, val)
                assert "cannot select device" in msg, msg


def test_cpp_spelling_compiles():
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not found")
    src = """
#include <vexcl/vexcl.hpp>
#include <vexcl/spmat.hpp>
void f(const std::vector<vex::backend::command_queue> &ctx, size_t n, const std::vector<size_t> &row,
       const std::vector<int> &col, const std::vector<double> &val) {
    vex::SpMat<double, int, size_t> A(ctx, n, n, row.data(), col.data(), val.data(), VEXB_FMT_AUTO | VEXB_FMT_VALUES_F32);
    vex::vector<double> X(ctx, n), Y(ctx, n);
    Y = A * X;
    Y -= 2 * (A * X);
    Y = X + A * X;
    Y = X + vex::make_inline(A * X);
    vexb_dspmat_info i = A.info();
    (void)i.loc.val_bytes;
}
"""
    r = subprocess.run([gxx, "-std=c++17", "-fsyntax-only", "-I", str(ROOT / "include"), "-x", "c++", "-"],
                       input=src, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
