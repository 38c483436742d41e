"""The product kernel of user value types (vexb_usr_spmv), checked without a GPU: its source compiles for sm_90a with the
snippets of a 2 x 2 block, a complex and a double3 type in double and float, a host/device size mismatch fails in NVRTC
at the generated static_assert, and vexb_usr_create, vexb_usr_spmv and vexb_jit_source_usr refuse every malformed argument
before they touch a device."""
import ctypes as C

import numpy as np
import pytest

import usr_ops

NO_DEVICE = 4096          # an ordinal no machine has: valid arguments then fail at device selection, with VEXB_ERR_CUDA


@pytest.fixture(scope="module")
def L(built):
    from vexcl_b200 import _lib
    _lib.lib()
    return _lib


def make_ops(L, d):
    keep = [d[k].encode() for k in ("val_type", "rhs_type", "decl", "product", "append")]
    ops = L.UsrOps(keep[0], keep[1], d["rhs_bytes"], keep[2], keep[3], keep[4])
    ops._keep = keep
    return ops


def source(L, d, val_bytes, compile=True):
    ops = make_ops(L, d)
    n = C.c_size_t(0)
    code = L.lib().vexb_jit_source_usr(C.byref(ops), val_bytes, None, C.byref(n), compile)
    if code != L.OK:
        return code, L.lib().vexb_last_error().decode(errors="replace")
    buf = C.create_string_buffer(n.value)
    L.check(L.lib().vexb_jit_source_usr(C.byref(ops), val_bytes, buf, C.byref(n), compile))
    return code, buf.value.decode()


CASES = {
    "block_f64": (usr_ops.block(np.float64), 32), "block_f32": (usr_ops.block(np.float32), 16),
    "complex_f64": (usr_ops.complex_(np.float64), 16), "complex_f32": (usr_ops.complex_(np.float32), 8),
    "triple": (usr_ops.TRIPLE, 24),
}


@pytest.mark.parametrize("case", list(CASES))
def test_source_compiles_for_sm90a(L, case):
    d, vb = CASES[case]
    code, src = source(L, d, vb)
    assert code == L.OK, src
    assert "NVRTC: ok" in src
    # the snippets appear as written, in the batched loop and in the remainder loop; the accumulator is declared once
    assert src.count(d["product"]) == 2 and src.count(d["decl"]) == 1 and src.count(d["append"]) == 1
    assert f"sizeof(vexb_val_t) == {vb} && sizeof(vexb_rhs_t) == {d['rhs_bytes']}" in src


@pytest.mark.parametrize("val_bytes, rhs_bytes", [(24, 16), (32, 24), (16, 16)])
def test_size_mismatch_fails_in_nvrtc(L, val_bytes, rhs_bytes):
    d = dict(usr_ops.block(np.float64), rhs_bytes=rhs_bytes)      # double4 / double2: 32 and 16 bytes on the device
    code, msg = source(L, d, val_bytes)
    assert code == L.ERR_INVALID
    assert "NVRTC" in msg and "must have the sizes" in msg, msg


def test_syntax_error_carries_the_log(L):
    d = dict(usr_ops.TRIPLE, product="sum.x = sum.x + v.x * xv.x")   # no semicolon
    code, msg = source(L, d, 24)
    assert code == L.ERR_INVALID
    assert "NVRTC" in msg and "error" in msg and "expected a \";\"" in msg, msg


def test_source_without_compiling(L):
    code, src = source(L, usr_ops.TRIPLE, 24, compile=False)
    assert code == L.OK and "NVRTC: ok" not in src and "vexb_usr_kernel" in src


@pytest.mark.parametrize("case", ["ops_null", "val_type_null", "val_type_brace", "rhs_type_semicolon", "rhs_type_empty",
                                  "rhs_bytes_0", "rhs_bytes_65", "decl_null", "product_null", "append_null",
                                  "val_bytes_0", "val_bytes_6", "val_bytes_68", "len_null"])
def test_jit_source_rejects(L, case):
    d = dict(usr_ops.TRIPLE)
    vb = 24
    if case.startswith("val_type") or case.startswith("rhs_type") or case in ("decl_null", "product_null", "append_null"):
        key = case.rsplit("_", 1)[0]
        d[key] = {"null": None, "brace": "double3 {", "semicolon": "double3; int", "empty": ""}[case.rsplit("_", 1)[1]]
    elif case.startswith("rhs_bytes"):
        d["rhs_bytes"] = int(case.rsplit("_", 1)[1])
    elif case.startswith("val_bytes"):
        vb = int(case.rsplit("_", 1)[1])
    keep = [None if d[k] is None else d[k].encode() for k in ("val_type", "rhs_type", "decl", "product", "append")]
    ops = L.UsrOps(keep[0], keep[1], d["rhs_bytes"], keep[2], keep[3], keep[4])
    n = C.c_size_t(0)
    ops_arg = None if case == "ops_null" else C.byref(ops)
    len_arg = None if case == "len_null" else C.byref(n)
    assert L.lib().vexb_jit_source_usr(ops_arg, vb, None, len_arg, 0) == L.ERR_INVALID


# ---- vexb_usr_create argument checks (no device needed) ----------------------------------------------------------------
def _create(L, n=4, m=4, ptr=None, col=None, val=None, pb=4, cb=4, vb=24, dev=NO_DEVICE, out=True):
    ptr = np.array([0, 1, 1, 3, 4], np.int32) if ptr is None else ptr
    col = np.array([0, 3, 1, 2], np.int32) if col is None else col
    val = np.ones((4, 3), np.float64) if val is None else val
    h = C.c_void_p()
    arg = lambda a: a.ctypes.data_as(C.c_void_p) if isinstance(a, np.ndarray) else a
    return L.lib().vexb_usr_create(dev, None, n, m, arg(ptr), pb, arg(col), cb, arg(val), vb, C.byref(h) if out else None)


def test_create_with_valid_arguments_needs_a_device(L):
    assert _create(L) == L.ERR_CUDA
    assert _create(L, ptr=np.array([0, 1, 1, 3, 4], np.int64), col=np.array([0, 3, 1, 2], np.int64), pb=8, cb=8) == L.ERR_CUDA
    assert _create(L, vb=4, val=np.ones(4, np.float32)) == L.ERR_CUDA
    assert _create(L, vb=64, val=np.ones((4, 8), np.float64)) == L.ERR_CUDA
    assert _create(L, n=0, m=0, ptr=np.zeros(1, np.int32), col=np.zeros(0, np.int32), val=np.zeros((0, 3))) == L.ERR_CUDA


@pytest.mark.parametrize("case", [
    "val_bytes_0", "val_bytes_negative", "val_bytes_6", "val_bytes_68", "ptr_bytes2", "col_bytes16",
    "decreasing", "decreasing_first", "col_negative", "col_ncols", "ptr_null", "col_null", "val_null", "out_null",
    "nrows_overflow", "ncols_overflow", "nnz_overflow",
])
def test_create_rejects(L, case):
    kw = {
        "val_bytes_0": dict(vb=0), "val_bytes_negative": dict(vb=-8), "val_bytes_6": dict(vb=6), "val_bytes_68": dict(vb=68),
        "ptr_bytes2": dict(pb=2), "col_bytes16": dict(cb=16),
        "decreasing": dict(ptr=np.array([0, 2, 1, 3, 4], np.int32)),
        "decreasing_first": dict(ptr=np.array([1, 0, 1, 3, 4], np.int32)),
        "col_negative": dict(col=np.array([0, -1, 1, 2], np.int32)),
        "col_ncols": dict(col=np.array([0, 4, 1, 2], np.int32)),
        "ptr_null": dict(ptr=C.c_void_p(None)), "col_null": dict(col=C.c_void_p(None)), "val_null": dict(val=C.c_void_p(None)),
        "out_null": dict(out=False),
        "nrows_overflow": dict(n=2 ** 31),
        "ncols_overflow": dict(m=2 ** 31),
        "nnz_overflow": dict(n=1, ptr=np.array([0, 2 ** 31], np.int64), pb=8),
    }[case]
    assert _create(L, **kw) == L.ERR_INVALID, L.lib().vexb_last_error()


def test_spmv_rejects_a_null_matrix_or_ops(L):
    ops = make_ops(L, usr_ops.TRIPLE)
    assert L.lib().vexb_usr_spmv(0, None, None, C.byref(ops), None, None, 0) == L.ERR_INVALID
    assert L.lib().vexb_usrmat_get_info(None, None) == L.ERR_INVALID
    assert L.lib().vexb_usrmat_destroy(None) == L.OK
