"""CPU checks of complex sparse matrices (vexb_zsr_create, tests/complex_oracle.py): the oracle gives the bits of the block
oracle on the [[a, -b], [b, a]] expansion, it reproduces the closed form of the reference's examples/complex_spmv.cpp, and
vexb_zsr_create rejects every malformed argument before it touches a device."""
import ctypes as C

import numpy as np
import pytest

import oracle
from block_oracle import bsr_spmv
from complex_oracle import as_blocks, zsr_spmv

CDTYPES = (np.complex128, np.complex64)
REAL = {np.complex128: np.float64, np.complex64: np.float32}
OPS = ((1.0, False), (1.0, True), (-1.0, True), (0.5, True), (0.37, False))


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def random_complex(n, m, cdtype, seed):
    row, col, _ = oracle.random_matrix(n, m, 32, seed)                 # widths U[0, 32)
    rng = np.random.default_rng(seed)
    val = (rng.standard_normal(col.size) + 1j * rng.standard_normal(col.size)).astype(cdtype)
    return row, col, val


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("cdtype", CDTYPES)
def test_oracle_matches_block_expansion(cdtype, seed):
    n, m = 700, 523
    ptr, col, val = random_complex(n, m, cdtype, seed)
    rng = np.random.default_rng(100 + seed)
    dt = REAL[cdtype]
    x = rng.standard_normal(2 * m).astype(dt)
    y = rng.standard_normal(2 * n).astype(dt)
    blocks = as_blocks(val)
    assert blocks.dtype == dt and blocks.shape == (val.size, 2, 2)
    for alpha, append in OPS:
        got = zsr_spmv(ptr, col, val, x, y if append else None, alpha, append)
        want = bsr_spmv(ptr, col, blocks, x, y if append else None, alpha, append)
        assert same_bits(got, want), (alpha, append)


@pytest.mark.parametrize("cdtype", CDTYPES)
def test_oracle_matches_complex_arithmetic(cdtype):
    """Against numpy's own complex product in float64 (exact enough at these sizes): the formula is a complex product."""
    ptr, col, val = random_complex(200, 150, cdtype, 9)
    x = np.random.default_rng(4).standard_normal(300).astype(REAL[cdtype])
    got = zsr_spmv(ptr, col, val, x).astype(np.float64).view(np.complex128)
    xz = x.astype(np.float64).view(np.complex128)
    want = np.array([np.sum(val[ptr[i]:ptr[i + 1]].astype(np.complex128) * xz[col[ptr[i]:ptr[i + 1]]]) for i in range(200)])
    tol = 1e-12 if cdtype == np.complex128 else 1e-4
    assert np.allclose(got, want, rtol=tol, atol=tol * 10)


@pytest.mark.parametrize("n", [4, 1000])
@pytest.mark.parametrize("cdtype", CDTYPES)
def test_example_closed_form(cdtype, n):
    """examples/complex_spmv.cpp: the diagonal (k+1)(1+i) times x = 1+i is exactly 0 + 2(k+1)i."""
    k = np.arange(n)
    ptr, col = np.arange(n + 1, dtype=np.int32), k.astype(np.int32)
    val = ((k + 1) * (1 + 1j)).astype(cdtype)
    x = np.ones(2 * n, REAL[cdtype])
    y = zsr_spmv(ptr, col, val, x)
    assert y.dtype == REAL[cdtype]
    assert np.all(y[0::2] == 0) and np.array_equal(y[1::2], (2 * (k + 1)).astype(REAL[cdtype]))


def test_empty_matrix():
    ptr, col, val = np.zeros(6, np.int32), np.zeros(0, np.int32), np.zeros(0, np.complex128)
    y0 = np.arange(10, dtype=np.float64)
    assert np.all(zsr_spmv(ptr, col, val, np.ones(8)) == 0)
    assert same_bits(zsr_spmv(ptr, col, val, np.ones(8), y0, 0.5, True), y0)


# ---- vexb_zsr_create argument checks (no device needed) ----------------------------------------------------------------
NO_DEVICE = 4096          # an ordinal no machine has: valid arguments then fail at device selection, with VEXB_ERR_CUDA


@pytest.fixture(scope="module")
def L(built):
    from vexcl_b200 import _lib
    _lib.lib()
    return _lib


def _create(L, n=4, m=4, ptr=None, col=None, val=None, pb=4, cb=4, vdt=None, dev=NO_DEVICE, out=True):
    ptr = np.array([0, 1, 1, 3, 4], np.int32) if ptr is None else ptr
    col = np.array([0, 3, 1, 2], np.int32) if col is None else col
    val = np.ones(4, np.complex128) if val is None else val
    vdt = L.F64 if vdt is None else vdt
    h = C.c_void_p()
    arg = lambda a: a.ctypes.data_as(C.c_void_p) if isinstance(a, np.ndarray) else a
    return L.lib().vexb_zsr_create(dev, None, n, m, arg(ptr), pb, arg(col), cb, arg(val), vdt, C.byref(h) if out else None)


def test_create_with_valid_arguments_needs_a_device(L):
    assert _create(L) == L.ERR_CUDA
    assert _create(L, ptr=np.array([0, 1, 1, 3, 4], np.int64), col=np.array([0, 3, 1, 2], np.int64), pb=8, cb=8) == L.ERR_CUDA
    assert _create(L, vdt=L.F32, val=np.ones(4, np.complex64)) == L.ERR_CUDA
    assert _create(L, n=0, m=0, ptr=np.zeros(1, np.int32), col=np.zeros(0, np.int32), val=np.zeros(0, np.complex128)) == L.ERR_CUDA


@pytest.mark.parametrize("case", [
    "dtype_i32", "dtype_bad", "ptr_bytes2", "col_bytes16",
    "decreasing", "decreasing_first", "col_negative", "col_ncols", "ptr_null", "col_null", "val_null", "out_null",
    "nrows_overflow", "ncols_overflow", "nnz_overflow",
])
def test_create_rejects(L, case):
    kw = {
        "dtype_i32": dict(vdt=L.I32), "dtype_bad": dict(vdt=77),
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


def test_spmv_rejects_a_null_matrix(L):
    assert L.lib().vexb_zspmv(0, None, None, None, None, 1.0, 0) == L.ERR_INVALID
    assert L.lib().vexb_zspmat_get_info(None, None) == L.ERR_INVALID
    assert L.lib().vexb_zspmat_destroy(None) == L.OK
