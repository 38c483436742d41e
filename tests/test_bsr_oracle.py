"""CPU checks of block sparse matrices (vexb_bsr_create, tests/block_oracle.py): the oracle restates the reference's
custom_values loop bit for bit, it reproduces that case's closed form, and vexb_bsr_create rejects every malformed
argument before it touches a device."""
import ctypes as C

import numpy as np
import pytest

from block_oracle import bsr_spmv, expand

BLOCKS = (2, 3, 4)
DTYPES = (np.float64, np.float32)


def loop_reference(ptr, col, val, x, y, alpha, append):
    """tests/sparse_matrices.cpp:271-281 written out for any B, one scalar operation at a time."""
    B = val.shape[1]
    dt = val.dtype.type
    n = len(ptr) - 1
    out = [dt(v) for v in y]
    for i in range(n):
        s = [dt(0)] * B
        for j in range(ptr[i], ptr[i + 1]):
            c = col[j]
            for r in range(B):
                t = val[j][r][0] * x[c * B]
                for q in range(1, B):
                    t = t + val[j][r][q] * x[c * B + q]
                s[r] = s[r] + t
        for r in range(B):
            v = dt(alpha) * s[r]
            out[i * B + r] = out[i * B + r] + v if append else v
    return np.array(out, dtype=val.dtype)


def small_matrix(rng, n, m, B, dtype):
    """Block rows of width 0..5 (some empty), columns in random order, one block row repeating a column."""
    ptr, col = [0], []
    for i in range(n):
        w = int(rng.integers(0, 6)) if i % 4 else 0
        cs = list(rng.integers(0, m, size=w))
        if i == 1:
            cs = [m - 1, 0, m - 1]
        col += cs
        ptr.append(len(col))
    val = rng.standard_normal((len(col), B, B)).astype(dtype)
    return np.array(ptr, np.int64), np.array(col, np.int64), val


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", BLOCKS)
def test_oracle_matches_reference_loop(B, dtype):
    rng = np.random.default_rng(10 * B + (dtype == np.float32))
    n, m = 23, 17
    ptr, col, val = small_matrix(rng, n, m, B, dtype)
    x = rng.standard_normal(m * B).astype(dtype)
    y = rng.standard_normal(n * B).astype(dtype)
    for alpha, append in ((1.0, False), (1.0, True), (-1.0, True), (0.5, True), (0.37, False)):
        want = loop_reference(ptr, col, val, x, y, alpha, append)
        got = bsr_spmv(ptr, col, val, x, y if append else None, alpha, append)
        assert same_bits(got, want), (alpha, append)


def mconst(c, B, dtype):
    return np.full((B, B), c, dtype)


def custom_values_matrix(n, B, dtype):
    """The matrix of the reference's custom_values case: tridiagonal blocks mconst(-1), mconst(2), mconst(-1)."""
    ptr, col, val = [0], [], []
    for i in range(n):
        if i > 0:
            col.append(i - 1); val.append(mconst(-1, B, dtype))
        col.append(i); val.append(mconst(2, B, dtype))
        if i + 1 < n:
            col.append(i + 1); val.append(mconst(-1, B, dtype))
        ptr.append(len(col))
    return np.array(ptr, np.int32), np.array(col, np.int32), np.array(val, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", BLOCKS)
def test_custom_values_closed_form(B, dtype):
    n = 1024
    ptr, col, val = custom_values_matrix(n, B, dtype)
    y = bsr_spmv(ptr, col, val, np.ones(n * B, dtype)).reshape(n, B)
    assert y.dtype == dtype
    assert np.all(y[0] == B) and np.all(y[-1] == B)
    assert np.all(y[1:-1] == 0)


@pytest.mark.parametrize("B", BLOCKS)
def test_expanded_csr_is_the_same_matrix(B):
    rng = np.random.default_rng(B)
    ptr, col, val = small_matrix(rng, 19, 11, B, np.float64)
    row, ecol, evals = expand(ptr, col, val)
    dense_b = np.zeros((19 * B, 11 * B))
    for i in range(19):
        for j in range(ptr[i], ptr[i + 1]):
            dense_b[i * B:(i + 1) * B, col[j] * B:(col[j] + 1) * B] += val[j]
    dense_e = np.zeros_like(dense_b)
    for i in range(19 * B):
        for j in range(row[i], row[i + 1]):
            dense_e[i, ecol[j]] += evals[j]
    assert np.array_equal(dense_b, dense_e)


# ---- vexb_bsr_create argument checks (no device needed) ----------------------------------------------------------------
NO_DEVICE = 4096          # an ordinal no machine has: valid arguments then fail at device selection, with VEXB_ERR_CUDA


@pytest.fixture(scope="module")
def L(built):
    from vexcl_b200 import _lib
    _lib.lib()
    return _lib


def _create(L, n=4, m=4, block=2, ptr=None, col=None, val=None, pb=4, cb=4, vdt=None, dev=NO_DEVICE, out=True):
    ptr = np.array([0, 1, 1, 3, 4], np.int32) if ptr is None else ptr
    col = np.array([0, 3, 1, 2], np.int32) if col is None else col
    val = np.ones(4 * block * block) if val is None else val
    vdt = L.F64 if vdt is None else vdt
    h = C.c_void_p()
    arg = lambda a: a.ctypes.data_as(C.c_void_p) if isinstance(a, np.ndarray) else a
    return L.lib().vexb_bsr_create(dev, None, n, m, block, arg(ptr), pb, arg(col), cb, arg(val), vdt,
                                   C.byref(h) if out else None)


def test_create_with_valid_arguments_needs_a_device(L):
    assert _create(L) == L.ERR_CUDA
    assert _create(L, ptr=np.array([0, 1, 1, 3, 4], np.int64), col=np.array([0, 3, 1, 2], np.int64), pb=8, cb=8) == L.ERR_CUDA
    assert _create(L, block=4, vdt=L.F32, val=np.ones(64, np.float32)) == L.ERR_CUDA
    assert _create(L, n=0, m=0, ptr=np.zeros(1, np.int32), col=np.zeros(0, np.int32), val=np.zeros(0)) == L.ERR_CUDA


@pytest.mark.parametrize("case", [
    "block1", "block5", "block0", "dtype_i32", "dtype_bad", "ptr_bytes2", "col_bytes16",
    "decreasing", "decreasing_first", "col_negative", "col_ncols", "ptr_null", "col_null", "val_null", "out_null",
    "nrows_overflow", "ncols_overflow", "nnzb_overflow",
])
def test_create_rejects(L, case):
    kw = {
        "block1": dict(block=1), "block5": dict(block=5), "block0": dict(block=0),
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
        "nnzb_overflow": dict(n=1, ptr=np.array([0, 2 ** 31], np.int64), pb=8),
    }[case]
    assert _create(L, **kw) == L.ERR_INVALID, L.lib().vexb_last_error()
