"""Sparse products of user value types on the GPU (vexb_usr_spmv, the kernel generated from spmv_ops_impl snippets):
bit-identical to the built-in vexb_bspmv (B = 2) and vexb_zspmv when the snippets spell their arithmetic, in float64 and
float32; bit-identical to a numpy restatement for a double3 type with `=` and `+=`, at the slice and sorting-window
boundaries with widths 0 to 40 and 32- and 64-bit indices; nothing written past y; info() against the host layout; an
NVRTC error carries its log; and the C++ front-end test tests/cpp/test_sparse_user_values.cpp."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle
import usr_ops

pytestmark = pytest.mark.gpu
BIN = Path(__file__).resolve().parent / "cpp" / "bin"
DTYPES = (np.float64, np.float32)
SIGMA = 1024                                   # spmv.sell_sigma default: the sorting window of the layout


def _vx():
    import vexcl_b200 as vx
    return vx


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def usr(ctx, n, m, ptr, col, val, ops):
    return _vx().UserValueMatrix(ctx, n, m, ptr, col, val, ops["val_type"], ops["rhs_type"], ops["rhs_bytes"],
                                 ops["decl"], ops["product"], ops["append"])


def random_pattern(n, m, seed, idx=np.int32):
    row, col, _ = oracle.random_matrix(n, m, 32, seed)                # widths U[0, 32), sorted unique columns
    return row.astype(idx), col.astype(idx)


def tridiagonal(n):
    ptr, col = [0], []
    for i in range(n):
        col += [c for c in (i - 1, i, i + 1) if 0 <= c < n]
        ptr.append(len(col))
    return np.array(ptr, np.int32), np.array(col, np.int32)


def boundary_pattern(n, idx, m=97):
    """Row i has width (7 i) mod 41: every width 0..40 appears, so both the batched slot loop and its remainder run."""
    w = (7 * np.arange(n)) % 41
    ptr = np.zeros(n + 1, np.int64); ptr[1:] = np.cumsum(w)
    col = np.random.default_rng(n).integers(0, m, size=int(ptr[-1]))
    return ptr.astype(idx), col.astype(idx)


def patterns():
    yield "tridiagonal", 1024, 1024, *tridiagonal(1024)
    yield "random", 3000, 2500, *random_pattern(3000, 2500, 13)
    yield "one_row", 1, 40, np.array([0, 5], np.int32), np.array([39, 0, 7, 7, 20], np.int32)
    yield "boundary", 8 * SIGMA + 17, 97, *boundary_pattern(8 * SIGMA + 17, np.int64)
    yield "empty", 17, 9, np.zeros(18, np.int32), np.zeros(0, np.int32)


@pytest.mark.parametrize("dt", DTYPES)
def test_block_matches_bspmv(ctx1, dt):
    """The custom_values arithmetic as snippets on a user 2 x 2 block type against the built-in block kernel (B = 2)."""
    vx = _vx()
    for name, n, m, ptr, col in patterns():
        rng = np.random.default_rng(n + m)
        blocks = rng.standard_normal((col.size, 2, 2)).astype(dt)
        x = rng.standard_normal(2 * m).astype(dt)
        y0 = rng.standard_normal(2 * n).astype(dt)
        U = usr(ctx1, n, m, ptr, col, blocks.reshape(-1, 4), usr_ops.block(dt))
        B = vx.BlockMatrix(ctx1, n, m, ptr, col, blocks)
        X = vx.vector(ctx1, x)
        for append in (False, True):
            Yu, Yb = vx.vector(ctx1, y0), vx.vector(ctx1, y0)
            U.apply(X, Yu, append)
            B.apply(X, Yb, 1.0, append)
            got, want = Yu.read(), Yb.read()
            assert same_bits(got.view(np.uint8), want.view(np.uint8)), f"{name} {append}: {np.count_nonzero(got != want)} differ"


@pytest.mark.parametrize("dt", DTYPES)
def test_complex_matches_zspmv(ctx1, dt):
    """The complex_spmv arithmetic as snippets on a user complex type against the built-in complex kernel."""
    vx = _vx()
    cdt = np.complex128 if dt == np.float64 else np.complex64
    for name, n, m, ptr, col in patterns():
        rng = np.random.default_rng(n + 3 * m)
        val = (rng.standard_normal(col.size) + 1j * rng.standard_normal(col.size)).astype(cdt)
        x = rng.standard_normal(2 * m).astype(dt)
        y0 = rng.standard_normal(2 * n).astype(dt)
        U = usr(ctx1, n, m, ptr, col, val.view(dt).reshape(-1, 2), usr_ops.complex_(dt))
        Z = vx.ComplexMatrix(ctx1, n, m, ptr, col, val)
        X = vx.vector(ctx1, x)
        for append in (False, True):
            Yu, Yz = vx.vector(ctx1, y0), vx.vector(ctx1, y0)
            U.apply(X, Yu, append)
            Z.apply(X, Yz, 1.0, append)
            got, want = Yu.read(), Yz.read()
            assert same_bits(got.view(np.uint8), want.view(np.uint8)), f"{name} {append}: {np.count_nonzero(got != want)} differ"


def triple_run(ctx, n, m, ptr, col, val, x, y0, append):
    vx = _vx()
    A = usr(ctx, n, m, ptr, col, val, usr_ops.TRIPLE)
    X, Y = vx.vector(ctx, x.ravel()), vx.vector(ctx, y0.ravel())
    A.apply(X, Y, append)
    return Y.read().reshape(-1, 3), A


@pytest.mark.parametrize("idx", [np.int32, np.int64])
@pytest.mark.parametrize("n", [1, 31, 32, 33, SIGMA - 1, SIGMA, SIGMA + 1, 8 * SIGMA + 17])
def test_triple_boundaries(ctx1, n, idx):
    m = 97
    ptr, col = boundary_pattern(n, idx, m)
    rng = np.random.default_rng(5 + n)
    val = rng.standard_normal((col.size, 3))
    x = rng.standard_normal((m, 3))
    y0 = rng.standard_normal((n, 3))
    for append in (False, True):
        got, _ = triple_run(ctx1, n, m, ptr, col, val, x, y0, append)
        want = usr_ops.triple_spmv(ptr, col, val, x, y0 if append else None)
        assert same_bits(got.view(np.uint64), want.view(np.uint64)), (append, np.count_nonzero(got != want))


def test_triple_random_and_empty(ctx1):
    for name, n, m, ptr, col in patterns():
        rng = np.random.default_rng(n)
        val = rng.standard_normal((col.size, 3))
        x = rng.standard_normal((m, 3))
        y0 = rng.standard_normal((n, 3))
        for append in (False, True):
            got, _ = triple_run(ctx1, n, m, ptr, col, val, x, y0, append)
            want = usr_ops.triple_spmv(ptr, col, val, x, y0 if append else None)
            assert same_bits(got.view(np.uint64), want.view(np.uint64)), (name, append)


@pytest.mark.parametrize("case", ["random", "empty"])
def test_no_writes_past_y(ctx1, case):
    vx = _vx()
    n, m = 1000, 800
    if case == "random":
        ptr, col = random_pattern(n, m, 5)
    else:
        ptr, col = np.zeros(n + 1, np.int32), np.zeros(0, np.int32)
    rng = np.random.default_rng(1)
    val, x = rng.standard_normal((col.size, 3)), rng.standard_normal((m, 3))
    tail = 333
    sentinel = np.full(3 * n + tail, 12345.5)
    A = usr(ctx1, n, m, ptr, col, val, usr_ops.TRIPLE)
    X, Y = vx.vector(ctx1, x.ravel()), vx.vector(ctx1, sentinel)
    from vexcl_b200 import _lib as L
    k = ctx1.local[0]
    for append in (True, False, True):
        L.check(L.lib().vexb_usr_spmv(ctx1.devs[k], ctx1.streams[k], A.h, C.byref(A.ops), X.bufs[k], Y.bufs[k], int(append)))
    got = Y.read()
    assert np.all(got[3 * n:] == 12345.5)
    want = sentinel[:3 * n].reshape(n, 3)
    for append in (True, False, True):
        want = usr_ops.triple_spmv(ptr, col, val, x, want if append else None)
    assert same_bits(got[:3 * n], want.ravel())


def test_info_matches_host_layout(ctx1):
    from vexcl_b200 import _lib as L
    for name, n, m, ptr, col in patterns():
        for ops, k, vb in ((usr_ops.TRIPLE, 3, 24), (usr_ops.block(np.float32), 4, 16)):
            val = np.zeros((col.size, k), np.float64 if vb == 24 else np.float32)
            A = usr(ctx1, n, m, ptr, col, val, ops)
            info = A.info()
            p = np.ascontiguousarray(ptr)
            ns, nsl = C.c_size_t(), C.c_size_t()
            L.check(L.lib().vexb_csr_sell_layout(n, p.ctypes.data, p.dtype.itemsize, SIGMA, C.byref(ns), C.byref(nsl), None, None))
            assert (info.nrows, info.ncols, info.nnz, info.val_bytes) == (n, m, col.size, vb), name
            assert (info.n_slices, info.n_slots) == (ns.value, nsl.value), name
            want = nsl.value * (vb + 4) + 32 * 4 * ns.value + 4 * (ns.value + 1)
            assert info.device_bytes == want, name
            assert (A.rows(), A.cols(), A.nonzeros()) == (n, m, col.size)


def test_nvrtc_error_carries_the_log(ctx1):
    vx = _vx()
    ptr, col = tridiagonal(64)
    bad = dict(usr_ops.TRIPLE, product="sum.x = sum.x + v.x * xv.q;")             # double3 has no member q
    A = usr(ctx1, 64, 64, ptr, col, np.ones((col.size, 3)), bad)
    X, Y = vx.vector(ctx1, np.ones(192)), vx.vector(ctx1, np.zeros(192))
    with pytest.raises(vx.VexbError) as e:
        A.apply(X, Y)
    assert "NVRTC" in str(e.value) and "has no member" in str(e.value) and "q" in str(e.value), str(e.value)


def test_empty_matrix_zeroes_or_keeps_y(ctx1):
    vx = _vx()
    A = usr(ctx1, 17, 9, np.zeros(18, np.int32), np.zeros(0, np.int32), np.zeros((0, 3)), usr_ops.TRIPLE)
    y0 = np.arange(51, dtype=np.float64) + 1
    Y = vx.vector(ctx1, y0)
    A.apply(vx.vector(ctx1, np.ones(27)), Y, append=True)
    assert same_bits(Y.read(), y0)
    A.apply(vx.vector(ctx1, np.ones(27)), Y)
    assert np.all(Y.read() == 0)


def test_two_part_context_is_refused(ctx2):
    ptr, col = tridiagonal(8)
    with pytest.raises(ValueError):
        usr(ctx2, 8, 8, ptr, col, np.ones((col.size, 3)), usr_ops.TRIPLE)


def test_cpp_sparse_user_values(built):
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = BIN / "test_sparse_user_values"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS="1"),
                       timeout=300)
    print(r.stdout[-3000:])
    print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"exit {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
