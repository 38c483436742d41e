"""Block sparse products on the GPU (vexb_bspmv, bsell_kernel): bit-identical to tests/block_oracle.py for B = 2, 3, 4
in float64 and float32 with `=`, `+=`, `-=` and alpha = 0.5 with append, on the reference's custom_values matrix,
random widths, a block 7-point stencil, a rectangular matrix, one block row and no block at all; at the slice and
sorting-window boundaries with widths 0 to 40 and 32- and 64-bit indices; nothing written past y; info() against the
host layout; and the C++ front-end test tests/cpp/test_sparse_blocks.cpp."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle
from block_oracle import bsr_spmv, block_stencil

pytestmark = pytest.mark.gpu
BIN = Path(__file__).resolve().parent / "cpp" / "bin"
BLOCKS = (2, 3, 4)
DTYPES = (np.float64, np.float32)
SIGMA = 1024                                   # spmv.sell_sigma default: the sorting window of the layout
OPS = {"set": (1.0, False), "add": (1.0, True), "sub": (-1.0, True), "half_append": (0.5, True)}


def _vx():
    import vexcl_b200 as vx
    return vx


def custom_values(n, B, dtype):
    ptr, col, val = [0], [], []
    for i in range(n):
        if i > 0:
            col.append(i - 1); val.append(np.full((B, B), -1, dtype))
        col.append(i); val.append(np.full((B, B), 2, dtype))
        if i + 1 < n:
            col.append(i + 1); val.append(np.full((B, B), -1, dtype))
        ptr.append(len(col))
    return n, n, np.array(ptr, np.int32), np.array(col, np.int32), np.array(val, dtype)


def random_widths(n, m, B, dtype, seed):
    row, col, _ = oracle.random_matrix(n, m, 32, seed)                # widths U[0, 32), sorted unique columns
    rng = np.random.default_rng(seed)
    return n, m, row, col, rng.standard_normal((col.size, B, B)).astype(dtype)


def rectangular(B, dtype):
    n, m = 300, 451
    rng = np.random.default_rng(7)
    ptr, col = [0], []
    for i in range(n):
        w = int(rng.integers(0, 9))
        cs = list(rng.integers(0, m, size=w))
        if i % 50 == 3:
            cs.append(m - 1)                                           # touches the last block column
        col += cs
        ptr.append(len(col))
    return n, m, np.array(ptr, np.int64), np.array(col, np.int64), rng.standard_normal((len(col), B, B)).astype(dtype)


def matrices(B, dtype):
    yield "custom_values", custom_values(1024, B, dtype)
    yield "random", random_widths(3000, 2500, B, dtype, 11 + B)
    ptr, col, val = block_stencil(32, B, dtype, seed=B)
    yield "stencil32", (32 ** 3, 32 ** 3, ptr, col, val)
    yield "rectangular", rectangular(B, dtype)
    rng = np.random.default_rng(3)
    yield "one_row", (1, 40, np.array([0, 5], np.int32), np.array([39, 0, 7, 7, 20], np.int32),
                      rng.standard_normal((5, B, B)).astype(dtype))
    yield "empty", (17, 9, np.zeros(18, np.int32), np.zeros(0, np.int32), np.zeros((0, B, B), dtype))


def run(ctx, n, m, ptr, col, val, x, y0, alpha, append):
    vx = _vx()
    A = vx.BlockMatrix(ctx, n, m, ptr, col, val)
    X, Y = vx.vector(ctx, x), vx.vector(ctx, y0)
    A.apply(X, Y, alpha, append)
    return Y.read(), A


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", BLOCKS)
def test_parity(ctx1, B, dtype, op):
    alpha, append = OPS[op]
    for name, (n, m, ptr, col, val) in matrices(B, dtype):
        rng = np.random.default_rng(n + m)
        x = rng.standard_normal(m * B).astype(dtype)
        y0 = rng.standard_normal(n * B).astype(dtype)
        got, _ = run(ctx1, n, m, ptr, col, val, x, y0, alpha, append)
        want = bsr_spmv(ptr, col, val, x, y0 if append else None, alpha, append)
        assert same_bits(got, want), f"{name}: {np.count_nonzero(got != want)} of {got.size} differ"


def boundary_matrix(n, B, dtype, idx):
    """Block row i has width (7 i) mod 41: every width 0..40 appears, so both the batched slot loop and its remainder run."""
    w = (7 * np.arange(n)) % 41
    ptr = np.zeros(n + 1, np.int64); ptr[1:] = np.cumsum(w)
    m = 97
    rng = np.random.default_rng(n * B)
    col = rng.integers(0, m, size=int(ptr[-1]))
    val = rng.standard_normal((col.size, B, B)).astype(dtype)
    return m, ptr.astype(idx), col.astype(idx), val


@pytest.mark.parametrize("idx", [np.int32, np.int64])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", BLOCKS)
@pytest.mark.parametrize("n", [1, 31, 32, 33, SIGMA - 1, SIGMA, SIGMA + 1, 8 * SIGMA + 17])
def test_boundaries(ctx1, n, B, dtype, idx):
    m, ptr, col, val = boundary_matrix(n, B, dtype, idx)
    rng = np.random.default_rng(5)
    x = rng.standard_normal(m * B).astype(dtype)
    y0 = rng.standard_normal(n * B).astype(dtype)
    for alpha, append in OPS.values():
        got, _ = run(ctx1, n, m, ptr, col, val, x, y0, alpha, append)
        assert same_bits(got, bsr_spmv(ptr, col, val, x, y0 if append else None, alpha, append)), (alpha, append)


@pytest.mark.parametrize("case", ["random", "empty"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", BLOCKS)
def test_no_writes_past_y(ctx1, B, dtype, case):
    vx = _vx()
    from vexcl_b200 import _lib as L
    if case == "random":
        n, m, ptr, col, val = random_widths(1000, 800, B, dtype, 5)
    else:
        n, m, ptr, col, val = 1000, 800, np.zeros(1001, np.int32), np.zeros(0, np.int32), np.zeros((0, B, B), dtype)
    tail = 333
    x = np.random.default_rng(1).standard_normal(m * B).astype(dtype)
    sentinel = np.full(n * B + tail, 12345.5, dtype)
    A = vx.BlockMatrix(ctx1, n, m, ptr, col, val)
    X, Y = vx.vector(ctx1, x), vx.vector(ctx1, sentinel)
    k = ctx1.local[0]
    for alpha, append in OPS.values():
        L.check(L.lib().vexb_bspmv(ctx1.devs[k], ctx1.streams[k], A.h, X.bufs[k], Y.bufs[k], alpha, int(append)))
    got = Y.read()
    assert np.all(got[n * B:] == 12345.5)
    want = sentinel[:n * B]
    for alpha, append in OPS.values():
        want = bsr_spmv(ptr, col, val, x, want if append else None, alpha, append)
    assert same_bits(got[:n * B], want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B", BLOCKS)
def test_info_matches_host_layout(ctx1, B, dtype):
    from vexcl_b200 import _lib as L
    for name, (n, m, ptr, col, val) in matrices(B, dtype):
        _, A = run(ctx1, n, m, ptr, col, val, np.zeros(m * B, dtype), np.zeros(n * B, dtype), 1.0, False)
        info = A.info()
        p = np.ascontiguousarray(ptr)
        ns, nsl = C.c_size_t(), C.c_size_t()
        L.check(L.lib().vexb_csr_sell_layout(n, p.ctypes.data, p.dtype.itemsize, SIGMA, C.byref(ns), C.byref(nsl), None, None))
        assert (info.nrows, info.ncols, info.nnzb, info.block) == (n, m, val.shape[0], B), name
        assert info.val_dtype == (L.F64 if dtype == np.float64 else L.F32)
        assert (info.n_slices, info.n_slots) == (ns.value, nsl.value), name
        es = np.dtype(dtype).itemsize
        want = nsl.value * (B * B * es + 4) + ns.value * 32 * 4 + (ns.value + 1) * 4
        assert info.device_bytes == want, name
        assert (A.rows(), A.cols(), A.nonzeros()) == (n, m, val.shape[0])


def test_two_part_context_is_refused(ctx2):
    vx = _vx()
    n, m, ptr, col, val = custom_values(8, 2, np.float64)
    with pytest.raises(ValueError):
        vx.BlockMatrix(ctx2, n, m, ptr, col, val)


@pytest.mark.parametrize("parts", ["2", "1"])
def test_cpp_sparse_blocks(built, parts):
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = BIN / "test_sparse_blocks"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts),
                       timeout=300)
    print(r.stdout[-3000:])
    print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"exit {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
