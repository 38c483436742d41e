"""Complex sparse products on the GPU (vexb_zspmv, zsell_kernel): bit-identical to tests/complex_oracle.py in float64 and
float32 with `=`, `+=`, `-=` and alpha = 0.5 with append, on the diagonal of the reference's examples/complex_spmv.cpp, a
complex tridiagonal, random widths, a complex 7-point stencil, a rectangular matrix, one row and no entry at all; at the
slice and sorting-window boundaries with widths 0 to 40 and 32- and 64-bit indices; bit-identical to vexb_bspmv on the
[[a, -b], [b, a]] expansion of the same matrix; nothing written past y; info() against the host layout; and the C++
front-end test tests/cpp/test_sparse_complex.cpp."""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle
from complex_oracle import as_blocks, complex_stencil, zsr_spmv

pytestmark = pytest.mark.gpu
BIN = Path(__file__).resolve().parent / "cpp" / "bin"
CDTYPES = (np.complex128, np.complex64)
REAL = {np.complex128: np.float64, np.complex64: np.float32}
SIGMA = 1024                                   # spmv.sell_sigma default: the sorting window of the layout
OPS = {"set": (1.0, False), "add": (1.0, True), "sub": (-1.0, True), "half_append": (0.5, True)}


def _vx():
    import vexcl_b200 as vx
    return vx


def cvals(rng, size, cdtype):
    return (rng.standard_normal(size) + 1j * rng.standard_normal(size)).astype(cdtype)


def example_diagonal(n, cdtype):
    k = np.arange(n)
    return n, n, np.arange(n + 1, dtype=np.int32), k.astype(np.int32), ((k + 1) * (1 + 1j)).astype(cdtype)


def tridiagonal(n, cdtype):
    """The custom_values pattern with complex values: -1 + i/2, 2 - i, -1 + i/2."""
    ptr, col, val = [0], [], []
    for i in range(n):
        if i > 0:
            col.append(i - 1); val.append(-1 + 0.5j)
        col.append(i); val.append(2 - 1j)
        if i + 1 < n:
            col.append(i + 1); val.append(-1 + 0.5j)
        ptr.append(len(col))
    return n, n, np.array(ptr, np.int32), np.array(col, np.int32), np.array(val, cdtype)


def random_widths(n, m, cdtype, seed):
    row, col, _ = oracle.random_matrix(n, m, 32, seed)                # widths U[0, 32), sorted unique columns
    return n, m, row, col, cvals(np.random.default_rng(seed), col.size, cdtype)


def rectangular(cdtype):
    n, m = 300, 451
    rng = np.random.default_rng(7)
    ptr, col = [0], []
    for i in range(n):
        w = int(rng.integers(0, 9))
        cs = list(rng.integers(0, m, size=w))
        if i % 50 == 3:
            cs.append(m - 1)                                           # touches the last column
        col += cs
        ptr.append(len(col))
    return n, m, np.array(ptr, np.int64), np.array(col, np.int64), cvals(rng, len(col), cdtype)


def matrices(cdtype):
    yield "example", example_diagonal(4, cdtype)
    yield "tridiagonal", tridiagonal(1024, cdtype)
    yield "random", random_widths(3000, 2500, cdtype, 13)
    ptr, col, val = complex_stencil(32, cdtype, seed=2)
    yield "stencil32", (32 ** 3, 32 ** 3, ptr, col, val)
    yield "rectangular", rectangular(cdtype)
    yield "one_row", (1, 40, np.array([0, 5], np.int32), np.array([39, 0, 7, 7, 20], np.int32),
                      cvals(np.random.default_rng(3), 5, cdtype))
    yield "empty", (17, 9, np.zeros(18, np.int32), np.zeros(0, np.int32), np.zeros(0, cdtype))


def run(ctx, n, m, ptr, col, val, x, y0, alpha, append):
    vx = _vx()
    A = vx.ComplexMatrix(ctx, n, m, ptr, col, val)
    X, Y = vx.vector(ctx, x), vx.vector(ctx, y0)
    A.apply(X, Y, alpha, append)
    return Y.read(), A


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("cdtype", CDTYPES)
def test_parity(ctx1, cdtype, op):
    alpha, append = OPS[op]
    dt = REAL[cdtype]
    for name, (n, m, ptr, col, val) in matrices(cdtype):
        rng = np.random.default_rng(n + m)
        x = rng.standard_normal(2 * m).astype(dt)
        y0 = rng.standard_normal(2 * n).astype(dt)
        got, _ = run(ctx1, n, m, ptr, col, val, x, y0, alpha, append)
        want = zsr_spmv(ptr, col, val, x, y0 if append else None, alpha, append)
        assert same_bits(got, want), f"{name}: {np.count_nonzero(got != want)} of {got.size} differ"


@pytest.mark.parametrize("cdtype", CDTYPES)
def test_example_closed_form(ctx1, cdtype):
    """examples/complex_spmv.cpp: (k+1)(1+i) times 1+i is 0 + 2(k+1)i, exactly."""
    n, m, ptr, col, val = example_diagonal(4, cdtype)
    x = np.ones(2 * m, REAL[cdtype])
    got, _ = run(ctx1, n, m, ptr, col, val, x, np.zeros(2 * n, REAL[cdtype]), 1.0, False)
    assert np.array_equal(got.view(cdtype), np.array([2j, 4j, 6j, 8j], cdtype))


def boundary_matrix(n, cdtype, idx):
    """Row i has width (7 i) mod 41: every width 0..40 appears, so both the batched slot loop and its remainder run."""
    w = (7 * np.arange(n)) % 41
    ptr = np.zeros(n + 1, np.int64); ptr[1:] = np.cumsum(w)
    m = 97
    rng = np.random.default_rng(n)
    col = rng.integers(0, m, size=int(ptr[-1]))
    return m, ptr.astype(idx), col.astype(idx), cvals(rng, col.size, cdtype)


@pytest.mark.parametrize("idx", [np.int32, np.int64])
@pytest.mark.parametrize("cdtype", CDTYPES)
@pytest.mark.parametrize("n", [1, 31, 32, 33, SIGMA - 1, SIGMA, SIGMA + 1, 8 * SIGMA + 17])
def test_boundaries(ctx1, n, cdtype, idx):
    m, ptr, col, val = boundary_matrix(n, cdtype, idx)
    dt = REAL[cdtype]
    rng = np.random.default_rng(5)
    x = rng.standard_normal(2 * m).astype(dt)
    y0 = rng.standard_normal(2 * n).astype(dt)
    for alpha, append in OPS.values():
        got, _ = run(ctx1, n, m, ptr, col, val, x, y0, alpha, append)
        assert same_bits(got, zsr_spmv(ptr, col, val, x, y0 if append else None, alpha, append)), (alpha, append)


@pytest.mark.parametrize("cdtype", CDTYPES)
def test_matches_block_product(ctx1, cdtype):
    """vexb_zspmv against vexb_bspmv on the 2x2 expansion of the same matrix: two kernels, the same bits."""
    vx = _vx()
    dt = REAL[cdtype]
    for name, (n, m, ptr, col, val) in list(matrices(cdtype)) + [("boundary", (8 * SIGMA + 17,) + boundary_matrix(8 * SIGMA + 17, cdtype, np.int32))]:
        rng = np.random.default_rng(n + 2 * m)
        x = rng.standard_normal(2 * m).astype(dt)
        y0 = rng.standard_normal(2 * n).astype(dt)
        Z = vx.ComplexMatrix(ctx1, n, m, ptr, col, val)
        Bm = vx.BlockMatrix(ctx1, n, m, ptr, col, as_blocks(val))
        X = vx.vector(ctx1, x)
        for alpha, append in OPS.values():
            Yz, Yb = vx.vector(ctx1, y0), vx.vector(ctx1, y0)
            Z.apply(X, Yz, alpha, append)
            Bm.apply(X, Yb, alpha, append)
            got, want = Yz.read(), Yb.read()
            assert same_bits(got, want), f"{name} {alpha} {append}: {np.count_nonzero(got != want)} of {got.size} differ"


@pytest.mark.parametrize("case", ["random", "empty"])
@pytest.mark.parametrize("cdtype", CDTYPES)
def test_no_writes_past_y(ctx1, cdtype, case):
    vx = _vx()
    from vexcl_b200 import _lib as L
    dt = REAL[cdtype]
    if case == "random":
        n, m, ptr, col, val = random_widths(1000, 800, cdtype, 5)
    else:
        n, m, ptr, col, val = 1000, 800, np.zeros(1001, np.int32), np.zeros(0, np.int32), np.zeros(0, cdtype)
    tail = 333
    x = np.random.default_rng(1).standard_normal(2 * m).astype(dt)
    sentinel = np.full(2 * n + tail, 12345.5, dt)
    A = vx.ComplexMatrix(ctx1, n, m, ptr, col, val)
    X, Y = vx.vector(ctx1, x), vx.vector(ctx1, sentinel)
    k = ctx1.local[0]
    for alpha, append in OPS.values():
        L.check(L.lib().vexb_zspmv(ctx1.devs[k], ctx1.streams[k], A.h, X.bufs[k], Y.bufs[k], alpha, int(append)))
    got = Y.read()
    assert np.all(got[2 * n:] == 12345.5)
    want = sentinel[:2 * n]
    for alpha, append in OPS.values():
        want = zsr_spmv(ptr, col, val, x, want if append else None, alpha, append)
    assert same_bits(got[:2 * n], want)


@pytest.mark.parametrize("cdtype", CDTYPES)
def test_misaligned_x_is_refused(ctx1, cdtype):
    """x must hold whole complex elements: a pointer half an element in is refused before any launch."""
    vx = _vx()
    from vexcl_b200 import _lib as L
    n, m, ptr, col, val = tridiagonal(64, cdtype)
    dt = REAL[cdtype]
    A = vx.ComplexMatrix(ctx1, n, m, ptr, col, val)
    X, Y = vx.vector(ctx1, np.zeros(2 * m + 2, dt)), vx.vector(ctx1, np.zeros(2 * n, dt))
    k = ctx1.local[0]
    half = C.c_void_p(X.bufs[k].value + np.dtype(dt).itemsize)
    assert L.lib().vexb_zspmv(ctx1.devs[k], ctx1.streams[k], A.h, half, Y.bufs[k], 1.0, 0) == L.ERR_INVALID


@pytest.mark.parametrize("cdtype", CDTYPES)
def test_info_matches_host_layout(ctx1, cdtype):
    from vexcl_b200 import _lib as L
    dt = REAL[cdtype]
    for name, (n, m, ptr, col, val) in matrices(cdtype):
        _, A = run(ctx1, n, m, ptr, col, val, np.zeros(2 * m, dt), np.zeros(2 * n, dt), 1.0, False)
        info = A.info()
        p = np.ascontiguousarray(ptr)
        ns, nsl = C.c_size_t(), C.c_size_t()
        L.check(L.lib().vexb_csr_sell_layout(n, p.ctypes.data, p.dtype.itemsize, SIGMA, C.byref(ns), C.byref(nsl), None, None))
        assert (info.nrows, info.ncols, info.nnz) == (n, m, val.size), name
        assert info.val_dtype == (L.F64 if cdtype == np.complex128 else L.F32)
        assert (info.n_slices, info.n_slots) == (ns.value, nsl.value), name
        es = np.dtype(dt).itemsize
        want = nsl.value * (2 * es + 4) + ns.value * 32 * 4 + (ns.value + 1) * 4
        assert info.device_bytes == want, name
        assert (A.rows(), A.cols(), A.nonzeros()) == (n, m, val.size)


def test_two_part_context_is_refused(ctx2):
    vx = _vx()
    n, m, ptr, col, val = tridiagonal(8, np.complex128)
    with pytest.raises(ValueError):
        vx.ComplexMatrix(ctx2, n, m, ptr, col, val)


@pytest.mark.parametrize("parts", ["2", "1"])
def test_cpp_sparse_complex(built, parts):
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = BIN / "test_sparse_complex"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts),
                       timeout=300)
    print(r.stdout[-3000:])
    print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"exit {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
