"""Hybrid ELL with row classes (spmv.ell_classes): a slot-mask strip whose rows take at most 256 distinct (slot mask,
slot values) tuples stores one class byte per row and a table of masks and values instead of the masks and the values.
Only the storage changes, so every reader of the strip must give the same bits as with slot masks.  By default the
encoding engages only above the L2 size; the tests force it at small sizes with spmv.ell_classes = 2."""
import ctypes as C

import numpy as np
import pytest

import oracle
import vexcl_b200 as vx
from vexcl_b200 import _lib as L
from vexcl_b200 import gen
from vexcl_b200.api import DeviceScalar

pytestmark = pytest.mark.gpu

STRUCTURED = [("poisson2d", lambda: oracle.poisson(2, 200)), ("poisson3d", lambda: oracle.poisson(3, 24)),
              ("tridiagonal", lambda: oracle.tridiagonal(5000))]


def spmat(ctx, n, row, col, val, classes, fmt=vx.FMT_HELL):
    vx.set_param("spmv.ell_classes", classes)              # read at construction
    try:
        return vx.SpMat(ctx, n, n, row, col, val, fmt)
    finally:
        vx.set_param("spmv.ell_classes", 1)


def check_product(ctx, row, col, val, classes):
    n = row.size - 1
    xh = oracle.uniform_real(11, n)
    A = spmat(ctx, n, row, col, val, classes)
    x, y = vx.vector(ctx, xh), vx.vector(ctx, n)
    y.assign(A * x)
    want = oracle.csr_spmv(row, col, val, xh)
    mag = oracle.csr_absrow(row, col, val, xh)
    if ctx.nparts == 1:
        assert np.array_equal(y.read(), want)
    else:
        assert np.all(np.abs(y.read() - want) <= 1e-10 * mag)
    y += 3.0 * (A * x)
    assert np.all(np.abs(y.read() - 4.0 * want) <= 1e-10 * 4 * mag)
    return A


@pytest.mark.parametrize("classes", [2, 0])
@pytest.mark.parametrize("nparts", [1, 2, 3])
@pytest.mark.parametrize("case", [name for name, _ in STRUCTURED])
def test_structured_strips_store_row_classes(ctx1, ctx2, ctx3, nparts, case, classes):
    ctx = {1: ctx1, 2: ctx2, 3: ctx3}[nparts]
    row, col, val = dict(STRUCTURED)[case]()
    A = check_product(ctx, row, col, val, classes)
    # Each part's interior strip (the rows dist_apply_kernel runs) with no column array -- the strips that qualify --
    # took the encoding asked for.  An interior that is row-compressed (its ghost-free rows are less than 80 % of the
    # part, e.g. the middle part of poisson3d in three) cannot drop its columns and has neither encoding.
    parts = [A.info(k).loc for k in A.parts]
    assert parts[0].fmt == vx.FMT_HELL and parts[0].ell_col_bytes == 0
    for k, loc in enumerate(parts):
        if loc.fmt == vx.FMT_HELL and loc.ell_col_bytes == 0:
            assert (loc.ell_classes > 0) == bool(classes), k
        else:
            assert loc.ell_classes == 0, k
    if nparts == 1:
        info = A.info().loc
        assert info.ell_col_bytes == 0
        if classes:
            # the oracle's matrices hold an interior row, boundary rows and the padding rows' empty class
            assert 2 <= info.ell_classes <= 256
            # one class byte per row, then the table: 256 mask bytes and W values per class
            assert info.device_bytes == info.ell_pitch + 256 + info.ell_classes * info.ell_width * 8
        else:
            assert info.ell_classes == 0
            assert info.device_bytes == info.ell_pitch * info.ell_width * 8 + info.ell_pitch


def test_small_strips_keep_slot_masks_by_default(ctx1):
    row, col, val = oracle.poisson(2, 200)
    n = row.size - 1
    info = vx.SpMat(ctx1, n, n, row, col, val, vx.FMT_HELL).info().loc
    assert info.ell_col_bytes == 0 and info.ell_classes == 0


def with_long_rows(row, col, val, long_rows, reach):
    """The matrix with two more entries, `reach` and `reach` + 3 to the right of the diagonal, in each of `long_rows`
    (interior rows, so their first entries keep the stencil's distances): a few rows wider than the ELL width."""
    n = row.size - 1
    r2, c2, v2 = [0], [], []
    for i in range(n):
        c2.extend(col[row[i]:row[i + 1]].tolist()); v2.extend(val[row[i]:row[i + 1]].tolist())
        if i in long_rows:
            c2.extend([i + reach, i + reach + 3]); v2.extend([0.5, -0.25])
        r2.append(len(c2))
    return np.array(r2, np.int64), np.array(c2, np.int64), np.array(v2, np.float64)


@pytest.mark.parametrize("nparts", [1, 2])
def test_row_classes_with_a_csr_tail(ctx1, ctx2, nparts):
    """Rows wider than the ELL width put their last entries in the CSR tail: the tail loop of the class row body (in
    hell_kernel, including the repeated last row of its two rows per thread, and in dist_apply_kernel) and of the
    generated row function."""
    ctx = {1: ctx1, 2: ctx2}[nparts]
    row, col, val = with_long_rows(*oracle.poisson(2, 100), long_rows={4321, 5050, 9750}, reach=150)
    n = row.size - 1
    A = check_product(ctx, row, col, val, 2)
    for k in A.parts:
        assert A.info(k).loc.ell_classes > 0, k
    if nparts == 1:
        info = A.info().loc
        assert info.ell_width == 5 and info.csr_tail_nnz == 6 and n % 512 != 0
        X = oracle.uniform_real(3, n)
        x, y = vx.vector(ctx, X), vx.vector(ctx, n)
        n0 = vx.launch_count()
        y.assign(x + A * x)
        assert vx.launch_count() - n0 == 1
        assert np.array_equal(y.read(), X + oracle.csr_spmv(row, col, val, X))


@pytest.mark.parametrize("nparts", [1, 2])
def test_many_distinct_rows_keep_slot_masks(ctx1, ctx2, nparts):
    """Random values on a Poisson pattern: far more than 256 distinct rows, so the strip keeps its slot masks."""
    ctx = {1: ctx1, 2: ctx2}[nparts]
    row, col, _ = oracle.poisson(2, 100)
    val = np.random.default_rng(7).random(col.size) - 0.5
    A = check_product(ctx, row, col, val, 2)
    if nparts == 1:
        info = A.info().loc
        assert info.ell_col_bytes == 0 and info.ell_classes == 0


def test_multivector_product_on_row_classes(ctx1):
    row, col, val = oracle.poisson(2, 150)
    n = row.size - 1
    A = spmat(ctx1, n, row, col, val, 2)
    assert A.info().loc.ell_classes > 0
    X = [oracle.uniform_real(20 + r, n) for r in range(4)]
    for k in (4, 3, 2):
        xs = [vx.vector(ctx1, h) for h in X[:k]]
        ys = [vx.vector(ctx1, n) for _ in range(k)]
        A.apply_multi(xs, ys, 1.0, False)
        for r in range(k):
            assert np.array_equal(ys[r].read(), oracle.csr_spmv(row, col, val, X[r]))
        A.apply_multi(xs, ys, -0.5, True)
        for r in range(k):
            want = oracle.csr_spmv(row, col, val, X[r])
            assert np.all(np.abs(ys[r].read() - 0.5 * want) <= 1e-10 * oracle.csr_absrow(row, col, val, X[r]))


def test_inlined_product_on_row_classes(ctx1):
    """y = x + A*x as one generated kernel reading the class table; a slot-mask strip of the same shape needs a kernel
    of its own (the encoding is part of the kernel cache key)."""
    row, col, val = oracle.poisson(3, 20)
    n = row.size - 1
    X = oracle.uniform_real(3, n)
    ax = oracle.csr_spmv(row, col, val, X)
    x, y = vx.vector(ctx1, X), vx.vector(ctx1, n)
    for classes in (2, 0, 2):
        A = spmat(ctx1, n, row, col, val, classes)
        assert (A.info().loc.ell_classes > 0) == bool(classes)
        y.assign(0.0)
        n0 = vx.launch_count()
        y.assign(x + A * x)
        assert vx.launch_count() - n0 == 1
        assert np.array_equal(y.read(), X + ax)


def test_fused_cg_on_row_classes(ctx1):
    """The product + dot kernel (dist_apply_kernel with the dot epilogue) and CGFused on a 3-D SPD strip."""
    from vexcl_b200.solvers import CGFused
    nx = 18
    row, col, val = gen.poisson_strip(3, nx, spd=True)
    N = nx ** 3
    A = spmat(ctx1, N, row, col, val, 2)
    info = A.info().loc
    assert info.ell_width == 7 and 0 < info.ell_classes <= 256
    X, W = oracle.uniform_real(4, N), oracle.uniform_real(5, N)
    x, w, y, y2 = vx.vector(ctx1, X), vx.vector(ctx1, W), vx.vector(ctx1, N), vx.vector(ctx1, N)
    d = DeviceScalar(ctx1)
    assert A.apply_dot(x, y, d, dot_with=w)
    A.apply(x, y2)
    got = y.read()
    assert np.array_equal(got, y2.read()) and np.array_equal(got, oracle.csr_spmv(row, col, val, X))
    assert abs(d.get() - float(np.dot(W, got))) <= 1e-10 * np.sum(np.abs(W * got))
    b = oracle.uniform_real(3, N)
    iters = 20
    xo, hist_o = oracle.cg(row, col, val, b, np.zeros(N), iters)
    bv, xv = vx.vector(ctx1, b), vx.vector(ctx1, N)
    xv.assign(0.0)
    cg = CGFused(A, bv, xv)
    hist = []
    for _ in range(iters):
        cg.run(1)
        hist.append(cg.residual2())
    ctx1.finish()
    assert cg.fused_product
    assert np.allclose(hist, hist_o, rtol=1e-8)
    assert np.allclose(xv.read(), xo, rtol=1e-8, atol=1e-12)


def test_row_class_download_matches_reference_packing(ctx1):
    row, col, val = oracle.poisson(2, 60)
    n = row.size - 1
    want = oracle.hell_pack(row, col, val)
    h = C.c_void_p()
    lib = L.lib()
    vx.set_param("spmv.ell_classes", 2)
    try:
        L.check(lib.vexb_csr_create(0, ctx1.streams[0], n, n, row.ctypes.data, 8, col.ctypes.data, 8, val.ctypes.data,
                                    L.F64, L.FMT_HELL, C.byref(h)))
    finally:
        vx.set_param("spmv.ell_classes", 1)
    try:
        info = L.SpmatInfo()
        L.check(lib.vexb_spmat_get_info(h, C.byref(info)))
        assert info.ell_col_bytes == 0 and info.ell_classes > 0
        assert (info.ell_width, info.ell_pitch, info.csr_tail_nnz) == (want["width"], want["pitch"], want["csr_col"].size)
        ec = np.empty(info.ell_pitch * info.ell_width, np.int32)
        ev = np.empty(info.ell_pitch * info.ell_width)
        tp = np.empty(n + 1, np.int64)
        L.check(lib.vexb_spmat_hell_download(h, ec.ctypes.data, ev.ctypes.data, tp.ctypes.data, None, None))
        assert np.array_equal(ec, want["ell_col"].astype(np.int32)) and np.array_equal(ev, want["ell_val"])
        assert np.array_equal(tp, want["csr_row"])
    finally:
        L.check(lib.vexb_spmat_destroy(h))


def test_single_precision_row_classes(ctx1):
    row, col, val = oracle.poisson(2, 120)
    n = row.size - 1
    val32 = val.astype(np.float32)
    X = oracle.uniform_real(24, n).astype(np.float32)
    got = {}
    for classes in (2, 0):
        A = spmat(ctx1, n, row, col, val32, classes)
        info = A.info().loc
        assert info.ell_col_bytes == 0 and (info.ell_classes > 0) == bool(classes)
        if classes:
            assert info.device_bytes == info.ell_pitch + 256 + info.ell_classes * info.ell_width * 4
        x, y = vx.vector(ctx1, X), vx.vector(ctx1, n, np.float32)
        y.assign(A * x)
        got[classes] = y.read()
    assert np.array_equal(got[2], got[0])
    ref = oracle.csr_spmv(row, col, val32.astype(np.float64), X.astype(np.float64))
    assert np.all(np.abs(got[2] - ref) <= 2e-6 * oracle.csr_absrow(row, col, val32.astype(np.float64), X.astype(np.float64)))
