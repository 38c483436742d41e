"""Hybrid ELL at the edges of its encodings, widths, shapes and lengths.

Every strip here is a band (row i holds entries at columns i + offset) built in this file, multiplied through every reader
of a hybrid-ELL strip -- hell_kernel (y = A*x, y += a*A*x), hell_multi_kernel (apply_multi, 1 to 6 right-hand sides),
the generated row function of an inlined product (y = z + A*x, one launch) and dist_apply_kernel (apply_dot) -- in each
of the four encodings: row classes (spmv.ell_classes = 2), slot masks (spmv.ell_classes = 0), 16-bit columns
(spmv.ell_diag = 0) and 32-bit columns (spmv.col16 = 0).

On one part every reader adds a row's products in storage order with separately rounded multiplies and adds, so y must
equal `ell_ref` bit for bit, in float64 and in float32.  Over 2 and 3 parts the local and ghost entries are added
separately; y is then checked within 2 (w + 2) u |A| |x| per row (u the unit round-off, w the row length), a bound
on two orderings of the same sum.

The shapes aim at the kernels' edges: widths 1 to 10 and 27 (the unrolled widths 3, 5, 7, 9 against the run-time width
loop), row counts around the 256-row blocks, the 512-row blocks of the class kernel and the row where its L2 prefetch
(132 blocks ahead) starts to issue, one-sided and rectangular bands (the clamp of padding gathers to x_max), strips with
255, 256 and 257 row classes, and a 16-bit column span of exactly 65 534."""
import numpy as np
import pytest

import oracle
import vexcl_b200 as vx
from vexcl_b200.api import DeviceScalar, Scalar

# ------------------------------------------------------------------------------------------------ generators

def band(n, m, offsets, values):
    """CSR of a constant-coefficient band: row i holds values[k] at column i + offsets[k] where that column lies in
    [0, m).  Columns are sorted.  The values keep their dtype."""
    return band_rows(n, m, offsets, np.asarray(values)[None, :])


def band_rows(n, m, offsets, tuples):
    """The band of `offsets`, with row i taking its values from tuples[i mod K] (tuples: K x len(offsets))."""
    offsets = np.asarray(offsets, np.int64)
    tuples = np.asarray(tuples)
    order = np.argsort(offsets, kind="stable")
    offsets, tuples = offsets[order], tuples[:, order]
    cols = np.arange(n, dtype=np.int64)[:, None] + offsets[None, :]
    inside = (cols >= 0) & (cols < m)
    row = np.zeros(n + 1, np.int64)
    np.cumsum(inside.sum(axis=1), out=row[1:])
    vals = tuples[np.arange(n) % tuples.shape[0]]
    return row, cols[inside], np.ascontiguousarray(vals[inside])


def with_long_rows(row, col, val, long_rows, reach=50):
    """The matrix with two more entries, `reach` and `reach` + 3 right of the diagonal, in each of `long_rows`: rows
    wider than the ELL width, whose last entries go to the CSR tail."""
    r2, c2, v2 = [0], [], []
    for i in range(row.size - 1):
        c2 += list(col[row[i]:row[i + 1]]); v2 += list(val[row[i]:row[i + 1]])
        if i in long_rows:
            c2 += [i + reach, i + reach + 3]; v2 += [0.75, -0.375]
        r2.append(len(c2))
    return np.array(r2, np.int64), np.array(c2, np.int64), np.array(v2, val.dtype)


def ell_width(row):
    return oracle.hell_width(np.diff(row))


def _slots(dist, w, ref):
    """ELL slots build() gives a row with distances `dist` (column - row) from the diagonal: rows shorter than the
    width are aligned on the distances of the first full row (`ref`), other rows fill slots 0, 1, ... (entries past
    the width go to the CSR tail and get no slot)."""
    cnt = len(dist)
    if ref is None or cnt == 0 or cnt >= w:
        return list(range(min(cnt, w)))
    out, s0 = [], 0
    for q, d in enumerate(dist):
        last = w - (cnt - q)
        t = next((c for c in range(s0, last + 1) if ref[c] == d), None)
        if t is None:
            t = next((c for c in range(s0, last + 1) if abs(ref[c] - d) <= 16384), s0)
        out.append(t)
        s0 = t + 1
    return out


def row_class_ids(row, col, val):
    """Class of every stored row (pitch = n rounded up to 16, padding rows included) as build() numbers them: distinct
    (slot mask, W slot values) tuples in order of first appearance, values compared bit for bit."""
    n = row.size - 1
    w = ell_width(row)
    pitch = (n + 15) // 16 * 16
    ref = None
    for i in range(n):
        if w > 0 and row[i + 1] - row[i] >= w:
            ref = [int(c) - i for c in col[row[i]:row[i] + w]]
            break
    zero = np.zeros(1, val.dtype).tobytes()
    seen, ids = {}, np.empty(pitch, np.int64)
    for i in range(pitch):
        mask, slot_vals = 0, [zero] * w
        if i < n:
            a, b = int(row[i]), int(row[i + 1])
            for k, j in enumerate(_slots([int(c) - i for c in col[a:b]], w, ref)):
                mask |= 1 << j
                slot_vals[j] = val[a + k].tobytes()
        ids[i] = seen.setdefault((mask, b"".join(slot_vals)), len(seen))
    return ids


def classes_expected(row, col, val):
    """Number of row classes build() finds on the strip (padding rows and empty rows share the empty class)."""
    return int(row_class_ids(row, col, val).max()) + 1


def ell_ref(row, col, val, x, dtype):
    """y = A*x accumulated in storage order -- the ELL slots in order, then the entries past the ELL width, which is
    the order of the row in CSR -- slot by slot, vectorised over rows, every product and sum rounded in `dtype`:
    s = dtype(s + dtype(v * x)).  numpy rounds each operation to nearest and never fuses, so this is a bit-exact
    reference for every reader on one part."""
    dtype = np.dtype(dtype).type
    n = row.size - 1
    val, x = val.astype(dtype), x.astype(dtype)
    cnt = np.diff(row)
    s = np.zeros(n, dtype)
    for k in range(int(cnt.max()) if n else 0):
        r = np.nonzero(cnt > k)[0]
        j = row[r] + k
        s[r] = (s[r] + (val[j] * x[col[j]]).astype(dtype)).astype(dtype)
    return s


def axpy_ref(y, alpha, s, dtype):
    """y + alpha * s, each operation rounded in dtype (y += alpha*A*x on the device)."""
    dtype = np.dtype(dtype).type
    return (y.astype(dtype) + (dtype(alpha) * s.astype(dtype)).astype(dtype)).astype(dtype)


# ------------------------------------------------------------------------------------------------ CPU self-checks

def test_band_matches_reference_packing():
    """band() against the reference packing: width, pitch, and row i's slots hold column i + offset."""
    offsets = (-3, -1, 0, 2, 7)
    n, m = 61, 64
    vals = np.array([1.5, -2.0, 4.0, 0.25, -0.5])
    row, col, val = band(n, m, offsets, vals)
    want_nnz = sum(1 for i in range(n) for d in offsets if 0 <= i + d < m)
    assert row[-1] == want_nnz and np.all(np.diff(row) <= len(offsets))
    h = oracle.hell_pack(row, col, val)
    assert (h["width"], h["pitch"], h["csr_col"].size) == (5, 64, 0)
    for i in range(3, 57):                                   # full rows: slot k holds offset k
        assert [h["ell_col"][i + h["pitch"] * k] - i for k in range(5)] == list(offsets)
        assert [h["ell_val"][i + h["pitch"] * k] for k in range(5)] == list(vals)
    for i in range(n):
        assert np.all(np.diff(col[row[i]:row[i + 1]]) > 0)
    # band_rows: the values of row i come from tuple i mod K, in the order of the sorted offsets
    row2, col2, val2 = band_rows(10, 10, (1, -1, 0), np.array([[10.0, 20.0, 30.0], [11.0, 21.0, 31.0]]))
    assert list(col2[row2[4]:row2[5]]) == [3, 4, 5] and list(val2[row2[4]:row2[5]]) == [20.0, 30.0, 10.0]
    assert list(val2[row2[5]:row2[6]]) == [21.0, 31.0, 11.0]


def _classes_from_reference_packing(row, col, val):
    """Distinct (distances, values) tuples of the reference packing's rows, padding rows included.  On a band the set
    of distances a row holds fixes its slot mask, so this counts the same classes by another route."""
    h = oracle.hell_pack(row, col, val)
    p, w = h["pitch"], h["width"]
    keys = set()
    for i in range(p):
        c = [int(h["ell_col"][i + p * k]) for k in range(w)]
        keys.add((tuple(ci - i for ci in c if ci >= 0), tuple(float(h["ell_val"][i + p * k]) for k in range(w) if c[k] >= 0)))
    return len(keys)


@pytest.mark.parametrize("n, m, offsets, K", [(100, 100, (-1, 0, 1), 1), (101, 100, (-2, 0, 3), 3), (64, 66, (0, 1, 2), 7),
                                              (50, 70, (-7, -3, -1), 5), (33, 33, (-1, 0, 1, 2, 5), 4)])
def test_classes_expected_agrees_with_reference_packing(n, m, offsets, K):
    tuples = 1.0 + np.arange(K * len(offsets), dtype=np.float64).reshape(K, len(offsets))
    row, col, val = band_rows(n, m, offsets, tuples)
    assert classes_expected(row, col, val) == _classes_from_reference_packing(row, col, val)


def test_classes_expected_on_hand_built_strips():
    # tridiagonal, n % 16 == 0: interior, first row, last row
    assert classes_expected(*band(64, 64, (-1, 0, 1), np.array([-1.0, 2.0, -1.0]))) == 3
    # ... n % 16 != 0: and the padding rows' empty class
    assert classes_expected(*band(65, 65, (-1, 0, 1), np.array([-1.0, 2.0, -1.0]))) == 4
    # every row full (m = n + 2), K value tuples: K classes, + 1 with padding rows
    tup = np.array([[1.0, 2.0, 3.0], [1.0, 2.0, 4.0], [1.0, 2.0, 3.0]])
    assert classes_expected(*band_rows(32, 34, (0, 1, 2), tup)) == 2
    assert classes_expected(*band_rows(33, 35, (0, 1, 2), tup)) == 3
    # values are compared bit for bit: -0.0 and 0.0 are two classes
    assert classes_expected(*band_rows(32, 34, (0, 1, 2), np.array([[1.0, 0.0, 3.0], [1.0, -0.0, 3.0]]))) == 2
    # empty rows (all columns outside [0, m)) share the padding rows' class: first row, interior, rows 19 and 20, empty
    row, col, val = band(40, 20, (-1, 0, 1), np.array([1.0, 2.0, 3.0]))
    ids = row_class_ids(row, col, val)
    assert ids[25] == ids[39] == ids[45] and classes_expected(row, col, val) == 5
    # a row with fewer entries than the width keeps each entry in the slot of its distance
    row = np.array([0, 2, 5, 8, 10]); col = np.array([0, 1, 0, 1, 2, 1, 2, 3, 2, 3])
    val = np.ones(10)
    ids = row_class_ids(row, col, val)
    assert list(ids[:5]) == [0, 1, 1, 2, 3] and classes_expected(row, col, val) == 4


@pytest.mark.parametrize("case", ["band", "one-sided", "rectangular", "tail", "random"])
def test_ell_ref_float64_is_csr_spmv(case):
    if case == "band":
        row, col, val = band(5003, 5003, (-70, -1, 0, 1, 70), oracle.uniform_real(1, 5) - 0.5)
    elif case == "one-sided":
        row, col, val = band(777, 777, (-7, -3, -1), oracle.uniform_real(2, 3))
    elif case == "rectangular":
        row, col, val = band(900, 600, (-2, 0, 1, 4), oracle.uniform_real(3, 4) - 0.5)
    elif case == "tail":
        row, col, val = with_long_rows(*band_rows(300, 300, (-1, 0, 1), oracle.uniform_real(5, 30).reshape(10, 3)),
                                       long_rows={7, 100, 240})
        assert ell_width(row) == 3 and row[-1] == 3 * 300 - 2 + 6
    else:
        row, col, val = oracle.random_matrix(2000, 2500, 12, 9)
    m = int(col.max()) + 1 if col.size else 1
    x = oracle.uniform_real(17, m) - 0.5
    assert np.array_equal(ell_ref(row, col, val, x, np.float64), oracle.csr_spmv(row, col, val, x))


def test_ell_ref_float32_rounds_every_operation():
    """One row, two entries: the float32 reference must round the products and the sum separately."""
    row, col = np.array([0, 2]), np.array([0, 1])
    val = np.array([1 + 2.0 ** -12, 1 + 2.0 ** -12], np.float32)
    x = np.array([1 + 2.0 ** -12, -1.0], np.float32)
    p0 = np.float32(val[0] * x[0])                          # 1 + 2^-11 (+ 2^-24 rounded away)
    assert ell_ref(row, col, val, x, np.float32)[0] == np.float32(p0 - val[1])
    assert ell_ref(row, col, val, x, np.float32).dtype == np.float32


# ------------------------------------------------------------------------------------------------ GPU helpers

ENCODINGS = {                       # what each encoding sets at construction, on top of the defaults
    "classes": {"spmv.ell_classes": 2},
    "masks": {"spmv.ell_classes": 0},
    "col16": {"spmv.ell_classes": 0, "spmv.ell_diag": 0},
    "col32": {"spmv.col16": 0},
}
DEFAULTS = {"spmv.ell_classes": 1, "spmv.ell_diag": 1, "spmv.col16": 1}


def spmat(ctx, n, m, row, col, val, enc):
    for k, v in ENCODINGS[enc].items():
        vx.set_param(k, v)
    try:
        return vx.SpMat(ctx, n, m, row, col, val, vx.FMT_HELL)
    finally:
        for k, v in DEFAULTS.items():
            vx.set_param(k, v)


def check_encoding(info, enc, classes_ok=True):
    """The encoding a one-part strip took: row classes and slot masks only at the widths with an unrolled kernel and one
    slot mask byte (3, 5, 7); every other width keeps a column array."""
    if info.ell_width in (3, 5, 7) and enc in ("classes", "masks"):
        assert info.ell_col_bytes == 0
        assert (info.ell_classes > 0) == (enc == "classes" and classes_ok)
    else:
        assert info.ell_classes == 0
        assert info.ell_col_bytes == (4 if enc == "col32" else 2)


def check_y(got, want, mag, w, exact, dtype):
    if exact:
        assert got.dtype == want.dtype and np.array_equal(got, want), np.nonzero(got != want)[0][:8]
    else:
        u = np.finfo(dtype).eps / 2
        bad = np.abs(got.astype(np.float64) - want.astype(np.float64)) > 2 * (w + 2) * u * mag
        assert not bad.any(), np.nonzero(bad)[0][:8]


def check_readers(ctx, A, row, col, val, m, dtype=np.float64, seed=0):
    """Every reader of the strip against ell_ref: bit-exact on one part, within the ordering bound otherwise."""
    n = row.size - 1
    exact = ctx.nparts == 1
    w = int(np.diff(row).max()) if n else 0
    X = [(oracle.uniform_real(100 + seed + r, m) - 0.5).astype(dtype) for r in range(6)]
    ref = [ell_ref(row, col, val, Xr, dtype) for Xr in X]
    mag = [oracle.csr_absrow(row, col, val.astype(np.float64), Xr.astype(np.float64)) for Xr in X]
    x, y = vx.vector(ctx, X[0]), vx.vector(ctx, n, dtype)
    # hell_kernel: y = A*x, then y += 3 A*x
    y.assign(A * x)
    check_y(y.read(), ref[0], mag[0], w, exact, dtype)
    y += 3.0 * (A * x)
    check_y(y.read(), axpy_ref(ref[0], 3.0, ref[0], dtype), 4 * mag[0], w + 1, exact, dtype)
    # hell_multi_kernel: 1 to 6 right-hand sides (groups of 4, then 3 / 2 / 1)
    xs = [vx.vector(ctx, Xr) for Xr in X]
    ys = [vx.vector(ctx, n, dtype) for _ in X]
    for K in range(1, 7):
        A.apply_multi(xs[:K], ys[:K], 1.0, False)
        for r in range(K):
            check_y(ys[r].read(), ref[r], mag[r], w, exact, dtype)
        A.apply_multi(xs[:K], ys[:K], -0.5, True)
        for r in range(K):
            check_y(ys[r].read(), axpy_ref(ref[r], -0.5, ref[r], dtype), 1.5 * mag[r], w + 1, exact, dtype)
    if ctx.nparts == 1:
        # dist_apply_kernel: the fused product + dot (several slots of one device would need NCCL for the dot)
        W = (oracle.uniform_real(200 + seed, n) - 0.5).astype(dtype)
        wv, d = vx.vector(ctx, W), DeviceScalar(ctx, dtype)
        y.assign(Scalar(dtype(0)))
        assert A.apply_dot(x, y, d, dot_with=wv)
        got = y.read()
        check_y(got, ref[0], mag[0], w, exact, dtype)
        u = np.finfo(dtype).eps / 2
        dot = float(np.dot(W.astype(np.float64), got.astype(np.float64)))
        assert abs(float(d.get()) - dot) <= (n + 2) * u * float(np.sum(np.abs(W.astype(np.float64) * got.astype(np.float64))))
        # generated row function: y = z + A*x as one kernel (strips without a halo)
        Z = (oracle.uniform_real(300 + seed, n) - 0.5).astype(dtype)
        z = vx.vector(ctx, Z)
        n0 = vx.launch_count()
        y.assign(z + A * x)
        assert vx.launch_count() - n0 == 1
        check_y(y.read(), (Z + ref[0]).astype(dtype), mag[0], w, True, dtype)


# ------------------------------------------------------------------------------------------------ 1. widths

WIDTH_OFFSETS = {1: (0,), 2: (-1, 1), 3: (-1, 0, 1), 4: (-2, -1, 1, 2), 5: (-50, -1, 0, 1, 50), 6: (-3, -2, -1, 0, 1, 4),
                 7: (-400, -20, -1, 0, 1, 20, 400), 8: (-4, -3, -2, -1, 1, 2, 3, 4), 9: tuple(range(-4, 5)),
                 10: (-9, -5, -3, -2, -1, 0, 1, 2, 3, 5), 27: tuple(range(-13, 14))}


def width_band(w, n=6000, dtype=np.float64):
    vals = (np.linspace(-1.0, 1.0, w) + 0.125 * w).astype(dtype)
    vals[len(vals) // 2] = dtype(2.0 * w)
    return band(n, n, WIDTH_OFFSETS[w], vals)


@pytest.mark.gpu
@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("w", list(WIDTH_OFFSETS))
@pytest.mark.parametrize("nparts", [1, 2, 3])
def test_band_widths(ctx1, ctx2, ctx3, nparts, w, enc):
    ctx = {1: ctx1, 2: ctx2, 3: ctx3}[nparts]
    row, col, val = width_band(w)
    n = row.size - 1
    A = spmat(ctx, n, n, row, col, val, enc)
    if nparts == 1:
        info = A.info().loc
        assert info.ell_width == w and info.csr_tail_nnz == 0
        check_encoding(info, enc)
    check_readers(ctx, A, row, col, val, n, seed=w)


@pytest.mark.gpu
@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("w", list(WIDTH_OFFSETS))
def test_band_widths_float32(ctx1, w, enc):
    row, col, val = width_band(w, dtype=np.float32)
    n = row.size - 1
    A = spmat(ctx1, n, n, row, col, val, enc)
    check_encoding(A.info().loc, enc)
    check_readers(ctx1, A, row, col, val, n, np.float32, seed=w)


# ------------------------------------------------------------------------------------------------ 2. row counts

ROW_COUNTS = [1, 2, 3, 15, 16, 17, 255, 256, 257, 511, 512, 513, 1023, 1025, 67583, 67584, 67585, 68097, 200003]
ROW_COUNTS_SUBSET = [1, 17, 257, 513, 1025, 67583, 67585, 200003]
STENCIL = {3: ((-1, 0, 1), [-1.0, 2.5, -1.25]), 5: ((-300, -1, 0, 1, 300), [-0.5, -1.0, 4.25, -1.5, -0.75]),
           7: ((-5000, -70, -1, 0, 1, 70, 5000), [-0.25, -0.5, -1.0, 6.5, -1.25, -0.75, -0.125])}
_matrices = {}


def stencil_band(w, n, dtype=np.float64):
    key = (w, n, np.dtype(dtype).name)
    if key not in _matrices:
        offsets, vals = STENCIL[w]
        _matrices[key] = band(n, n, offsets, np.array(vals, dtype))
    return _matrices[key]


def _row_count_cases():
    cases = [(5, n) for n in ROW_COUNTS]
    cases += [(w, n) for w in (3, 7) for n in ROW_COUNTS_SUBSET]
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("w, n", _row_count_cases())
def test_row_counts(ctx1, w, n, enc):
    row, col, val = stencil_band(w, n)
    A = spmat(ctx1, n, n, row, col, val, enc)
    info = A.info().loc
    assert info.ell_pitch == (n + 15) // 16 * 16
    check_encoding(info, enc)
    check_readers(ctx1, A, row, col, val, n, seed=n % 97)


@pytest.mark.gpu
@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("n", [1, 17, 257, 513, 67585, 200003])
@pytest.mark.parametrize("nparts", [2, 3])
def test_row_counts_in_parts(ctx2, ctx3, nparts, n, enc):
    ctx = {2: ctx2, 3: ctx3}[nparts]
    row, col, val = stencil_band(5, n)
    A = spmat(ctx, n, n, row, col, val, enc)
    check_readers(ctx, A, row, col, val, n, seed=n % 89)


@pytest.mark.gpu
@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("w, n", [(5, n) for n in ROW_COUNTS] + [(3, 67585), (7, 1025), (7, 200003)])
def test_row_counts_float32(ctx1, w, n, enc):
    row, col, val = stencil_band(w, n, np.float32)
    A = spmat(ctx1, n, n, row, col, val, enc)
    check_encoding(A.info().loc, enc)
    check_readers(ctx1, A, row, col, val, n, np.float32, seed=n % 97)


# ------------------------------------------------------------------------------------------------ 3. shift geometry

GEOMETRY = {                            # (n, m, offsets): all long enough for the class kernel's prefetch to issue
    "positive": (100000, 100000, (1, 2, 5)),
    "negative": (100000, 100000, (-7, -3, -1)),
    "tall": (100000, 70000, (-2, -1, 0, 1, 3)),
    "wide": (70000, 100000, (-1, 0, 1, 4, 6)),
    "wide-far": (70000, 140000, (-3, 0, 30000, 70000, 70003)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("geom", list(GEOMETRY))
@pytest.mark.parametrize("nparts", [1, 2, 3])
def test_shift_geometry(ctx1, ctx2, ctx3, nparts, geom, enc):
    ctx = {1: ctx1, 2: ctx2, 3: ctx3}[nparts]
    n, m, offsets = GEOMETRY[geom]
    key = ("geom", geom)
    if key not in _matrices:
        _matrices[key] = band(n, m, offsets, np.array([1.5, -0.75, 2.25, -1.0, 0.5][:len(offsets)]))
    row, col, val = _matrices[key]
    A = spmat(ctx, n, m, row, col, val, enc)
    if nparts == 1:
        info = A.info().loc
        assert info.ell_width == len(offsets)
        check_encoding(info, enc)
    check_readers(ctx, A, row, col, val, m, seed=len(geom))


# ------------------------------------------------------------------------------------------------ 4. class count

def class_tuples(K, dtype):
    k = np.arange(K, dtype=np.float64)[:, None]
    return (np.array([[1.0, -2.0, 0.5]]) + k * np.array([[2.0 ** -9, -(2.0 ** -10), 2.0 ** -12]])).astype(dtype)


# (K value tuples, n): every row full (band (0, 1, 2) on n + 2 columns), so the classes are the K tuples and, when
# n % 16 != 0, the padding rows' empty class
CLASS_COUNTS = [(255, 4096, 255), (255, 4099, 256), (256, 4096, 256), (256, 4099, 257), (257, 4096, 257)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("K, n, count", CLASS_COUNTS)
def test_class_count_boundary(ctx1, K, n, count, dtype):
    row, col, val = band_rows(n, n + 2, (0, 1, 2), class_tuples(K, dtype))
    ids = row_class_ids(row, col, val)
    assert classes_expected(row, col, val) == count
    A = spmat(ctx1, n, n + 2, row, col, val, "classes")
    info = A.info().loc
    assert info.ell_width == 3 and info.ell_col_bytes == 0
    if count <= 256:
        assert info.ell_classes == count
        assert info.device_bytes == info.ell_pitch + 256 + count * 3 * np.dtype(dtype).itemsize
        if count == 256 and n % 16 == 0:
            assert np.count_nonzero(ids[:n] == 255) == len(range(255, n, K))    # the last table row multiplies rows
    else:
        assert info.ell_classes == 0                                           # too many: slot masks
    check_readers(ctx1, A, row, col, val, n + 2, dtype, seed=K)


@pytest.mark.gpu
@pytest.mark.parametrize("K, n, count", [(256, 4096, 256), (257, 4096, 257)])
def test_class_count_boundary_in_parts(ctx2, K, n, count):
    row, col, val = band_rows(n, n + 2, (0, 1, 2), class_tuples(K, np.float64))
    A = spmat(ctx2, n, n + 2, row, col, val, "classes")
    check_readers(ctx2, A, row, col, val, n + 2, seed=K)


# ------------------------------------------------------------------------------------------------ 5. 16-bit span

def span_strip(n, S):
    """Width 3: distances -1, 0 and, in the third slot, 1 on even rows and 1 + S on odd rows (span S)."""
    m = n + S + 2
    row = [0]; col = []
    for i in range(n):
        if i > 0:
            col.append(i - 1)
        col += [i, i + 1 + (S if i % 2 else 0)]
        row.append(len(col))
    row, col = np.array(row, np.int64), np.array(col, np.int64)
    return row, col, oracle.uniform_real(31, col.size) - 0.5, m


@pytest.mark.gpu
@pytest.mark.parametrize("S, col_bytes", [(65534, 2), (65535, 4)])
def test_16bit_column_span(ctx1, S, col_bytes):
    n = 3001
    row, col, val, m = span_strip(n, S)
    assert m >= n + 65536
    A = vx.SpMat(ctx1, n, m, row, col, val, vx.FMT_HELL)
    info = A.info().loc
    assert info.ell_width == 3 and info.ell_classes == 0 and info.ell_col_bytes == col_bytes
    check_readers(ctx1, A, row, col, val, m, seed=S % 7)
