"""Double vex::SpMat products from float-stored values (VEXB_FMT_VALUES_F32).

A double matrix created with the flag stores each value as (float)v and multiplies double x into double y, every
product double(v_f) * x_j and every sum in double, by the kernel and in the order of the double strip.  So for every
format, encoding, tunable, part count and assign op y must have the bits of the double SpMat built from the rounded
values val.astype(float32).astype(float64) with the same fmt -- which is what every test here compares, with
np.array_equal on uint64 views.  The layout (format, ELL width, encoding, classes, tiles) must match that strip too;
only the value arrays shrink, by 4 bytes per stored value, padding included.

Values carry full 53-bit mantissas, so a flag that were ignored would give the unrounded product (checked once below).
Readers without a float-valued kernel must refuse such strips and fall back to a path that exists: apply_multi runs one
product per vector, an inlined product goes to a temporary, the peer-memory halo does not connect and the fused
product + dot is composed."""
import ctypes as C

import numpy as np
import pytest

import vexcl_b200 as vx
from vexcl_b200 import _lib as L
from vexcl_b200.api import DeviceScalar, Reductor

pytestmark = pytest.mark.gpu

F32 = vx.FMT_VALUES_F32
OPS = {"=": (1.0, False), "+=": (1.0, True), "-=": (-1.0, True), "0.5+=": (0.5, True)}
ENCODINGS = {                       # as tests/test_gpu_ell_edges.py
    "classes": {"spmv.ell_classes": 2},
    "masks": {"spmv.ell_classes": 0},
    "col16": {"spmv.ell_classes": 0, "spmv.ell_diag": 0},
    "col32": {"spmv.col16": 0},
}
DEFAULTS = {"spmv.ell_classes": 1, "spmv.ell_diag": 1, "spmv.col16": 1, "spmv.kernel": -1}


@pytest.fixture
def params(built):
    """vx.set_param, with every parameter used here back at its default afterwards."""
    try:
        yield vx.set_param
    finally:
        for k, v in DEFAULTS.items():
            vx.set_param(k, v)


def rounded(val):
    return val.astype(np.float32).astype(np.float64)


def full_mantissa(rng, size):
    """Values in +-[0.5, 2) whose low 29 mantissa bits are not all zero: float rounding changes every one of them."""
    v = (rng.random(size) * 1.5 + 0.5) * np.where(rng.random(size) < 0.5, -1.0, 1.0)
    bits = v.view(np.uint64) | np.uint64(1)
    return bits.view(np.float64)


# ------------------------------------------------------------------------------------------------ matrices

def band(n, m, offsets, tuples):
    """Row i holds tuples[i mod K][k] at column i + offsets[k] where that column lies in [0, m)."""
    offsets = np.sort(np.asarray(offsets, np.int64))
    cols = np.arange(n, dtype=np.int64)[:, None] + offsets[None, :]
    inside = (cols >= 0) & (cols < m)
    row = np.zeros(n + 1, np.int64)
    np.cumsum(inside.sum(axis=1), out=row[1:])
    vals = np.asarray(tuples)[np.arange(n) % len(tuples)]
    return row, cols[inside], np.ascontiguousarray(vals[inside])


def poisson2d(g, rng, distinct=3):
    """5-point stencil on a g x g grid; `distinct` value tuples repeat over the rows (row classes stay possible)."""
    return band(g * g, g * g, [-g, -1, 0, 1, g], full_mantissa(rng, (distinct, 5)))


def poisson3d(g, rng, distinct=3):
    return band(g ** 3, g ** 3, [-g * g, -g, -1, 0, 1, g, g * g], full_mantissa(rng, (distinct, 7)))


def from_lengths(lengths, m, rng, spread=None):
    """Rows of the given lengths; columns anywhere in [0, m) or within +-spread of the diagonal, sorted, distinct."""
    n = len(lengths)
    row = np.zeros(n + 1, np.int64)
    np.cumsum(lengths, out=row[1:])
    col = np.empty(row[-1], np.int64)
    for i, w in enumerate(lengths):
        if spread is None:
            c = rng.choice(m, size=w, replace=False)
        else:
            lo, hi = max(0, i - spread), min(m, i + spread + 1)
            c = lo + rng.choice(hi - lo, size=w, replace=False)
        col[row[i]:row[i + 1]] = np.sort(c)
    return row, col, full_mantissa(rng, row[-1])


def with_tail(row, col, val, every, rng):
    """Two more entries (50 and 53 right of the diagonal) in every `every`-th row: rows past the ELL width."""
    n = row.size - 1
    r2, c2, v2 = [0], [], []
    for i in range(n):
        c = list(col[row[i]:row[i + 1]]); v = list(val[row[i]:row[i + 1]])
        if i % every == 0 and i + 53 < n:
            c += [i + 50, i + 53]; v += list(full_mantissa(rng, 2))
        c2 += c; v2 += v
        r2.append(len(c2))
    return np.array(r2, np.int64), np.array(c2, np.int64), np.array(v2, np.float64)


# ------------------------------------------------------------------------------------------------ checks

def build_pair(ctx, n, m, row, col, val, fmt, settings):
    """(float-valued SpMat, double SpMat of the rounded values), both built under `settings`."""
    for k, v in settings.items():
        vx.set_param(k, v)
    try:
        return vx.SpMat(ctx, n, m, row, col, val, fmt | F32), vx.SpMat(ctx, n, m, row, col, rounded(val), fmt)
    finally:
        for k in settings:
            vx.set_param(k, DEFAULTS[k])


INFO_FIELDS = [f for f, _ in L.SpmatInfo._fields_ if f not in ("val_bytes", "device_bytes")]


def check_info(ctx, A, D):
    """Same layout on every part; val_bytes 4 (8 on the double strip) except on row-class / row-pattern strips (0)."""
    for k in ctx.local:
        a, d = A.info(k), D.info(k)
        for f in ("nrows", "ncols_local", "n_ghost", "n_send", "loc_nnz", "rem_nnz"):
            assert getattr(a, f) == getattr(d, f), f
        for sa, sd in ((a.loc, d.loc), (a.rem, d.rem)):
            for f in INFO_FIELDS:
                assert getattr(sa, f) == getattr(sd, f), f
            if sd.val_bytes == 0:
                assert sa.val_bytes == 0 and sa.device_bytes == sd.device_bytes
            elif sd.nrows:
                assert (sa.val_bytes, sd.val_bytes) == (4, 8)
                assert sa.device_bytes <= sd.device_bytes          # equal only when no value is stored


def value_slots(info, row):
    """Stored values of a one-part strip, padding included, from the host layout: what the flag saves 4 bytes on."""
    if info.val_bytes == 0:
        return 0
    if info.fmt == L.FMT_CSR:
        return info.nnz + 16
    if info.fmt == L.FMT_HELL:
        return info.ell_pitch * info.ell_width + info.csr_tail_nnz
    assert info.fmt == L.FMT_SELL
    n = row.size - 1
    ptr = np.ascontiguousarray(row, np.int64)
    ns, slots = C.c_size_t(), C.c_size_t()
    L.check(L.lib().vexb_csr_sell_layout(n, ptr.ctypes.data, 8, 1024, C.byref(ns), C.byref(slots), None, None))
    return slots.value + 32


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def assert_same(got, want, what=""):
    g, w = bits(got), bits(want)
    assert np.array_equal(g, w), f"{what}: {np.count_nonzero(g != w)} of {g.size} differ, first at {np.nonzero(g != w)[0][:8]}"


def check_products(ctx, A, D, n, m, seed, ops=OPS):
    """Every assign op in sequence on the same y: float-valued strip against the double strip of the rounded values."""
    rng = np.random.default_rng(seed)
    X = full_mantissa(rng, m)
    Y0 = full_mantissa(rng, n)
    x = vx.vector(ctx, X)
    ya, yd = vx.vector(ctx, Y0), vx.vector(ctx, Y0)
    for name, (alpha, append) in ops.items():
        A.apply(x, ya, alpha, append)
        D.apply(x, yd, alpha, append)
        assert_same(ya.read(), yd.read(), name)
    return X


def run_case(ctx, row, col, val, m, fmt, settings=None, seed=0):
    n = row.size - 1
    A, D = build_pair(ctx, n, m, row, col, val, fmt, settings or {})
    check_info(ctx, A, D)
    if len(ctx.local) == 1:
        assert D.info().loc.device_bytes - A.info().loc.device_bytes == 4 * value_slots(D.info().loc, row)
    check_products(ctx, A, D, n, m, seed)
    return A, D


# ------------------------------------------------------------------------------------------------ 1. families

@pytest.mark.parametrize("enc", list(ENCODINGS))
@pytest.mark.parametrize("dim", [2, 3])
def test_poisson_encodings(ctx, params, dim, enc):
    rng = np.random.default_rng(dim)
    row, col, val = poisson2d(150, rng) if dim == 2 else poisson3d(28, rng)
    m = row.size - 1
    A, D = run_case(ctx, row, col, val, m, vx.FMT_HELL, ENCODINGS[enc], seed=dim)
    info = D.info().loc
    assert info.fmt == L.FMT_HELL
    if len(ctx.local) == 1:
        assert info.ell_classes > 0 if enc == "classes" else info.ell_classes == 0
        assert info.ell_col_bytes == {"classes": 0, "masks": 0, "col16": 2, "col32": 4}[enc]
        assert A.info().loc.val_bytes == (0 if enc == "classes" else 4)


@pytest.mark.parametrize("enc", ["masks", "col16", "col32"])
def test_poisson_random_coefficients_auto(ctx, params, enc):
    """Every row distinct (no row classes at any setting), format picked by VEXB_FMT_AUTO."""
    rng = np.random.default_rng(5)
    g = 120
    row, col, _ = poisson2d(g, rng)
    val = full_mantissa(rng, col.size)
    run_case(ctx, row, col, val, g * g, vx.FMT_AUTO, ENCODINGS[enc], seed=6)


@pytest.mark.parametrize("enc", ["masks", "col16", "col32"])
def test_hybrid_ell_with_tail(ctx, params, enc):
    rng = np.random.default_rng(7)
    row, col, val = poisson2d(100, rng, distinct=5)
    row, col, val = with_tail(row, col, val, 37, rng)
    A, D = run_case(ctx, row, col, val, row.size - 1, vx.FMT_HELL, ENCODINGS[enc], seed=8)
    if len(ctx.local) == 1:
        assert D.info().loc.csr_tail_nnz > 0


@pytest.mark.parametrize("cols", ["col16", "col32"])
def test_sliced_ell_irregular(ctx, params, cols):
    rng = np.random.default_rng(9)
    n = 20000
    lengths = rng.integers(0, 32, n)
    spread = 3000 if cols == "col16" else None
    row, col, val = from_lengths(lengths, n, rng, spread)
    A, D = run_case(ctx, row, col, val, n, vx.FMT_AUTO, {"spmv.col16": 1 if cols == "col16" else 0}, seed=10)
    if len(ctx.local) == 1:
        assert D.info().loc.fmt == L.FMT_SELL


@pytest.mark.parametrize("kernel", [-1, 3, 4])
@pytest.mark.parametrize("shape", ["short", "mixed"])
def test_csr_variants(ctx, params, kernel, shape):
    """Forced CSR: thread per row (3), warp tiles (4), and the strip's own choice; rows of up to 900 entries take the
    warp-tile long-row branch."""
    rng = np.random.default_rng(11)
    n = 12000
    lengths = rng.integers(0, 9, n) if shape == "short" else rng.integers(0, 40, n)
    if shape == "mixed":
        lengths[::1500] = 900
    row, col, val = from_lengths(lengths, n, rng)
    A, D = build_pair(ctx, n, n, row, col, val, vx.FMT_CSR, {})
    check_info(ctx, A, D)
    if len(ctx.local) == 1:
        assert D.info().loc.device_bytes - A.info().loc.device_bytes == 4 * value_slots(D.info().loc, row)
    params("spmv.kernel", kernel)
    check_products(ctx, A, D, n, n, seed=12)


@pytest.mark.parametrize("fmt", [vx.FMT_AUTO, vx.FMT_CSR, vx.FMT_HELL, vx.FMT_SELL])
def test_small_shapes(ctx, params, fmt):
    """Mostly empty rows, no entries at all, one row, and rectangular strips (wider and taller)."""
    rng = np.random.default_rng(13)
    lengths = np.where(rng.random(3000) < 0.9, 0, rng.integers(1, 12, 3000))
    cases = [
        (from_lengths(lengths, 3000, rng), 3000),
        ((np.zeros(101, np.int64), np.zeros(0, np.int64), np.zeros(0)), 100),
        (from_lengths([7], 40, rng), 40),
        (from_lengths(rng.integers(0, 20, 500), 7000, rng), 7000),
        (from_lengths(rng.integers(0, 20, 5000), 300, rng), 300),
    ]
    for i, ((row, col, val), m) in enumerate(cases):
        run_case(ctx, row, col, val, m, fmt, seed=14 + i)


def test_flag_is_not_ignored(ctx1, params):
    """With full-mantissa values the float-valued product differs from the unrounded double product."""
    rng = np.random.default_rng(15)
    row, col, val = poisson2d(60, rng)
    n = row.size - 1
    for fmt, settings in ((vx.FMT_HELL, ENCODINGS["masks"]), (vx.FMT_SELL, {}), (vx.FMT_CSR, {})):
        A, D = build_pair(ctx1, n, n, row, col, val, fmt, settings)
        U = vx.SpMat(ctx1, n, n, row, col, val, fmt)
        x = vx.vector(ctx1, full_mantissa(rng, n))
        ya, yu = vx.vector(ctx1, n), vx.vector(ctx1, n)
        A.apply(x, ya); U.apply(x, yu)
        assert np.count_nonzero(bits(ya.read()) != bits(yu.read())) > n // 2, fmt


# ------------------------------------------------------------------------------------------------ 2. launches, bounds, downloads

def test_one_launch_per_product(ctx1, params):
    rng = np.random.default_rng(16)
    row, col, val = poisson2d(80, rng)
    n = row.size - 1
    lengths = rng.integers(0, 32, 5000)
    irow, icol, ival = from_lengths(lengths, 5000, rng)
    for (r, c, v, m), fmt in (((row, col, val, n), vx.FMT_HELL), ((irow, icol, ival, 5000), vx.FMT_SELL),
                              ((irow, icol, ival, 5000), vx.FMT_CSR)):
        A = vx.SpMat(ctx1, r.size - 1, m, r, c, v, fmt | F32)
        x, y = vx.vector(ctx1, np.ones(m)), vx.vector(ctx1, r.size - 1)
        A.apply(x, y)
        n0 = vx.launch_count()
        A.apply(x, y, 0.5, True)
        assert vx.launch_count() - n0 == 1, fmt


@pytest.mark.parametrize("fmt", [vx.FMT_HELL, vx.FMT_SELL, vx.FMT_CSR])
def test_nothing_past_y(ctx1, params, fmt):
    """vexb_spmv on a vexb_csr_create strip, y longer than n: the entries past n keep their sentinel."""
    rng = np.random.default_rng(17)
    row, col, val = from_lengths(rng.integers(1, 9, 4000), 4000, rng, spread=100)
    n, m, extra = 4000, 4000, 77
    lib, k = L.lib(), ctx1.local[0]
    hs = []
    try:
        for v, f in ((val, fmt | F32), (rounded(val), fmt)):
            h = C.c_void_p()
            L.check(lib.vexb_csr_create(ctx1.devs[k], ctx1.streams[k], n, m, row.ctypes.data, 8, col.ctypes.data, 8,
                                        v.ctypes.data, L.F64, f, C.byref(h)))
            hs.append(h)
        x = vx.vector(ctx1, full_mantissa(rng, m))
        ys = [vx.vector(ctx1, np.full(n + extra, 12345.5)) for _ in hs]
        for alpha, append in OPS.values():
            for h, y in zip(hs, ys):
                L.check(lib.vexb_spmv(ctx1.devs[k], ctx1.streams[k], h, x.bufs[k], y.bufs[k], alpha, int(append)))
        a, d = ys[0].read(), ys[1].read()
        assert np.all(a[n:] == 12345.5)
        assert_same(a[:n], d[:n], "y")
    finally:
        for h in hs:
            lib.vexb_spmat_destroy(h)


def test_downloads_return_rounded_values(ctx2, params):
    """vexb_spmat_hell_download and vexb_dspmat_download_split give the rounded values as double."""
    rng = np.random.default_rng(18)
    row, col, val = poisson2d(50, rng, distinct=4)
    row, col, val = with_tail(row, col, val, 11, rng)
    n = row.size - 1
    A, D = build_pair(ctx2, n, n, row, col, val, vx.FMT_HELL, ENCODINGS["col16"])
    lib = L.lib()
    for k in ctx2.local:
        ia = A.info(k)
        nl, nr = ia.loc_nnz, ia.rem_nnz
        got = [np.zeros(nl), np.zeros(nr)]
        want = [np.zeros(nl), np.zeros(nr)]
        L.check(lib.vexb_dspmat_download_split(A.parts[k], None, None, got[0].ctypes.data, None, None, got[1].ctypes.data))
        L.check(lib.vexb_dspmat_download_split(D.parts[k], None, None, want[0].ctypes.data, None, None, want[1].ctypes.data))
        for g, w in zip(got, want):
            assert_same(g, w, "split")
    # one strip: the hybrid-ELL arrays and the CSR tail themselves
    k = ctx2.local[0]
    hs, got = [], []
    try:
        for v, f in ((val, vx.FMT_HELL | F32), (rounded(val), vx.FMT_HELL)):
            h = C.c_void_p()
            L.check(lib.vexb_csr_create(ctx2.devs[k], ctx2.streams[k], n, n, row.ctypes.data, 8, col.ctypes.data, 8,
                                        v.ctypes.data, L.F64, f, C.byref(h)))
            hs.append(h)
            info = L.SpmatInfo()
            L.check(lib.vexb_spmat_get_info(h, C.byref(info)))
            ne, nt = info.ell_pitch * info.ell_width, info.csr_tail_nnz
            assert nt > 0
            ev, tv = np.zeros(ne), np.zeros(nt)
            L.check(lib.vexb_spmat_hell_download(h, None, ev.ctypes.data, None, None, tv.ctypes.data))
            got.append((ev, tv))
        assert_same(got[0][0], got[1][0], "ELL values")
        assert_same(got[0][1], got[1][1], "tail values")
    finally:
        for h in hs:
            lib.vexb_spmat_destroy(h)


# ------------------------------------------------------------------------------------------------ 3. readers that refuse

def hell_pair(ctx, g=90, seed=19):
    rng = np.random.default_rng(seed)
    row, col, val = poisson2d(g, rng)
    val = full_mantissa(rng, col.size)
    n = row.size - 1
    return (*build_pair(ctx, n, n, row, col, val, vx.FMT_HELL, ENCODINGS["masks"]), n, rng)


def test_multi_vector_is_one_product_per_vector(ctx, params):
    A, D, n, rng = hell_pair(ctx)
    xs = [vx.vector(ctx, full_mantissa(rng, n)) for _ in range(3)]
    ya = [vx.vector(ctx, n) for _ in range(3)]
    yd = [vx.vector(ctx, n) for _ in range(3)]
    n0 = vx.launch_count()
    A.apply_multi(xs, ya, 0.5, False)
    if len(ctx.local) == 1:
        assert vx.launch_count() - n0 == 3
    for x, y in zip(xs, yd):
        D.apply(x, y, 0.5, False)
    for a, d in zip(ya, yd):
        assert_same(a.read(), d.read(), "apply_multi")


def test_inlined_product_goes_through_a_temporary(ctx, params):
    A, D, n, rng = hell_pair(ctx)
    lib = L.lib()
    for k in ctx.local:
        h = C.c_void_p()
        L.check(lib.vexb_dspmat_inline_strip(A.parts[k], C.byref(h)))
        assert not h.value
    Z = full_mantissa(rng, n)
    x, z = vx.vector(ctx, full_mantissa(rng, n)), vx.vector(ctx, Z)
    y, tmp = vx.vector(ctx, n), vx.vector(ctx, n)
    y.assign(z + vx.make_inline(A * x))
    D.apply(x, tmp)
    assert_same(y.read(), Z + tmp.read(), "y = z + make_inline(A*x)")
    # the additive spelling, against the same spelling on the double strip (over several parts the ghost entries are
    # added to y after the local ones, on both)
    ya, yd = vx.vector(ctx, n), vx.vector(ctx, n)
    ya.assign(z + A * x)
    yd.assign(z + D * x)
    assert_same(ya.read(), yd.read(), "y = z + A*x")


def test_peer_halo_refused(ctx2, params):
    A, D, n, rng = hell_pair(ctx2)
    lib = L.lib()
    assert lib.vexb_dspmat_halo_connect_local(len(ctx2.local), ctx2._arr(A.parts)) == L.ERR_UNSUPPORTED
    handles = C.create_string_buffer(64 * ctx2.nparts)
    for k in ctx2.local:
        assert lib.vexb_dspmat_halo_connect(A.parts[k], handles) == L.ERR_UNSUPPORTED
        c = C.c_int(1)
        L.check(lib.vexb_dspmat_halo_connected(A.parts[k], C.byref(c)))
        assert c.value == 0
    # the product itself takes the copy path
    x = vx.vector(ctx2, full_mantissa(rng, n))
    ya, yd = vx.vector(ctx2, n), vx.vector(ctx2, n)
    A.apply(x, ya); D.apply(x, yd)
    assert_same(ya.read(), yd.read(), "apply over copies")


def test_fused_dot_is_composed(ctx1, params):
    A, D, n, rng = hell_pair(ctx1)
    lib, k = L.lib(), ctx1.local[0]
    x = vx.vector(ctx1, full_mantissa(rng, n))
    ya, yd = vx.vector(ctx1, n), vx.vector(ctx1, n)
    out = DeviceScalar(ctx1)
    code = lib.vexb_dspmat_apply_dot(1, ctx1._arr(A.parts), ctx1._arr(ctx1.streams), ctx1._arr(x.bufs), ctx1._arr(ya.bufs),
                                     1.0, 0, ctx1._arr(x.bufs), ctx1._arr(out.bufs), None)
    assert code == L.ERR_UNSUPPORTED
    assert A.apply_dot(x, ya, out) is False
    D.apply(x, yd)
    assert_same(ya.read(), yd.read(), "y")
    ref = DeviceScalar(ctx1)
    Reductor(ctx1, np.float64, L.SUM).device(x * yd, ref)
    assert_same(np.array([out.get()]), np.array([ref.get()]), "(x, y)")


@pytest.mark.parametrize("kernel", [0, 1, 2, 5, 6])
def test_other_csr_kernels_unsupported(ctx1, params, kernel):
    rng = np.random.default_rng(20)
    row, col, val = from_lengths(rng.integers(0, 20, 3000), 3000, rng)
    A = vx.SpMat(ctx1, 3000, 3000, row, col, val, vx.FMT_CSR | F32)
    x, y = vx.vector(ctx1, np.ones(3000)), vx.vector(ctx1, 3000)
    params("spmv.kernel", kernel)
    with pytest.raises(vx.VexbError) as e:
        A.apply(x, y)
    assert e.value.code == L.ERR_UNSUPPORTED


# ------------------------------------------------------------------------------------------------ 4. C++ front end

@pytest.mark.parametrize("parts", ["1", "2"])
def test_cpp_float_values(built, parts):
    """tests/cpp/test_spmat_f32_values.cpp: Y = A*X, Y -= 2*(A*X), Y = X + A*X and make_inline against SpMat<double> of
    the rounded values, exactly."""
    import os
    import subprocess
    from pathlib import Path
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = Path(__file__).resolve().parent / "cpp" / "bin" / "test_spmat_f32_values"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts),
                       timeout=300)
    print(r.stdout[-3000:]); print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"status {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
