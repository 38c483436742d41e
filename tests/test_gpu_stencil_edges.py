"""The stencil kernels bit for bit at their tile, tap-chunk, halo and shared-memory boundaries.

The reference is tests/stencil_ref.py: `oracle/stencil.py::convolve` for the convolution over the whole vector (every
product and sum rounded in the vector's precision, taps in order, then alpha and y), its window restatement for one
call of the C ABI with caller-built halos, and the operator bodies restated in numpy.  Values are compared on their bits
(uint64 / uint32 views) in float64 and float32, with `=`, `+=`, `-=` and alpha = 0.5 with append.

Edges: full chunks of 8 taps against the 1..7-tap tail (widths 1-9, 15-17, 23-25, 64, centered at both ends and in the
middle); 1024-output tiles that clamp at one or both ends against `inside` tiles; one infinity in x, which may reach
exactly the outputs [p - rhalo, p + center] -- the only way to see a zero-weight padding tap, since 0 * inf is NaN; the
200 KB, 48 KB and 100 KB (pipe) shared-memory thresholds; the pipelined persistent kernel on one to eight turns; the
scalar store path for y off a 32-byte boundary, and nothing written outside [y, y + n); the generated operator kernel
at 256-output block edges with and without halos, up to its 4096-tap limit; VEX_STENCIL_OPERATOR through the C++ front
end (tests/cpp/test_stencil_operator.cpp) on one and two slices.
"""
import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle
import vexcl_b200 as vx
from vexcl_b200 import _lib as L
from vexcl_b200.api import _vdt
import stencil_ref as sr

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
UINT = {np.dtype(np.float64): np.uint64, np.dtype(np.float32): np.uint32}
THRESHOLDS = {np.float64: (11504, 11505, 2344, 3224), np.float32: (23544, 23545, 5240, 7160)}
CHUNK_WIDTHS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 23, 24, 25, 64]
TILE_NS = [1, 7, 8, 9, 1023, 1024, 1025, 2047, 2049, 3 * 1024 + 5]
# (name, alpha, append) as the front end calls vexb_stencil_apply for  y = x*S,  y += x*S,  y -= x*S,  y += 0.5*(x*S)
OPS = [("=", 1.0, False), ("+=", 1.0, True), ("-=", -1.0, True), ("+= 0.5", 0.5, True)]


@pytest.fixture(params=[1, 2, 3])
def anyctx(request, ctx1, ctx2, ctx3):
    return {1: ctx1, 2: ctx2, 3: ctx3}[request.param]


@pytest.fixture
def params():
    """vx.set_param for the stencil's parameters, back at their defaults afterwards."""
    defaults = {"stencil.kernel": 1, "stencil.blocks_per_sm": 0}
    try:
        yield vx.set_param
    finally:
        for k, v in defaults.items():
            vx.set_param(k, v)


def bits(a):
    a = np.asarray(a)
    return a.view(UINT[a.dtype])


def assert_bits(got, want, what=""):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, what
    bad = np.flatnonzero(bits(got) != bits(want))
    assert bad.size == 0, f"{what}: {bad.size} outputs differ, first at {bad[:8]}: {got[bad[:4]]} != {want[bad[:4]]}"


def assert_reach(got, want, p, center, rhalo, what=""):
    """x finite but for x[p]: outputs outside [p - rhalo, p + center] are finite and bit-exact, those inside match
    `want` (NaN positions compared, not NaN payloads)."""
    n = got.size
    inside = np.zeros(n, dtype=bool)
    inside[max(p - rhalo, 0):min(p + center, n - 1) + 1] = True
    assert np.all(np.isfinite(got[~inside])), f"{what}: non-finite outputs at {np.flatnonzero(~np.isfinite(got) & ~inside)[:8]}"
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN at {np.flatnonzero(np.isnan(got) != np.isnan(want))[:8]}"
    keep = ~np.isnan(want)
    assert_bits(got[keep], want[keep], what)


def apply_front_end(S, x, y, op):
    if op == "=":
        y.assign(x * S)
    elif op == "+=":
        y += S * x
    elif op == "-=":
        y -= x * S
    else:
        y += 0.5 * (x * S)


def check_ops(ctx, s, center, xh, ops=OPS, seed=0, reach=None):
    """Every op through vx.stencil against the whole vector's convolution; `reach`: the position of x's one infinity."""
    dt = xh.dtype
    n = xh.size
    S = vx.stencil(ctx, s, center, dtype=dt)
    x, y = vx.vector(ctx, xh), vx.vector(ctx, n, dtype=dt)
    acc = sr.convolve_slice(s, center, xh)                 # convolve's arithmetic, by shifted slices instead of gathers
    y0 = (oracle.uniform_real(seed + 1000, n) + 0.25).astype(dt)
    for name, alpha, append in ops:
        y.write(y0)
        apply_front_end(S, x, y, name)
        want = sr.finish(acc, alpha, y0, append)
        what = f"n={n} width={s.size} center={center} {dt.name} {name} parts={ctx.nparts}"
        if reach is None:
            assert_bits(y.read(), want, what)
        else:
            assert_reach(y.read(), want, reach, center, s.size - 1 - center, what)


def centers(width):
    return sorted({0, width // 2, width - 1})


def taps(width, dtype, seed=0):
    return (oracle.uniform_real(seed + width, width) + 0.125).astype(dtype)   # no zero tap: 0 * inf would hide a reach


# ---------------------------------------------------------------------------------------------- vx.stencil: shapes
@pytest.mark.parametrize("dtype", DTYPES)
def test_tap_chunks(anyctx, dtype):
    """Full chunks of 8 taps, the 1..7-tap tail, a tail of exactly 8 (widths 16, 24, 64) and the chunk after it."""
    n = 3 * 1024 + 5
    xh = oracle.uniform_real(7, n).astype(dtype)
    for width in CHUNK_WIDTHS:
        for c in centers(width):
            check_ops(anyctx, taps(width, dtype), c, xh, seed=width)


@pytest.mark.parametrize("dtype", DTYPES)
def test_tiles(anyctx, dtype):
    """Lengths around the 1024-output tile, windows clamped at both ends (n < width, n < center), and lengths whose
    first and last tiles clamp while the middle ones load directly."""
    for n in TILE_NS:
        xh = oracle.uniform_real(n, n).astype(dtype)
        for width in (1, 9, 24, 33):
            for c in centers(width):
                check_ops(anyctx, taps(width, dtype), c, xh, ops=(OPS[0], OPS[3]), seed=n)
    assert sr.tile_inside(1, 3 * 1024 + 5, 33, 16) and not sr.tile_inside(2, 3 * 1024 + 5, 33, 16)


@pytest.mark.parametrize("dtype", DTYPES)
def test_reach_of_one_infinity(anyctx, dtype):
    """One +-inf in x at the ends, next to tile boundaries and, over several slices, at distance rhalo and rhalo + 1
    past a slice's right edge and center and center + 1 before its left edge."""
    n = 3 * 1024 + 5
    base = oracle.uniform_real(11, n).astype(dtype)
    part = anyctx.partition(n)
    for width in (5, 21, 33):
        for c in centers(width):
            rh = width - 1 - c
            ps = {0, n - 1, 1023, 1024, 2048 + c, 2047 - rh}
            for e in part[1:-1]:
                ps |= {e - 1 + rh, e + rh, e - c, e - c - 1}
            for i, p in enumerate(sorted(q for q in ps if 0 <= q < n)):
                xh = base.copy()
                xh[p] = np.inf if i % 2 else -np.inf
                check_ops(anyctx, taps(width, dtype), c, xh, ops=(OPS[0], OPS[3]), reach=p)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("weights", [(1, 0, 1), (0, 1, 1), (1, 1, 0), (8, 1, 1)])
def test_short_and_empty_slices(built, dtype, weights):
    """Three slots whose slices are empty or shorter than the halos: the exchange pads with x[0] and x[n - 1]."""
    ctx = vx.Context([0, 0, 0], weights=weights)
    for n in (1, 17, 40, 70):
        xh = oracle.uniform_real(n + 3, n).astype(dtype)
        for width, c in ((41, 20), (41, 0), (41, 40), (9, 4)):
            check_ops(ctx, taps(width, dtype), c, xh, seed=n)


# -------------------------------------------------------------------------------------- shared-memory thresholds
@pytest.mark.parametrize("dtype", DTYPES)
def test_shared_memory_thresholds(ctx1, dtype):
    """The widest accepted width, the widths either side of 48 KB give the right bits; the first refused width raises
    VEXB_ERR_UNSUPPORTED before anything is launched and leaves y alone."""
    widest, refused, last48, _ = THRESHOLDS[dtype]
    assert sr.accepted(widest, dtype) and not sr.accepted(refused, dtype)
    assert not sr.attribute_path(last48, dtype) and sr.attribute_path(last48 + 1, dtype)
    for n, width in ((4099, widest), (1025, widest), (3000, last48), (3000, last48 + 1)):
        xh = oracle.uniform_real(width + n, n).astype(dtype)
        check_ops(ctx1, taps(width, dtype), width // 3, xh, ops=(OPS[0], OPS[3]))
    n = 1000
    S = vx.stencil(ctx1, taps(refused, dtype), refused // 2, dtype=dtype)
    x, y = vx.vector(ctx1, oracle.uniform_real(1, n).astype(dtype)), vx.vector(ctx1, np.full(n, 3.0, dtype=dtype))
    ctx1.finish()
    before = vx.launch_count()
    with pytest.raises(L.VexbError) as e:
        S.apply(x, y)
    assert e.value.code == L.ERR_UNSUPPORTED
    assert vx.launch_count() == before
    assert np.all(y.read() == 3.0)


# ------------------------------------------------------------------------------------------- the pipelined kernel
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("slots", [1, 2])
def test_pipelined_kernel(ctx1, ctx2, params, dtype, slots):
    """stencil.kernel = 0 with one resident block per SM: SMs * 1024 * k outputs and a ragged tail, so each block runs
    k or k + 1 tiles (first tile, both buffers, the last partial tile).  One infinity per vector, in a later turn."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = {1: ctx1, 2: ctx2}[slots]
    params("stencil.kernel", 0)
    params("stencil.blocks_per_sm", 1)
    for k in (1, 2, 8):
        n = sms * 1024 * k + 517
        base = oracle.uniform_real(k, n).astype(dtype)
        # two slots halve the tiles per call: at k = 1 each slice has fewer tiles than SMs and stays on stencil_kernel
        piped = [sr.uses_pipe(9, int(m), dtype, 0, 1, sms) for m in np.diff(ctx.partition(n))]
        assert all(piped) if slots == 1 or k > 1 else not any(piped)
        for width in (1, 8, 9, 33):
            c = width // 3
            p = n - 1024 * (k // 2) - 300
            xh = base.copy()
            xh[p] = np.inf
            check_ops(ctx, taps(width, dtype), c, xh, ops=(OPS[0], OPS[3]), seed=k, reach=p)


@pytest.mark.parametrize("dtype", DTYPES)
def test_pipe_window_limit(ctx1, params, dtype):
    """The last width whose two windows fit in 100 KB runs the pipe kernel, the next falls back to stencil_kernel:
    both with the right bits."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    lastpipe = THRESHOLDS[dtype][3]
    assert sr.pipe_fits(lastpipe, dtype) and not sr.pipe_fits(lastpipe + 1, dtype)
    params("stencil.kernel", 0)
    params("stencil.blocks_per_sm", 1)
    n = sms * 1024 + 5
    xh = oracle.uniform_real(13, n).astype(dtype)
    for width in (lastpipe, lastpipe + 1):
        assert sr.uses_pipe(width, n, dtype, 0, 1, sms) == (width == lastpipe)
        check_ops(ctx1, taps(width, dtype), width - 5, xh, ops=(OPS[0],))


# -------------------------------------------------------------------------------------------------- the C ABI
def _dev_array(ctx, host):
    """A device copy of `host` and its pointer; the caller keeps the vector, which frees the buffer when it goes."""
    v = vx.vector(ctx, host)
    return v, v.bufs[ctx.local[0]]


def _ptr(buf, elems, es):
    return C.c_void_p(buf.value + elems * es)


def _stencil_apply(ctx, dtype, sbuf, width, center, xbuf, n, left, right, ybuf, alpha, append):
    k = ctx.local[0]
    L.check(L.lib().vexb_stencil_apply(ctx.devs[k], ctx.streams[k], _vdt(np.dtype(dtype)), sbuf, width, center, xbuf, n,
                                       left, right, ybuf, float(alpha), int(append)))


@pytest.mark.parametrize("dtype", DTYPES)
def test_store_paths_and_guards(ctx1, dtype):
    """y one element off a 32-byte boundary takes the scalar stores, y one 32-byte chunk further stays on the vector
    stores: both give the aligned call's bits, and the sentinels around [y, y + n) keep theirs."""
    es, per, guard = np.dtype(dtype).itemsize, 32 // np.dtype(dtype).itemsize, 40
    for n in (1, 7, 8, 9, 1025, 3 * 1024 + 5):
        xh = oracle.uniform_real(n + 5, n).astype(dtype)
        xv, xbuf = _dev_array(ctx1, xh)
        y0 = (oracle.uniform_real(n + 6, n) + 1).astype(dtype)
        for width, c in ((9, 4), (24, 23), (17, 0)):
            s = taps(width, dtype)
            sv, sbuf = _dev_array(ctx1, s)
            acc = sr.convolve_slice(s, c, xh)
            for alpha, append in ((1.0, False), (0.5, True)):
                want = sr.finish(acc, alpha, y0, append)
                for off in (guard, guard + 1, guard + per):
                    host = np.full(n + 2 * guard + per, -7.25, dtype=dtype)
                    host[off:off + n] = y0
                    yv, ybuf = _dev_array(ctx1, host)
                    assert ybuf.value % 256 == 0
                    _stencil_apply(ctx1, dtype, sbuf, width, c, xbuf, n, None, None, _ptr(ybuf, off, es), alpha, append)
                    ctx1.finish()
                    got = yv.read()
                    what = f"n={n} width={width} center={c} off={off - guard} alpha={alpha}"
                    assert_bits(got[off:off + n], want, what)
                    assert np.all(got[:off] == -7.25) and np.all(got[off + n:] == -7.25), what


@pytest.mark.parametrize("dtype", DTYPES)
def test_caller_halos(ctx1, dtype):
    """Caller-built left and right halos of exactly `center` and `width - 1 - center` distinct values, each NULL in
    turn: a window position left of the slice reads left[center + j], one right of it right[min(j - n, rhalo - 1)]."""
    for n in (1, 5, 1024, 1025, 3 * 1024 + 5):
        xh = oracle.uniform_real(n + 9, n).astype(dtype)
        xv, xbuf = _dev_array(ctx1, xh)
        y0 = (oracle.uniform_real(n + 10, n) + 1).astype(dtype)
        yv, ybuf = _dev_array(ctx1, y0)
        for width, c in ((9, 3), (33, 0), (33, 32), (17, 8), (2, 1)):
            s = taps(width, dtype)
            sv, sbuf = _dev_array(ctx1, s)
            rh = width - 1 - c
            lh = (100.0 + np.arange(max(c, 1))).astype(dtype)             # distinct from x and from each other
            rhv = (-200.0 - np.arange(max(rh, 1))).astype(dtype)
            lv, lbuf = _dev_array(ctx1, lh)
            rv, rbuf = _dev_array(ctx1, rhv)
            for use_l, use_r in ((True, True), (True, False), (False, True), (False, False)):
                for alpha, append in ((1.0, False), (0.5, True)):
                    yv.write(y0)
                    _stencil_apply(ctx1, dtype, sbuf, width, c, xbuf, n, lbuf if use_l else None, rbuf if use_r else None,
                                   ybuf, alpha, append)
                    ctx1.finish()
                    want = sr.convolve_slice(s, c, xh, lh[:c] if use_l else None, rhv[:rh] if use_r else None, y0, alpha, append)
                    assert_bits(yv.read(), want, f"n={n} width={width} center={c} left={use_l} right={use_r} alpha={alpha}")


# --------------------------------------------------------------------------------------- user-defined operators
OPERATORS = [("second_difference", 3, 1), ("forward", 4, 0), ("backward", 4, 3), ("min_max", 3, 1),
             ("sum_squares", 257, 100), ("sum_squares", 4096, 1500)]


def _register(dtype, body, width, center):
    oid = C.c_int(-1)
    L.check(L.lib().vexb_stencil_operator_register(_vdt(np.dtype(dtype)), width, center,
                                                   sr.BODIES[body][0].encode(), C.byref(oid)))
    return oid.value


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("body,width,center", OPERATORS)
def test_stencil_operator(ctx1, dtype, body, width, center):
    """vexb_stencil_op at 256-output block edges, halos NULL and given, alpha = 1 and alpha = 0.5 with append."""
    oid = _register(dtype, body, width, center)
    k = ctx1.local[0]
    rh = width - 1 - center
    lh = (oracle.uniform_real(21, max(center, 1)) + 2).astype(dtype)
    rhv = (oracle.uniform_real(22, max(rh, 1)) - 3).astype(dtype)
    lv, lbuf = _dev_array(ctx1, lh)
    rv, rbuf = _dev_array(ctx1, rhv)
    for n in (1, 255, 256, 257, 511, 3 * 256 + 1):
        xh = (oracle.uniform_real(n + 30, n) - 0.5).astype(dtype)
        xv, xbuf = _dev_array(ctx1, xh)
        y0 = oracle.uniform_real(n + 31, n).astype(dtype)
        yv, ybuf = _dev_array(ctx1, y0)
        for halos in (False, True):
            for alpha, append in ((1.0, False), (0.5, True)):
                yv.write(y0)
                L.check(L.lib().vexb_stencil_operator_apply(ctx1.devs[k], ctx1.streams[k], oid, xbuf, n,
                                                            lbuf if halos else None, rbuf if halos else None, ybuf,
                                                            alpha, int(append)))
                ctx1.finish()
                want = sr.apply_operator(body, width, center, xh, lh[:center] if halos else None,
                                         rhv[:rh] if halos else None, y0, alpha, append)
                assert_bits(yv.read(), want, f"{body} width={width} n={n} halos={halos} alpha={alpha}")


def test_stencil_operator_registration(built):
    """An identical operator gets the id it already has; a different body, type or center a new one; width 4097 and
    a center outside the width are refused at registration."""
    a = _register(np.float64, "second_difference", 3, 1)
    assert _register(np.float64, "second_difference", 3, 1) == a
    assert len({a, _register(np.float32, "second_difference", 3, 1), _register(np.float64, "min_max", 3, 1)}) == 3
    lib, oid = L.lib(), C.c_int(-1)
    body = sr.BODIES["sum_squares"][0].encode()
    assert lib.vexb_stencil_operator_register(_vdt(np.dtype(np.float64)), 4097, 0, body, C.byref(oid)) == L.ERR_INVALID
    assert lib.vexb_stencil_operator_register(_vdt(np.dtype(np.float64)), 3, 3, body, C.byref(oid)) == L.ERR_INVALID
    assert _register(np.float64, "sum_squares", sr.OP_MAX_WIDTH, 0) >= 0


@pytest.mark.parametrize("parts", ["1", "2"])
def test_cpp_stencil_operator(built, parts):
    """tests/cpp/test_stencil_operator.cpp: exact VEX_STENCIL_OPERATOR cases, on two slices with halos padded past a
    one-element slice by detail::stencil_halos."""
    from vexcl_b200 import build
    build.build_cpp_tests()
    exe = Path(__file__).resolve().parent / "cpp" / "bin" / "test_stencil_operator"
    assert exe.exists(), f"{exe} was not built"
    r = subprocess.run([str(exe), "12345"], capture_output=True, text=True, env=dict(os.environ, VEXCL_TEST_PARTS=parts),
                       timeout=120)
    print(r.stdout[-3000:])
    print(r.stderr[-3000:])
    assert r.returncode == 0 and " 0 failures" in r.stdout, f"exit status {r.returncode}:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}"
