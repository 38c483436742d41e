"""The fused product + dot (SpMat.apply_dot, vexb_dspmat_apply_dot) and CGFused on sliced-ELL strips (VEXB_FMT_SELL):
dist_apply_kernel with a sliced-ELL interior body, one launch for the product and the dot partials plus dot_fold_kernel.

Everything is compared on bits (integer views), in float64 and float32:
  * y against A.apply (sell_kernel) on the same strip;
  * the dot against tests/sell_dot_order.py's restatement of the order of additions (lane terms in storage order, the
    block epilogue, dot_fold_kernel), from the y the product wrote;
  * CGFused's every rho' and final x against a CPU simulation of its four launches, stream-launched and graph-replayed.
Launches are counted with vx.launch_count(), writes past n with guard elements.

Several slots on ONE device never get the peer-memory halo (vexb_dspmat_halo_connect_local needs distinct devices), so
there the sliced-ELL interior keeps the copies path and apply_dot is composed; the one-launch product and the fused dot
across GPUs run only where at least two devices exist."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import reduce_order as ro
import sell_dot_order as so
import vexcl_b200 as vx
from test_gpu_sell_fused import assert_same, matrix, values
from vexcl_b200 import _lib as L
from vexcl_b200 import gen
from vexcl_b200.api import DeviceScalar
from vexcl_b200.solvers import CGFused

pytestmark = pytest.mark.gpu

DEFAULTS = {"spmv.sell_sigma": 1024, "spmv.col16": 1, "dspmat.no_fused_dot": 0}
DTYPES = [np.float64, np.float32]
OPS = {"=": (1.0, False), "+=": (1.0, True), "-0.5+=": (-0.5, True)}


@pytest.fixture
def params(built):
    try:
        yield vx.set_param
    finally:
        for k, v in DEFAULTS.items():
            vx.set_param(k, v)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def build(ctx, n, mat, fmt=vx.FMT_SELL):
    A = vx.SpMat(ctx, n, n, *mat, fmt)
    assert A.info().loc.fmt == L.FMT_SELL
    return A


def check_apply_dot(ctx, A, row, sigma, dtype, rng, what):
    """Every op with dot_with = None and with a w vector: True, two launches, y = A.apply's bits, the dot = the
    restatement's bits."""
    n = A.n
    perm = so.sell_layout(row, sigma)
    X, W = values(rng, n, dtype), values(rng, n, dtype)
    x, w = vx.vector(ctx, X), vx.vector(ctx, W)
    d = DeviceScalar(ctx, dtype)
    for op, (alpha, append) in OPS.items():
        Y0 = values(rng, n, dtype)
        for dw, Wh in ((None, X), (w, W)):
            y, yr = vx.vector(ctx, Y0), vx.vector(ctx, Y0)
            ctx.finish()
            l0 = vx.launch_count()
            assert A.apply_dot(x, y, d, dot_with=dw, alpha=alpha, append=append), (what, op)
            assert vx.launch_count() - l0 == 2, (what, op)
            A.apply(x, yr, alpha, append)
            got = y.read()
            assert_same(got, yr.read(), f"{what} {op} y")
            assert_same(np.array([d.get()], dtype), np.array([so.fused_dot(Wh, got, perm)], dtype),
                        f"{what} {op} dot_with={'w' if dw is not None else 'x'}")


# ------------------------------------------------------------------------------------------------ one part

SIZES = lambda sigma: [1, 31, 32, 33, sigma - 1, sigma + 1, 8 * sigma + 17]


def some_entries(rng, n, dtype, spread):
    """matrix(), with one entry on the diagonal if the draw left the strip empty (an empty strip is not fused)."""
    row, col, val = matrix(rng, n, n, dtype, spread=spread)
    if row[-1] == 0:
        row, col, val = np.r_[0, np.ones(n, np.int64)], np.zeros(1, np.int64), values(rng, 1, dtype)
    return row, col, val


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("sigma", [256, 1024])
@pytest.mark.parametrize("cols", ["col16", "col32"])
def test_one_part_sizes(ctx1, params, cols, sigma, dtype):
    """Forced sliced ELL at the slice and window boundaries, 16-bit offsets (spmv.col16 = 1 on a banded matrix) and
    32-bit columns (spmv.col16 = 0)."""
    params("spmv.sell_sigma", sigma)
    for n in SIZES(sigma):
        rng = np.random.default_rng(n + sigma)
        mat = some_entries(rng, n, dtype, 300 if cols == "col16" else None)
        params("spmv.col16", 1 if cols == "col16" else 0)
        A = build(ctx1, n, mat)
        params("spmv.col16", 0 if cols == "col16" else 1)
        other = build(ctx1, n, mat).info().loc.device_bytes          # 16-bit offsets: two bytes less per slot
        assert (other > A.info().loc.device_bytes) == (cols == "col16")
        check_apply_dot(ctx1, A, mat[0], sigma, dtype, rng, (cols, sigma, n))


@pytest.mark.parametrize("dtype", DTYPES)
def test_auto_chosen_strip(ctx1, params, dtype):
    """VEXB_FMT_AUTO stores the irregular matrix as sliced ELL, and apply_dot fuses on it."""
    n = 5 * 1024 + 3
    row, col, val = gen.irregular_rows(n, 0, 32, seed=7)
    A = build(ctx1, n, (row, col, val.astype(dtype)), vx.FMT_AUTO)
    check_apply_dot(ctx1, A, row, 1024, dtype, np.random.default_rng(7), "auto")


@pytest.mark.parametrize("dtype", DTYPES)
def test_many_partials(ctx1, params, dtype):
    """1028 and 16 387 interior blocks: dot_fold_kernel's threads take more than one partial, and with more than 16 * 1024
    partials thread 0 starts a second batch."""
    for n in (8 * 32 * 1027 + 200, 8 * 32 * 16385 + 300):
        row, col, val = gen.irregular_rows(n, 0, 4, seed=n % 97)
        perm = so.sell_layout(row, 1024)
        assert so.interior_blocks(perm) in (1028, 16387)
        A = build(ctx1, n, (row, col, val.astype(dtype)))
        rng = np.random.default_rng(n)
        X, W = values(rng, n, dtype), values(rng, n, dtype)
        x, w, y, yr = vx.vector(ctx1, X), vx.vector(ctx1, W), vx.vector(ctx1, n, dtype), vx.vector(ctx1, n, dtype)
        d = DeviceScalar(ctx1, dtype)
        assert A.apply_dot(x, y, d, dot_with=w)
        A.apply(x, yr)
        got = y.read()
        assert_same(got, yr.read(), f"{n} y")
        assert_same(np.array([d.get()], dtype), np.array([so.fused_dot(W, got, perm)], dtype), f"{n} dot")


@pytest.mark.parametrize("dtype", DTYPES)
def test_empty_rows_and_empty_strip(ctx1, params, dtype):
    rng = np.random.default_rng(11)
    n = 3 * 1024 + 40
    row, col, val = matrix(rng, n, n, dtype)
    keep = np.ones(n, bool); keep[5:700] = False; keep[n - 70:] = False; keep[rng.random(n) < 0.3] = False
    sel = np.repeat(keep, np.diff(row))
    row2 = np.concatenate([[0], np.cumsum(np.diff(row) * keep)]).astype(np.int64)
    A = build(ctx1, n, (row2, col[sel], val[sel]))
    check_apply_dot(ctx1, A, row2, 1024, dtype, rng, "empty rows")
    # a strip without any entry keeps the composed path: y zeroed (=) or kept (+=), the dot by a reduction
    E = build(ctx1, n, matrix(rng, n, n, dtype, empty=True))
    X, Y0 = values(rng, n, dtype), values(rng, n, dtype)
    x, d = vx.vector(ctx1, X), DeviceScalar(ctx1, dtype)
    for alpha, append in OPS.values():
        y = vx.vector(ctx1, Y0)
        assert not E.apply_dot(x, y, d, alpha=alpha, append=append)
        want = Y0 if append else np.zeros(n, dtype)
        assert_same(y.read(), want, "empty strip y")
        ref = DeviceScalar(ctx1, dtype)
        vx.Reductor(ctx1, dtype, L.SUM).device(x * y, ref)
        assert_same(np.array([d.get()], dtype), np.array([ref.get()], dtype), "empty strip dot")


@pytest.mark.parametrize("dtype", DTYPES)
def test_nothing_is_written_past_n(ctx1, params, dtype):
    """y 64 elements longer than the strip, the tail holding a sentinel; the C ABI takes the buffers as they are."""
    rng = np.random.default_rng(12)
    n, G = 1024 + 7, 64
    row, col, val = matrix(rng, n, n, dtype)
    A = build(ctx1, n, (row, col, val))
    sentinel = dtype(-12345.5)
    Y0 = np.concatenate([values(rng, n, dtype), np.full(G, sentinel, dtype)])
    X = values(rng, n, dtype)
    x, y, d = vx.vector(ctx1, X), vx.vector(ctx1, Y0), DeviceScalar(ctx1, dtype)
    lib = L.lib()
    for alpha, append in OPS.values():
        y.write(Y0)
        L.check(lib.vexb_dspmat_apply_dot(1, ctx1._arr(A.parts), ctx1._arr(ctx1.streams), ctx1._arr(x.bufs), ctx1._arr(y.bufs),
                                          alpha, int(append), ctx1._arr(x.bufs), ctx1._arr(d.bufs), None))
        yr = vx.vector(ctx1, Y0[:n])
        A.apply(x, yr, alpha, append)
        got = y.read()
        assert_same(got[:n], yr.read(), "y")
        assert_same(got[n:], Y0[n:], "guard")
        assert_same(np.array([d.get()], dtype), np.array([so.fused_dot(X, got[:n], so.sell_layout(row, 1024))], dtype), "dot")


def test_switch_and_float_values(ctx1, params):
    """dspmat.no_fused_dot and float-valued strips keep the composition, with apply's y."""
    rng = np.random.default_rng(13)
    n = 2 * 1024 + 5
    mat = matrix(rng, n, n, np.float64)
    for A, switch in ((build(ctx1, n, mat), True), (build(ctx1, n, mat, vx.FMT_SELL | vx.FMT_VALUES_F32), False)):
        if switch:
            params("dspmat.no_fused_dot", 1)
        x, y, yr, d = vx.vector(ctx1, values(rng, n, np.float64)), vx.vector(ctx1, n), vx.vector(ctx1, n), DeviceScalar(ctx1)
        A._fused_dot = True
        assert not A.apply_dot(x, y, d)
        A.apply(x, yr)
        assert_same(y.read(), yr.read(), "composed y")
        params("dspmat.no_fused_dot", 0)


# ------------------------------------------------------------------------------------------------ several slots

@pytest.mark.parametrize("nparts", [2, 3])
def test_several_slots_on_one_device(built, params, nparts):
    """peer_halo=True on slots of one device: the halo cannot connect, the product keeps the copies path with its bits,
    and vexb_dspmat_apply_dot refuses; the interior strip is sliced ELL and the boundary rows are split off."""
    rng = np.random.default_rng(20 + nparts)
    n = 3 * 1024 + 50
    ctx = vx.Context([0] * nparts, peer_halo=True)
    ref = vx.Context([0] * nparts, peer_halo=False)
    mat = matrix(rng, n, n, np.float64, spread=40)          # banded: ghosts only near the part boundaries
    A, B = vx.SpMat(ctx, n, n, *mat, vx.FMT_SELL), vx.SpMat(ref, n, n, *mat, vx.FMT_SELL)
    assert not A.peer_halo
    for k in range(nparts):
        info = A.info(k)
        assert info.loc.fmt == L.FMT_SELL and info.n_ghost > 0 and info.rem_nnz > 0 and 0 < info.loc.nrows <= info.nrows
    X = values(rng, n, np.float64)
    Y0 = values(rng, n, np.float64)
    for alpha, append in OPS.values():
        ya, yb = vx.vector(ctx, Y0), vx.vector(ref, Y0)
        A.apply(vx.vector(ctx, X), ya, alpha, append)
        B.apply(vx.vector(ref, X), yb, alpha, append)
        assert_same(ya.read(), yb.read(), "copies path")
    x, y, d = vx.vector(ctx, X), vx.vector(ctx, n), DeviceScalar(ctx)
    code = L.lib().vexb_dspmat_apply_dot(nparts, ctx._arr(A.parts), ctx._arr(ctx.streams), ctx._arr(x.bufs), ctx._arr(y.bufs),
                                         1.0, 0, ctx._arr(x.bufs), ctx._arr(d.bufs), None)
    assert code == L.ERR_UNSUPPORTED


@pytest.mark.parametrize("nparts", [2, 3])
def test_peer_halo_across_gpus(built, params, nparts):
    """The one-launch product with a sliced-ELL interior and the fused dot across GPUs through the peer group."""
    if torch.cuda.device_count() < nparts:
        pytest.skip(f"the peer-memory halo and the peer group need {nparts} distinct devices")
    rng = np.random.default_rng(30 + nparts)
    n = 20 * 1024 + 50
    devs = list(range(nparts))
    ctx = vx.Context(devs, peer_halo=True, use_peer=True)
    ref = vx.Context(devs, peer_halo=False)
    mat = matrix(rng, n, n, np.float64, spread=40)
    A, B = vx.SpMat(ctx, n, n, *mat, vx.FMT_SELL), vx.SpMat(ref, n, n, *mat, vx.FMT_SELL)
    assert A.peer_halo
    for k in range(nparts):
        info = A.info(k)
        assert info.loc.fmt == L.FMT_SELL and info.n_ghost > 0 and info.rem_nnz > 0 and info.loc.nrows < info.nrows
    X, W, Y0 = (values(rng, n, np.float64) for _ in range(3))
    x, w = vx.vector(ctx, X), vx.vector(ctx, W)
    d = DeviceScalar(ctx)
    for alpha, append in OPS.values():
        ya, yb, yd = vx.vector(ctx, Y0), vx.vector(ref, Y0), vx.vector(ctx, Y0)
        ctx.finish()
        l0 = vx.launch_count()
        A.apply(x, ya, alpha, append)
        assert vx.launch_count() - l0 == nparts
        B.apply(vx.vector(ref, X), yb, alpha, append)
        assert_same(ya.read(), yb.read(), "peer halo against copies")
        ctx.finish()
        l0 = vx.launch_count()
        assert A.apply_dot(x, yd, d, dot_with=w, alpha=alpha, append=append)
        assert vx.launch_count() - l0 == 2 * nparts
        got = yd.read()
        assert_same(got, yb.read(), "apply_dot y")
        terms = W.astype(np.float64) * got
        assert abs(float(d.get()) - float(np.sum(terms))) <= (n + 64) * 2.0 ** -53 * float(np.sum(np.abs(terms)))
        vals = [d.get()]
        for k in ctx.local[1:]:
            h = np.empty(1)
            L.check(L.lib().vexb_d2h(ctx.devs[k], h.ctypes.data, d.bufs[k], 8, ctx.streams[k], 1))
            vals.append(h[0])
        assert_same(np.array(vals), np.full(nparts, vals[0]), "every GPU holds the same dot")


# ------------------------------------------------------------------------------------------------ CGFused

@pytest.mark.parametrize("n", [3001, 100_003])
def test_cg_fused(ctx1, params, n):
    """20 iterations on the irregular SPD matrix, which VEXB_FMT_AUTO stores as sliced ELL: four launches per iteration,
    every rho' and the final x equal to the simulation bit for bit, stream-launched and replayed as two alternating CUDA
    graphs; the history within 1e-8 of oracle.cg's."""
    iters, S = 20, sms()
    row, col, val = gen.irregular_spd(n, seed=n % 1000)
    b = oracle.uniform_real(5, n)
    A = vx.SpMat(ctx1, n, n, row, col, val)
    assert A.info().loc.fmt == L.FMT_SELL
    x_sim, hist_sim = so.cg_fused(row, col, val, b, iters, S, so.sell_layout(row, 1024))
    _, hist_o = oracle.cg(row, col, val, b, np.zeros(n), iters)
    assert np.allclose(hist_sim, hist_o, rtol=1e-8, atol=0)
    runs = {}
    for use_graph in (False, True):
        bv, xv = vx.vector(ctx1, b), vx.vector(ctx1, n)
        xv.assign(0.0)
        cg = CGFused(A, bv, xv)
        hist = []
        if use_graph:
            cg.capture()
            hist = [cg.rho2[1].get(), cg.rho2[0].get()]
        while len(hist) < iters:
            cg.run(1)
            hist.append(cg.residual2())
        ctx1.finish()
        assert cg.fused_product
        assert_same(np.array(hist), np.array(hist_sim), f"history, graph={use_graph}")
        runs[use_graph] = xv.read()
        assert_same(runs[use_graph], x_sim, f"x, graph={use_graph}")
    n0 = vx.launch_count()
    cg.step()
    assert vx.launch_count() - n0 == 4
