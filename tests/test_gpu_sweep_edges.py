"""The streaming kernels at their vector and grid edges.

sweep_kernel and reduce_sweep_kernel move E = 4 doubles or 8 floats per vector access, U = 2 vectors per thread and 256
threads per block, loop over the grid when it is capped (sweep.persistent, reduce.blocks_per_sm), and handle the last
n mod E elements in a scalar tail; cg_update_r_kernel and cg_update_xp_kernel have the same tail.  Every result is
compared with numpy doing the same operations in the same precision:
  * elementwise sweeps (all 19 spellings match_shape recognises) bit for bit, including that nothing past n is written;
  * reductions on integer-valued data, where SUM and SUM_KAHAN are exact in any order and MIN / MAX / MINMAX are exact,
    with the extreme at index 0, at n - 1 and in the tail;
  * the CG updates with alpha and beta powers of two, so that r, x, p and rho' = (r, r) are exact.
Lengths: 1, E - 1, E, E + 1, 512 E - 1, 512 E, 512 E + 1 (one block's worth of vectors), 3 * 512 E + E - 1 and longer
vectors whose grid-stride loops turn more than once."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
import vexcl_b200 as vx
from vexcl_b200 import _lib as L
from vexcl_b200.api import DeviceScalar, Scalar, _Lowering, wrap

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]


def lanes(dtype):
    return 32 // np.dtype(dtype).itemsize                   # E: elements per 32-byte vector access


def lengths(dtype):
    E = lanes(dtype)
    return [1, E - 1, E, E + 1, 512 * E - 1, 512 * E, 512 * E + 1, 3 * 512 * E + E - 1, 1_000_003]


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


DEFAULTS = {"sweep.persistent": 0, "sweep.blocks_per_sm": 8, "reduce.blocks_per_sm": 8, "eval.force_interp": 0}


class params:
    """Set library parameters (sweep__persistent=1 sets sweep.persistent) for the duration of a with-block, then put
    back their defaults."""
    def __init__(self, **kw):
        self.kw = {k.replace("__", "."): v for k, v in kw.items()}

    def __enter__(self):
        for k, v in self.kw.items():
            vx.set_param(k, v)

    def __exit__(self, *exc):
        for k in self.kw:
            vx.set_param(k, DEFAULTS[k])


# ------------------------------------------------------------------------------------------------ 1. spellings

def spellings():
    """(shape, expression over vectors b, c, d and scalars s, t, numpy form): the 19 spellings of match_shape."""
    return [
        ("copy", lambda b, c, d, s, t: b, lambda B, C_, D, S, T: B),
        ("fill", lambda b, c, d, s, t: s, lambda B, C_, D, S, T: np.full_like(B, S)),
        ("add", lambda b, c, d, s, t: b + c, lambda B, C_, D, S, T: B + C_),
        ("sub", lambda b, c, d, s, t: b - c, lambda B, C_, D, S, T: B - C_),
        ("mul", lambda b, c, d, s, t: b * c, lambda B, C_, D, S, T: B * C_),
        ("div", lambda b, c, d, s, t: b / c, lambda B, C_, D, S, T: B / C_),
        ("sqr", lambda b, c, d, s, t: b * b, lambda B, C_, D, S, T: B * B),
        ("scale", lambda b, c, d, s, t: s * b, lambda B, C_, D, S, T: S * B),
        ("scale", lambda b, c, d, s, t: b * s, lambda B, C_, D, S, T: B * S),
        ("muladd", lambda b, c, d, s, t: b + c * d, lambda B, C_, D, S, T: B + C_ * D),
        ("muladd", lambda b, c, d, s, t: c * d + b, lambda B, C_, D, S, T: C_ * D + B),
        ("axpy", lambda b, c, d, s, t: s * b + c, lambda B, C_, D, S, T: S * B + C_),
        ("axpy", lambda b, c, d, s, t: b * s + c, lambda B, C_, D, S, T: B * S + C_),
        ("xpay", lambda b, c, d, s, t: b + s * c, lambda B, C_, D, S, T: B + S * C_),
        ("xpay", lambda b, c, d, s, t: b + c * s, lambda B, C_, D, S, T: B + C_ * S),
        ("xmay", lambda b, c, d, s, t: b - s * c, lambda B, C_, D, S, T: B - S * C_),
        ("xmay", lambda b, c, d, s, t: b - c * s, lambda B, C_, D, S, T: B - C_ * S),
        ("axpby", lambda b, c, d, s, t: s * b + t * c, lambda B, C_, D, S, T: S * B + T * C_),
        ("absdiff", lambda b, c, d, s, t: vx.fabs(b - c), lambda B, C_, D, S, T: np.abs(B - C_)),
    ]


def test_there_are_19_spellings():
    assert len(spellings()) == 19


def real_data(seed, n, dtype):
    """Non-integer values: products and quotients round, so the check sees the rounding of every operation."""
    return ((oracle.uniform_real(seed, n) - 0.5) * 8.0 + 0.25).astype(dtype)


@pytest.mark.parametrize("persistent", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_spelling_at_vector_edges(ctx1, dtype, persistent):
    """persistent = 1 also caps the grid at one block per SM, so at 1 000 003 elements the grid-stride loop turns
    several times."""
    typ = np.dtype(dtype).type
    S, T = typ(0.7109375), typ(-1.3)
    ops = {L.SET: lambda old, new: new, L.ADD: lambda old, new: old + new, L.SUB: lambda old, new: old - new}
    with params(sweep__persistent=persistent, sweep__blocks_per_sm=1 if persistent else 8):
        for n in lengths(dtype):
            B, Cc, D, A0 = (real_data(seed + n % 1000, n, dtype) for seed in (1, 2, 3, 4))
            b, c, d, a = vx.vector(ctx1, B), vx.vector(ctx1, Cc), vx.vector(ctx1, D), vx.vector(ctx1, A0)
            for scal in ("host", "device"):
                if scal == "host":
                    s, t = Scalar(S), Scalar(T)             # typed terminals: a numpy scalar on the left would take over
                else:
                    s, t = DeviceScalar(ctx1, dtype, S), DeviceScalar(ctx1, dtype, T)
                for shape, expr, ref in spellings():
                    rhs = expr(b, c, d, s, t)
                    want_rhs = ref(B, Cc, D, S, T)
                    assert want_rhs.dtype == dtype
                    for op, comb in ops.items():
                        assert a.eval_path(op, rhs) == f"sweep:{shape}", (shape, op)
                        a.write(A0)
                        a._assign(op, rhs)
                        want = comb(A0, want_rhs)
                        got = a.read()
                        assert np.array_equal(got, want), (n, scal, shape, op, np.nonzero(got != want)[0][:4])
            # in-place forms: the left-hand side is also an operand
            a.write(A0)
            a.assign(a * a)
            assert np.array_equal(a.read(), A0 * A0)
            a.write(A0)
            a.assign(a - Scalar(S) * b)
            assert np.array_equal(a.read(), A0 - S * B)
            a.write(A0)
            a -= a * b
            assert np.array_equal(a.read(), A0 - A0 * B)


def raw_eval(ctx, lhs, expr, op, n):
    """vexb_eval over the first n elements of lhs (which may be longer)."""
    low = _Lowering(ctx.local[0], 0)
    low.lower(wrap(expr))
    L.check(L.lib().vexb_eval(0, ctx.streams[0], lhs.bufs[0], lhs.dtype, op, C.byref(low.e), n, 0))


@pytest.mark.parametrize("interp", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES)
def test_nothing_is_written_past_n(ctx1, dtype, interp):
    typ = np.dtype(dtype).type
    pad = 3 * lanes(dtype) + 5
    sentinel = typ(-12345.0)
    with params(eval__force_interp=interp):
        for n in lengths(dtype):
            B, Cc = real_data(5, n + pad, dtype), real_data(6, n + pad, dtype)
            b, c = vx.vector(ctx1, B), vx.vector(ctx1, Cc)
            a = vx.vector(ctx1, np.full(n + pad, sentinel, dtype))
            for expr, ref in ((b + c * typ(0.5), B + Cc * typ(0.5)), (b * b, B * B), (typ(2.0), np.full(n + pad, typ(2.0)))):
                path = a.eval_path(L.SET, expr)
                assert path == "interp" if interp else path.startswith("sweep:")
                for op in (L.SET, L.ADD, L.SUB):
                    a.write(np.full(n + pad, sentinel, dtype))
                    raw_eval(ctx1, a, expr, op, n)
                    got = a.read()
                    base = np.full(n, sentinel, dtype)
                    want = ref[:n] if op == L.SET else base + ref[:n] if op == L.ADD else base - ref[:n]
                    assert np.array_equal(got[:n], want), (n, op)
                    assert np.all(got[n:] == sentinel), (n, op, np.nonzero(got[n:] != sentinel)[0][:4])


# ------------------------------------------------------------------------------------------------ 2. reductions

REDUCE_SHAPES = {
    "copy": lambda x, y: x, "mul": lambda x, y: x * y, "sqr": lambda x, y: x * x,
    "sub": lambda x, y: x - y, "absdiff": lambda x, y: vx.fabs(x - y),
}
REDUCE_REF = {
    "copy": lambda X, Y: X, "mul": lambda X, Y: X * Y, "sqr": lambda X, Y: X * X,
    "sub": lambda X, Y: X - Y, "absdiff": lambda X, Y: np.abs(X - Y),
}


def reduce_inputs(shape, n, seed):
    """Integer-valued inputs whose terms are never 0 (a dropped or repeated element changes the sum) and at most 2 in
    magnitude on average, so float32 partial sums stay below 2^24 at the longest length."""
    rng = np.random.default_rng(seed)
    X = rng.choice([1.0, 2.0], n)
    Y = rng.choice([1.0, -1.0], n) if shape == "mul" else rng.choice([0.0, 3.0], n)
    if shape == "sqr":
        X = rng.choice([1.0, -1.0], n)
    return X, Y


def place_extremes(shape, X, Y, hi, lo=None):
    """A unique largest term at index hi and (lo not None) a unique smallest at index lo: the other terms lie in
    [-2, 2] (in [1, 2] for sqr and absdiff)."""
    X, Y = X.copy(), Y.copy()
    X[hi] = 50.0
    Y[hi] = 1.0 if shape == "mul" else 0.0
    if lo is not None:
        X[lo] = 0.0 if shape in ("sqr", "absdiff") else -50.0
        Y[lo] = 1.0 if shape == "mul" else 0.0
    return X, Y


def reduce_lengths(dtype, bps):
    E = lanes(dtype)
    return [1, E - 1, E, E + 1, 512 * E - 1, 512 * E, 512 * E + 1, 3 * 512 * E + E - 1,
            sms() * bps * 512 * E + 512 * E + E - 1]


def reduce_ops(ctx, dtype, expr):
    out = {op: vx.Reductor(ctx, dtype, op)(expr) for op in (L.SUM, L.SUM_KAHAN, L.MAX, L.MIN)}
    out[L.MINMAX] = vx.Reductor(ctx, dtype, L.MINMAX)(expr)
    return out


@pytest.mark.parametrize("bps", [1, 8, 16])
@pytest.mark.parametrize("dtype", DTYPES)
def test_reduction_sweeps(ctx1, dtype, bps):
    E = lanes(dtype)
    with params(reduce__blocks_per_sm=bps):
        for n in reduce_lengths(dtype, bps):
            for k, (shape, expr) in enumerate(REDUCE_SHAPES.items()):
                X, Y = reduce_inputs(shape, n, seed=n % 1000 + k)
                F = REDUCE_REF[shape](X, Y)
                assert np.sum(np.abs(F)) < 2 ** 24
                x, y = vx.vector(ctx1, X.astype(dtype)), vx.vector(ctx1, Y.astype(dtype))
                assert x.eval_path(L.SET, expr(x, y)) == f"sweep:{shape}"
                total = int(F.sum())
                got = reduce_ops(ctx1, dtype, expr(x, y))
                assert got[L.SUM] == total and got[L.SUM_KAHAN] == total, (n, shape, got[L.SUM], total)
                with params(eval__force_interp=1):
                    slow = reduce_ops(ctx1, dtype, expr(x, y))
                assert slow == got, (n, shape)
                # extremes at index 0, at n - 1 and in the tail (the first of the last n mod E elements)
                places = sorted({0, n - 1} | ({n - n % E} if n % E > 1 else set()))
                for j, hi in enumerate(places):
                    lo = places[(j + 1) % len(places)]
                    Xe, Ye = place_extremes(shape, X, Y, hi, lo if lo != hi else None)
                    Fe = REDUCE_REF[shape](Xe, Ye)
                    if n > 1:
                        assert np.count_nonzero(Fe == Fe.max()) == 1 and Fe.argmax() == hi
                        assert np.count_nonzero(Fe == Fe.min()) == 1 and Fe.argmin() == lo
                    x.write(Xe.astype(dtype)); y.write(Ye.astype(dtype))
                    r = reduce_ops(ctx1, dtype, expr(x, y))
                    assert r[L.MAX] == Fe.max() and r[L.MIN] == Fe.min(), (n, shape, hi, lo)
                    assert r[L.MINMAX] == (Fe.min(), Fe.max()), (n, shape, hi, lo)
                    with params(eval__force_interp=1):
                        assert reduce_ops(ctx1, dtype, expr(x, y)) == r, (n, shape, hi, lo)


# ------------------------------------------------------------------------------------------------ 3. CG updates

@pytest.mark.parametrize("bps", [1, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_cg_update_kernels(ctx1, dtype, bps):
    """r -= alpha q with alpha = rho / pq = 1/4 and rho' = (r, r), then x += alpha p, p = r + beta p with beta =
    rho' / rho = 1/2: exact on integer-valued vectors.  The vectors are longer than n: nothing past n may change."""
    typ = np.dtype(dtype).type
    lib, vt = L.lib(), (L.F64 if dtype == np.float64 else L.F32)
    ws, _ = ctx1.workspace(0)
    pad = 11
    E = lanes(dtype)
    ns = [1, 7, 1001, 100003, sms() * bps * 512 * E + 3 * E + 3]
    with params(reduce__blocks_per_sm=bps):
        for n in ns:
            assert n % 8 not in (0, 4)
            rng = np.random.default_rng(n)
            R = rng.integers(-2, 3, n + pad).astype(dtype)
            Q = (4 * rng.integers(-1, 2, n + pad)).astype(dtype)
            Xh = rng.integers(-3, 4, n + pad).astype(dtype)
            P = rng.integers(-3, 4, n + pad).astype(dtype)
            r, q, x, p = (vx.vector(ctx1, h) for h in (R, Q, Xh, P))
            rho, pq, rho_new = DeviceScalar(ctx1, dtype, 2.0), DeviceScalar(ctx1, dtype, 8.0), DeviceScalar(ctx1, dtype, 0.0)
            L.check(lib.vexb_cg_update_r(0, ctx1.streams[0], vt, n, r.bufs[0], q.bufs[0], rho.bufs[0], pq.bufs[0],
                                         rho_new.bufs[0], ws, None))
            alpha = typ(2.0) / typ(8.0)
            Rn = R.copy()
            Rn[:n] = R[:n] - alpha * Q[:n]
            assert np.array_equal(r.read(), Rn), n
            assert rho_new.get() == np.sum(Rn[:n].astype(np.float64) ** 2)
            assert np.sum(Rn[:n].astype(np.float64) ** 2) < 2 ** 24
            rho_new.set(1.0)                                  # beta = 1/2
            L.check(lib.vexb_cg_update_xp(0, ctx1.streams[0], vt, n, x.bufs[0], p.bufs[0], r.bufs[0], rho.bufs[0],
                                          pq.bufs[0], rho_new.bufs[0]))
            Xn, Pn = Xh.copy(), P.copy()
            Xn[:n] = Xh[:n] + alpha * P[:n]
            Pn[:n] = Rn[:n] + typ(0.5) * P[:n]
            assert np.array_equal(x.read(), Xn) and np.array_equal(p.read(), Pn), n


def spd_laplacian(n):
    """7-point Laplacian on an n^3 grid with the Dirichlet neighbours dropped: symmetric positive definite."""
    idx = np.arange(n ** 3).reshape(n, n, n)
    rows, cols, vals = [idx.ravel()], [idx.ravel()], [np.full(n ** 3, 6.0)]
    for ax in range(3):
        for sh in (-1, 1):
            src = [slice(None)] * 3; dst = [slice(None)] * 3
            src[ax] = slice(1, None) if sh < 0 else slice(None, -1)
            dst[ax] = slice(None, -1) if sh < 0 else slice(1, None)
            rows.append(idx[tuple(src)].ravel()); cols.append(idx[tuple(dst)].ravel()); vals.append(np.full(rows[-1].size, -1.0))
    r, c, v = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
    order = np.lexsort((c, r))
    N = n ** 3
    row = np.concatenate([[0], np.cumsum(np.bincount(r[order], minlength=N))]).astype(np.int64)
    return row, c[order].astype(np.int64), v[order], N


def test_fused_cg_on_a_size_not_a_multiple_of_8(ctx1):
    from vexcl_b200.solvers import CGFused
    row, col, val, N = spd_laplacian(17)
    assert N % 8 not in (0, 4)
    b = oracle.uniform_real(3, N)
    iters = 20
    xo, hist_o = oracle.cg(row, col, val, b, np.zeros(N), iters)
    A = vx.SpMat(ctx1, N, N, row, col, val)
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
