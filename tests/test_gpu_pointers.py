"""vex::raw_pointer on the GPU, bit for bit against numpy, with the interpreter (eval.force_interp = 1, eval.jit = 0) and
the NVRTC kernel (eval.jit = 1) giving the same bits in the same run: neighbour access with clamped ends for all six
types and sizes around the grid's chunks, a gather through an index vector, a small table, a guarded (p + i)[-1] and
reads outside the vector (0),
compound assignment, vex::tie over pointer expressions, temporaries of loads, reductions, the N-body user function, and
a rotation through a pointer into the target."""
import numpy as np
import pytest

import vexcl_b200 as vx
from vexcl_b200 import _lib as L

pytestmark = pytest.mark.gpu

ALL = [np.float64, np.float32, np.int32, np.uint32, np.int64, np.uint64]
SIZES = [1, 255, 1023, 1024, 1025, 4097, 2**20 + 3]
MODES = {"interp": {"eval.force_interp": 1, "eval.jit": 0}, "jit": {"eval.jit": 1}}


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({8: np.uint64, 4: np.uint32}[a.dtype.itemsize])


def same(got, want, what=""):
    g, w = bits(np.asarray(got)), bits(np.asarray(want))
    assert g.shape == w.shape and np.array_equal(g, w), f"{what}: {np.count_nonzero(g != w)} of {g.size} differ"


def in_modes(fn):
    """fn() under each mode; every result is returned (the caller checks they agree)."""
    out = {}
    for name, prm in MODES.items():
        for k, v in prm.items():
            vx.set_param(k, v)
        try:
            out[name] = fn()
        finally:
            vx.set_param("eval.force_interp", 0)
            vx.set_param("eval.jit", 2)
    return out


def values(rng, n, dt):
    if np.dtype(dt).kind == "f":
        return (rng.random(n) + 0.25).astype(dt)
    return rng.integers(1, 1000, n).astype(dt)


def stencil_ref(X):
    n = X.size
    i = np.arange(n)
    left, right = np.where(i > 0, i - 1, i), np.where(i + 1 < n, i + 1, i)
    return (X.dtype.type(2) * X - X[left] - X[right]).astype(X.dtype)      # integers wrap, as on the device


@pytest.mark.parametrize("dt", ALL, ids=lambda d: np.dtype(d).name)
def test_neighbours_with_clamped_ends(ctx1, dt):
    rng = np.random.default_rng(1)
    for n in SIZES:
        X = values(rng, n, dt)
        x, y = vx.vector(ctx1, X), vx.vector(ctx1, n, dt)
        p, i = vx.raw_pointer(x), vx.ElementIndex()
        left = vx.if_else(i > 0, i - 1, i)
        right = vx.if_else(i + 1 < n, i + 1, i)
        def run():
            y.assign(2 * p[i] - p[left] - p[right])
            return y.read()
        r = in_modes(run)
        want = stencil_ref(X)
        same(r["interp"], want, f"interp n={n}")
        same(r["jit"], want, f"jit n={n}")


def test_gather_table_and_guarded_previous(ctx1):
    rng = np.random.default_rng(2)
    n = 100003
    X = values(rng, n, np.float64)
    IDX = rng.integers(0, n, n).astype(np.int32)
    T = np.array([1.5, -2.0, 3.25, 7.0])
    x, idx, t = vx.vector(ctx1, X), vx.vector(ctx1, IDX), vx.vector(ctx1, T)
    y = vx.vector(ctx1, n)
    p, q, i = vx.raw_pointer(x), vx.raw_pointer(t), vx.ElementIndex()
    def run():
        y.assign(p[idx]); a = y.read()
        y.assign(q[i % 4]); b = y.read()
        y.assign(vx.if_else(i > 0, (p + i)[-1], -1.0)); c = y.read()
        y.assign(vx.deref(p + idx) * 2.0 + vx.deref(q)); d = y.read()
        y.assign(p[i + 5] + (p - 3)[i]); e = y.read()          # reads outside x give 0
        return a, b, c, d, e
    r = in_modes(run)
    for got in r.values():
        same(got[0], X[IDX], "gather")
        same(got[1], T[np.arange(n) % 4], "table")
        same(got[2], np.concatenate([[-1.0], X[:-1]]), "guarded previous")
        same(got[3], X[IDX] * 2.0 + T[0], "deref")
        same(got[4], np.concatenate([X[5:], np.zeros(5)]) + np.concatenate([np.zeros(3), X[:-3]]), "outside")


def test_compound_assignment_tie_and_temporaries(ctx1):
    rng = np.random.default_rng(3)
    n = 70001
    X, Y0 = values(rng, n, np.float64), values(rng, n, np.float64)
    J = rng.integers(0, 1000, n).astype(np.int32)
    x, j = vx.vector(ctx1, X), vx.vector(ctx1, J)
    p, i = vx.raw_pointer(x), vx.ElementIndex()
    def run():
        y = vx.vector(ctx1, Y0)
        y += p[j] * 3.0
        a = y.read()
        y /= (p + 5)[j]
        b = y.read()
        u, v = vx.vector(ctx1, Y0), vx.vector(ctx1, Y0)
        vx.assign_multi([u, v], [p[j] + u, (p + 1)[j] - v])
        c = (u.read(), v.read())
        t = vx.make_temp(1, p[j] * 2.0)
        u.assign(t * t + t)
        d = u.read()
        return a, b, c, d
    r = in_modes(run)
    A = Y0 + X[J] * 3.0
    for got in r.values():
        same(got[0], A, "+=")
        same(got[1], A / X[J + 5], "/=")
        same(got[2][0], X[J] + Y0, "tie 0")
        same(got[2][1], X[J + 1] - Y0, "tie 1")
        T = X[J] * 2.0
        same(got[3], T * T + T, "temporary")


def test_guard_region_past_the_target_is_untouched(ctx1):
    rng = np.random.default_rng(4)
    n, guard = 4097, 64
    X = values(rng, n + guard, np.float64)
    x = vx.vector(ctx1, X)
    G = np.full(n + guard, 12345.0)
    big = vx.vector(ctx1, G)
    y = vx.vector.__new__(vx.vector)                           # the first n elements of `big`, as a vector of its own
    y.__dict__.update(big.__dict__)
    y.n, y.part = n, vx.partition(n, 1)
    y.bufs = dict(big.bufs)
    p, i = vx.raw_pointer(x), vx.ElementIndex()
    def run():
        y.assign(p[i + guard])
        return big.read()
    try:
        r = in_modes(run)
    finally:
        y.bufs = {}                                             # owned by `big`
    for got in r.values():
        same(got[:n], X[guard:guard + n], "head")
        same(got[n:], G[n:], "guard")


def test_reductions_have_the_bits_of_the_temporary(ctx1):
    rng = np.random.default_rng(5)
    n = 300007
    X = values(rng, n, np.float64)
    J = rng.integers(0, n, n).astype(np.int32)
    x, j = vx.vector(ctx1, X), vx.vector(ctx1, J)
    p = vx.raw_pointer(x)
    kinds = [L.SUM, L.SUM_KAHAN, L.MIN, L.MAX, [L.SUM, L.MAX, L.MIN, L.SUM_KAHAN]]
    def run():
        tmp = vx.vector(ctx1, n)
        tmp.assign(x * p[j])
        out = []
        for kind in kinds:
            R = vx.Reductor(ctx1, np.float64, kind)
            out.append((R(x * p[j]), R(tmp)))
        return out
    for name, got in in_modes(run).items():
        for kind, (a, b) in zip(kinds, got):
            same(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), f"{name} {kind}")


def test_nbody_user_function(ctx1):
    n = 2048
    rng = np.random.default_rng(6)
    X = rng.random(n)
    x, y = vx.vector(ctx1, X), vx.vector(ctx1, n)
    nbody = vx.UserFunction(np.float64, "nbody", [(np.uint64, "n"), (np.uint64, "j"), (vx.ptr(np.float64), "x")],
                            "double sum = 0; for (size_t i = 0; i < n; ++i) if (i != j) sum += x[i]; return sum;")
    y.assign(nbody(np.uint64(n), vx.ElementIndex(), vx.raw_pointer(x)))
    want = np.zeros(n)                                          # the body's loop, in its order, for every j at once
    every = np.arange(n)
    for k in range(n):
        want[every != k] += X[k]
    same(y.read(), want, "nbody")


def test_rotation_through_a_pointer_into_the_target(ctx1):
    n = 1000003
    X = np.arange(n, dtype=np.float64)
    def run():
        x = vx.vector(ctx1, X)
        p, i = vx.raw_pointer(x), vx.ElementIndex()
        x.assign(p[(i + 1) % n])
        a = x.read()
        u = vx.vector(ctx1, X)
        q = vx.raw_pointer(u)
        vx.assign_multi([x, u], [q[(i + n - 1) % n], q[i] * 2.0])
        return a, x.read(), u.read()
    for got in in_modes(run).values():
        same(got[0], np.roll(X, -1), "rotation")
        same(got[1], np.roll(X, 1), "tie rotation")
        same(got[2], X * 2.0, "tie doubled")
