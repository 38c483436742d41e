"""vx.inclusive_scan / exclusive_scan / inclusive_scan_by_key / exclusive_scan_by_key / reduce_by_key on the GPU, bit
for bit against the numpy restatement of csrc/scan.cu's order of additions (tests/scan_order.py) and exact against
np.cumsum / np.add.reduceat for integers: every type, at the tile boundaries (tile = 4096), in place and out of place,
with zero, non-zero, -0.0 and NaN init, on one to three parts, and keys with runs across tile boundaries, NaN and
signed zeros."""
import numpy as np
import pytest

import scan_order as so

import vexcl_b200 as vx

pytestmark = pytest.mark.gpu

TILE = so.TILE
TYPES = [np.float64, np.float32, np.int32, np.uint32, np.int64, np.uint64]
SIZES = [0, 1, 2, TILE - 1, TILE, TILE + 1, 7 * TILE - 1, 7 * TILE + 1, 1100 * TILE + 1]


def same(got, want):
    """Equal bits, NaN payloads aside (the GPU's adds give the canonical NaN)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        return False
    if got.dtype.kind == "f":
        nan = np.isnan(want)
        return bool(np.array_equal(np.isnan(got), nan) and np.array_equal(so_bits(got[~nan]), so_bits(want[~nan])))
    return bool(np.array_equal(got, want))


def so_bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def values(t, n, rng):
    t = np.dtype(t)
    if t.kind == "f":
        return rng.standard_normal(n).astype(t)
    info = np.iinfo(t)
    return rng.integers(info.min, info.max, n, dtype=t, endpoint=True)


def inits(t):
    t = np.dtype(t)
    if t.kind == "f":
        return [0, 1.5, -0.0, np.nan]
    return [0, np.iinfo(t).max - 5]


@pytest.mark.parametrize("t", TYPES, ids=lambda t: np.dtype(t).name)
def test_scans(ctx1, t):
    rng = np.random.default_rng(TYPES.index(t))
    for n in SIZES:
        x = values(t, n, rng)
        for exclusive in (False, True):
            for init in (inits(t) if exclusive else [0, 3]):
                want = so.scan(x, exclusive, init)
                if np.dtype(t).kind in "iu" and n:
                    c = np.cumsum(x, dtype=t)
                    if exclusive:
                        with np.errstate(over="ignore"):
                            iv = np.asarray(init).astype(t)
                            c = np.concatenate([[iv], iv + c[:-1]]).astype(t)
                    assert np.array_equal(want, c)
                fn = vx.exclusive_scan if exclusive else vx.inclusive_scan
                a, b = vx.vector(ctx1, x), vx.vector(ctx1, n, t)
                fn(a, b, init)
                assert same(b.read(), want), (n, exclusive, init)
                fn(a, a, init)                                          # in place
                assert same(a.read(), want), (n, exclusive, init, "in place")
                if exclusive and n:
                    assert so_bits(b.read()[:1])[0] == so_bits(np.asarray([init]).astype(t))[0]


def test_large_scans(ctx1):
    rng = np.random.default_rng(24)
    n = (1 << 24) + 3
    for t in (np.float32, np.int64):
        x = values(t, n, rng)
        a = vx.vector(ctx1, x)
        vx.inclusive_scan(a, a)
        assert same(a.read(), so.scan(x))
        b = vx.vector(ctx1, x)
        vx.exclusive_scan(b, b, 2)
        assert same(b.read(), so.scan(x, True, 2))


@pytest.mark.parametrize("cname", ["ctx1", "ctx2", "ctx3"])
@pytest.mark.parametrize("t", [np.float64, np.float32, np.int32, np.uint64])
def test_scans_on_parts_count_init_once(request, cname, t):
    ctx = request.getfixturevalue(cname)
    rng = np.random.default_rng(5)
    for n in (1, 2, 5, TILE + 1, 3 * TILE + 7):
        x = values(t, n, rng)
        a = vx.vector(ctx, x)
        sizes = [a.part_size(k) for k in range(ctx.nparts)]
        for exclusive in (False, True):
            init = 7
            want = so.scan_parts(x, sizes, exclusive, init)
            if np.dtype(t).kind in "iu":
                c = np.cumsum(x, dtype=t)
                if exclusive:
                    c = np.concatenate([[t(7)], t(7) + c[:-1]]).astype(t)
                assert np.array_equal(want, c)
            out = vx.vector(ctx, n, t)
            (vx.exclusive_scan if exclusive else vx.inclusive_scan)(a, out, init)
            assert same(out.read(), want), (cname, n, exclusive)
            b = vx.vector(ctx, x)
            (vx.exclusive_scan if exclusive else vx.inclusive_scan)(b, b, init)
            assert same(b.read(), want), (cname, n, exclusive, "in place")


# ------------------------------------------------------------------------------------------- by key
def key_patterns(kt, n, rng):
    kt = np.dtype(kt)
    yield "equal", np.full(n, 3, dtype=kt)
    yield "distinct", np.arange(n).astype(kt)
    yield "random_runs", np.sort(rng.integers(0, max(1, n // 3), n)).astype(kt)
    for off in (-1, 0, 1):                                   # runs that end one before, at and one after tile edges
        k = np.zeros(n, dtype=np.int64)
        for e in range(TILE + off, n, TILE):
            k[e:] += 1
        yield f"edges{off:+d}", k.astype(kt)


def by_key_cases(ctx, keys, x, inits_):
    """Every by-key function on one key pattern, in place and out of place."""
    dk = vx.vector(ctx, keys)
    for exclusive in (False, True):
        for init in (inits_ if exclusive else [0]):
            want = so.scan_by_key(keys, x, exclusive, init)
            fn = vx.exclusive_scan_by_key if exclusive else vx.inclusive_scan_by_key
            iv, ov = vx.vector(ctx, x), vx.vector(ctx, x.size, x.dtype)
            fn(dk, iv, ov, init)
            assert same(ov.read(), want), (exclusive, init)
            fn(dk, iv, iv, init)
            assert same(iv.read(), want), (exclusive, init, "in place")
    ok, ov = vx.reduce_by_key(dk, vx.vector(ctx, x))
    wk, wv = so.reduce_by_key(keys, x)
    assert ok.size() == wk.size and same(ok.read(), wk) and same(ov.read(), wv)


@pytest.mark.parametrize("kt", TYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("vt", TYPES, ids=lambda t: np.dtype(t).name)
def test_by_key(ctx1, kt, vt):
    rng = np.random.default_rng(10 * TYPES.index(kt) + TYPES.index(vt))
    for n in (0, 1, 2, TILE - 1, TILE + 1, 5 * TILE + 3):
        x = values(vt, n, rng)
        for name, keys in key_patterns(kt, n, rng):
            by_key_cases(ctx1, keys, x, inits(vt))


@pytest.mark.parametrize("kt", [np.float64, np.float32])
def test_nan_and_signed_zero_keys(ctx1, kt):
    keys = np.array([1.0, np.nan, np.nan, -0.0, 0.0, 0.0, 2.0, np.nan, 2.0, 2.0, -0.0], dtype=kt)
    x = np.arange(1, keys.size + 1, dtype=np.int64)
    dk = vx.vector(ctx1, keys)
    o = vx.vector(ctx1, x.size, np.int64)
    vx.inclusive_scan_by_key(dk, vx.vector(ctx1, x), o)
    assert o.read().tolist() == [1, 2, 3, 4, 9, 15, 7, 8, 9, 19, 11]
    vx.exclusive_scan_by_key(dk, vx.vector(ctx1, x), o, 100)
    assert o.read().tolist() == [100, 100, 100, 100, 104, 109, 100, 100, 100, 109, 100]
    ok, ov = vx.reduce_by_key(dk, vx.vector(ctx1, x))
    assert ov.read().tolist() == [1, 2, 3, 15, 7, 8, 19, 11]
    got = ok.read()
    assert not np.signbit(got[3]) and np.signbit(got[7]) and np.isnan(got[1]) and np.isnan(got[2])
    # the same keys spread across a tile edge
    big = np.concatenate([np.zeros(TILE - 5, kt), keys, np.full(7, 9, kt)])
    xb = values(np.float64, big.size, np.random.default_rng(0))
    by_key_cases(ctx1, big, xb, [0, -0.0, 2.5])


@pytest.mark.parametrize("kt, vt", [(np.int32, np.int64), (np.uint64, np.uint32), (np.float32, np.float64),
                                    (np.int64, np.float32)])
def test_sort_then_reduce_by_key(ctx1, kt, vt):
    rng = np.random.default_rng(11)
    n = 3 * 10 ** 6 + 17
    keys = rng.integers(0, 10 ** 5, n).astype(kt)
    x = values(vt, n, rng) if np.dtype(vt).kind == "f" else rng.integers(-1000, 1000, n).astype(vt)
    dk, dv = vx.vector(ctx1, keys), vx.vector(ctx1, x)
    vx.sort_by_key(dk, dv)
    ok, ov = vx.reduce_by_key(dk, dv)
    p = np.argsort(keys, kind="stable")
    sk, sv = keys[p], x[p]
    wk, wv = so.reduce_by_key(sk, sv)
    assert same(ok.read(), wk) and same(ov.read(), wv)
    if np.dtype(vt).kind in "iu":
        u, first = np.unique(sk, return_index=True)
        assert np.array_equal(ok.read(), u) and np.array_equal(ov.read(), np.add.reduceat(sv, first, dtype=vt))


def test_large_reduce_by_key(ctx1):
    rng = np.random.default_rng(12)
    n = (1 << 24) + 3
    keys = np.sort(rng.integers(0, 1 << 20, n)).astype(np.int64)
    x = rng.standard_normal(n)
    ok, ov = vx.reduce_by_key(vx.vector(ctx1, keys), vx.vector(ctx1, x))
    wk, wv = so.reduce_by_key(keys, x)
    assert same(ok.read(), wk) and same(ov.read(), wv)


@pytest.mark.parametrize("cname", ["ctx2", "ctx3"])
def test_by_key_on_several_parts_throws(request, cname):
    ctx = request.getfixturevalue(cname)
    k, v = vx.vector(ctx, np.zeros(100, np.int32)), vx.vector(ctx, np.ones(100))
    with pytest.raises(ValueError, match="scan_by_key is only supported for single device contexts"):
        vx.inclusive_scan_by_key(k, v, v)
    with pytest.raises(ValueError, match="scan_by_key is only supported for single device contexts"):
        vx.exclusive_scan_by_key(k, v, v)
    with pytest.raises(ValueError, match="reduce_by_key is only supported for single device contexts"):
        vx.reduce_by_key(k, v)


def test_by_key_sizes_must_match(ctx1):
    k, v, w = vx.vector(ctx1, np.zeros(100, np.int32)), vx.vector(ctx1, np.ones(100)), vx.vector(ctx1, np.ones(99))
    with pytest.raises(ValueError, match="input and output should have same size"):
        vx.inclusive_scan_by_key(k, v, w)
    with pytest.raises(ValueError, match="keys and values should have same size"):
        vx.reduce_by_key(k, w)
    with pytest.raises(ValueError, match="keys and ovals are the same buffer"):
        vx.inclusive_scan_by_key(k, vx.vector(ctx1, np.ones(100, np.int32)), k)
