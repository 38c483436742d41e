"""vx.sort / vx.sort_by_key (vexb_sort, and vexb_sort_merge for several parts) on the GPU, bit for bit against the
numpy restatement of the order in tests/sort_order.py: every key type, keys alone or with U32 values or I64 values =
arange, both directions, at the tile and grid boundaries of the shape rule in csrc/sort.cu (tile = 4096 elements,
G = min(tiles, 2 x SMs) runs of tiles), on random bit patterns (NaN, inf and subnormals among the floats), few distinct
keys, equal keys, sorted and reversed input, and keys that differ only in their top byte."""
import ctypes as C

import numpy as np
import pytest

from sort_order import bits, permutation, sorted_bits

import vexcl_b200 as vx
from vexcl_b200 import _lib as L

pytestmark = pytest.mark.gpu

TILE, CTAS_PER_SM = 4096, 2
KEYS = [np.float64, np.float32, np.int32, np.uint32, np.int64, np.uint64]
VALS = [None, np.uint32, np.int64]


def grid():
    p = L.DevProps()
    L.check(L.lib().vexb_device_props(0, C.byref(p)))
    return CTAS_PER_SM * p.sm_count


def boundary_sizes():
    G = grid()
    return [0, 1, 2, TILE - 1, TILE, TILE + 1, G * TILE - 1, G * TILE, G * TILE + 1, 3 * G * TILE + 5]


def make_keys(t, n, pattern, rng):
    t = np.dtype(t)
    u = {4: np.uint32, 8: np.uint64}[t.itemsize]
    if pattern == "random":
        return rng.integers(0, np.iinfo(u).max, n, dtype=u, endpoint=True).view(t)
    if pattern == "few":
        pool = rng.integers(0, np.iinfo(u).max, 5, dtype=u, endpoint=True).view(t)
        return pool[rng.integers(0, pool.size, n)]
    if pattern == "equal":
        return np.full(n, rng.integers(0, np.iinfo(u).max, dtype=u, endpoint=True), dtype=u).view(t)
    if pattern == "top_byte":
        return (rng.integers(0, 256, n, dtype=u) << u(8 * t.itemsize - 8)).view(t)
    k = sorted_bits(make_keys(t, n, "random", rng))[0]
    return k if pattern == "sorted" else k[::-1].copy()


def check(ctx, keys, desc, value_types=VALS):
    """Sort `keys` alone and by key with each value type; one oracle permutation serves all of them."""
    n = keys.size
    p = permutation(keys, desc)
    want_k = bits(keys[p])
    for vt in value_types:
        dk = vx.vector(ctx, keys)
        if vt is None:
            vx.sort(dk, descending=desc)
        else:
            vals = np.arange(n, dtype=vt) if vt == np.int64 else np.random.default_rng(n).integers(0, 1 << 32, n, dtype=np.uint32)
            dv = vx.vector(ctx, vals)
            vx.sort_by_key(dk, dv, descending=desc)
        got = bits(dk.read())
        assert np.array_equal(got, want_k), f"keys ({vt}) differ at {np.flatnonzero(got != want_k)[:8]} of {n}"
        if vt is not None:
            gv = dv.read()
            assert np.array_equal(gv, vals[p]), f"values ({vt}) differ at {np.flatnonzero(gv != vals[p])[:8]} of {n}"


@pytest.mark.parametrize("kt", KEYS, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("desc", [False, True], ids=["asc", "desc"])
def test_sort_at_the_boundaries(ctx1, kt, desc):
    rng = np.random.default_rng(10 * KEYS.index(kt) + desc)
    for n in boundary_sizes():
        check(ctx1, make_keys(kt, n, "random", rng), desc)


@pytest.mark.parametrize("kt", KEYS, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("desc", [False, True], ids=["asc", "desc"])
def test_sort_patterns(ctx1, kt, desc):
    rng = np.random.default_rng(7)
    for n in (TILE + 1, grid() * TILE + 1):
        for pattern in ("few", "equal", "sorted", "reversed", "top_byte"):
            check(ctx1, make_keys(kt, n, pattern, rng), desc)


@pytest.mark.parametrize("kt, vt, desc", [(np.uint32, np.int64, False), (np.float64, None, True)])
def test_sort_large(ctx1, kt, vt, desc):
    check(ctx1, make_keys(kt, (1 << 24) + 3, "random", np.random.default_rng(24)), desc, [vt])


@pytest.mark.parametrize("cname", ["ctx2", "ctx3"])
@pytest.mark.parametrize("kt, vt", [(np.float32, np.int64), (np.int64, np.uint32), (np.uint32, None), (np.float64, np.int64)])
@pytest.mark.parametrize("desc", [False, True], ids=["asc", "desc"])
def test_sort_parts_merge(request, cname, kt, vt, desc):
    ctx = request.getfixturevalue(cname)
    rng = np.random.default_rng(3)
    for n in (0, 1, 5, 40, TILE + 1, grid() * TILE + 1):
        for pattern in ("random", "few"):
            check(ctx, make_keys(kt, n, pattern, rng), desc, [vt])


def test_keys_and_values_of_different_sizes_are_refused(ctx2):
    k, v = vx.vector(ctx2, np.zeros(100, np.int32)), vx.vector(ctx2, np.zeros(99, np.int32))
    with pytest.raises(ValueError, match="span different devices"):
        vx.sort_by_key(k, v)
