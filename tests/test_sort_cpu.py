"""vexb_sort_merge (the host merge of sorted parts behind vex::sort and vex::sort_by_key on multi-part vectors) against
the numpy restatement of the order in tests/sort_order.py, bit for bit; and every argument vexb_sort and
vexb_sort_workspace_bytes refuse before they touch a device.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from sort_order import bits, permutation

import vexcl_b200 as vx
from vexcl_b200 import _lib as L

DTYPES = {L.F64: np.float64, L.F32: np.float32, L.I32: np.int32, L.U32: np.uint32, L.I64: np.int64, L.U64: np.uint64}


def special_keys(dt, n, rng):
    """Random keys with the values where orders differ: +-0, +-inf, NaNs of both signs with distinct payloads, extremes."""
    t = np.dtype(DTYPES[dt])
    if t.kind == "f":
        k = rng.standard_normal(n).astype(t)
        u = t.itemsize * 8
        ui = np.uint32 if u == 32 else np.uint64
        exp = np.array(0x7F800000 if u == 32 else 0x7FF0000000000000, dtype=ui)
        sign = np.array(1 << (u - 1), dtype=ui)
        nans = [(exp | ui(1)), (exp | ui(12345)), (exp | ui(1) | sign), (exp | ui(777) | sign), (exp | ui(1 << (23 if u == 32 else 52) - 1))]
        specials = np.array([0.0, -0.0, np.inf, -np.inf, np.finfo(t).max, -np.finfo(t).max, np.finfo(t).tiny], dtype=t)
        specials = np.concatenate([specials, np.array(nans, dtype=ui).view(t)])
    else:
        info = np.iinfo(t)
        k = rng.integers(info.min, info.max, n, dtype=t, endpoint=True)
        specials = np.array([info.min, info.max, 0, 1, info.min + 1, info.max - 1], dtype=t)
    idx = rng.integers(0, n, n // 3)
    k[idx] = specials[rng.integers(0, specials.size, idx.size)]
    k[rng.integers(0, n, n // 4)] = k[rng.integers(0, n, n // 4)]          # repeats, so that stability shows
    return k


def merge(parts_k, parts_v, kdt, vdt, desc):
    lib = L.lib()
    part = np.concatenate([[0], np.cumsum([p.size for p in parts_k])]).astype(np.uint64)
    hk = np.concatenate(parts_k)
    ok = np.empty_like(hk)
    hv = ov = None
    if parts_v is not None:
        hv = np.concatenate(parts_v)
        ov = np.empty_like(hv)
    parr = (C.c_size_t * part.size)(*[int(x) for x in part])
    L.check(lib.vexb_sort_merge(len(parts_k), parr, hk.ctypes.data, kdt, None if hv is None else hv.ctypes.data, vdt,
                                int(desc), ok.ctypes.data, None if ov is None else ov.ctypes.data))
    return ok, ov


@pytest.mark.parametrize("kdt", list(DTYPES))
@pytest.mark.parametrize("vdt", [-1, L.U32, L.I64])
@pytest.mark.parametrize("desc", [False, True])
def test_merge_matches_the_order(built, kdt, vdt, desc):
    rng = np.random.default_rng(100 * kdt + 10 * (vdt + 1) + desc)
    sizes = [0, 700, 1, 0, 333, 1200, 0]
    n = sum(sizes)
    keys = special_keys(kdt, n, rng)
    vals = np.arange(n, dtype=DTYPES[vdt]) if vdt >= 0 else None
    # each part sorted as vexb_sort leaves it; the merge of the parts must equal the stable sort of the whole
    pk, pv, o = [], [], 0
    for s in sizes:
        p = permutation(keys[o:o + s], desc) + o
        pk.append(keys[p])
        pv.append(vals[p] if vals is not None else None)
        o += s
    ok, ov = merge(pk, pv if vals is not None else None, kdt, vdt, desc)
    want = permutation(keys, desc)
    assert np.array_equal(bits(ok), bits(keys[want]))
    if vals is not None:
        assert np.array_equal(ov, vals[want])


def test_merge_ties_go_to_the_lower_part(built):
    a = np.array([1, 2, 2], dtype=np.int32)
    b = np.array([2, 2, 3], dtype=np.int32)
    va, vb = np.array([0, 1, 2], dtype=np.int32), np.array([10, 11, 12], dtype=np.int32)
    ok, ov = merge([a, b], [va, vb], L.I32, L.I32, False)
    assert ok.tolist() == [1, 2, 2, 2, 2, 3] and ov.tolist() == [0, 1, 2, 10, 11, 12]
    ok, ov = merge([b[::-1].copy(), a[::-1].copy()], [vb[::-1].copy(), va[::-1].copy()], L.I32, L.I32, True)
    assert ok.tolist() == [3, 2, 2, 2, 2, 1] and ov.tolist() == [12, 11, 10, 2, 1, 0]


def workspace(n, kdt, vdt):
    nb = C.c_size_t()
    L.check(L.lib().vexb_sort_workspace_bytes(n, kdt, vdt, C.byref(nb)))
    return nb.value


def test_workspace_bytes(built):
    assert workspace(0, L.F64, -1) == 0 and workspace(1, L.U32, L.I64) == 0
    for n in (2, 4096, 4097, 10 ** 6):
        for kdt in DTYPES:
            for vdt in (-1, L.F32, L.U64):
                kb, vb = np.dtype(DTYPES[kdt]).itemsize, (np.dtype(DTYPES[vdt]).itemsize if vdt >= 0 else 0)
                assert workspace(n, kdt, vdt) >= n * (kb + vb) + 1024 * ((n + 4095) // 4096)


def refusal(fn, *args):
    code = fn(*args)
    assert code == L.ERR_INVALID, code
    return L.lib().vexb_last_error().decode()


@pytest.mark.parametrize("kdt, vdt, msg", [(6, -1, "unknown key dtype 6"), (-1, -1, "unknown key dtype -1"),
                                           (L.F64, 6, "unknown value dtype 6"), (L.F64, -2, "unknown value dtype -2")])
def test_workspace_bytes_refuses_unknown_dtypes(built, kdt, vdt, msg):
    nb = C.c_size_t()
    assert msg in refusal(L.lib().vexb_sort_workspace_bytes, 10, kdt, vdt, C.byref(nb))


# vexb_sort is refused before any device call: these run on a machine without a GPU.  Pointers are never dereferenced.
K, V, WS = C.c_void_p(0x10000), C.c_void_p(0x20000), C.c_void_p(0x40000)


@pytest.mark.parametrize("args, msg", [
    ((K, 7, None, -1, 10, 0, WS, 1 << 20), "unknown key dtype 7"),
    ((K, L.F32, V, 9, 10, 0, WS, 1 << 20), "unknown value dtype 9"),
    ((None, L.F32, None, -1, 10, 0, WS, 1 << 20), "keys is NULL"),
    ((K, L.F32, V, -1, 10, 0, WS, 1 << 20), "vals is given without a val_dtype"),
    ((K, L.F32, None, L.I64, 10, 0, WS, 1 << 20), "without vals"),
    ((K, L.F32, K, L.I32, 10, 0, WS, 1 << 20), "vals and keys are the same buffer"),
    ((K, L.U64, None, -1, 1 << 31, 0, WS, 1 << 62), "at most 2^31 - 1"),
    ((K, L.F64, V, L.F64, 10, 0, None, 1 << 20), "d_workspace is NULL"),
    ((K, L.F64, V, L.F64, 5000, 0, WS, 5000 * 16), "workspace too small"),
])
def test_sort_refuses_bad_arguments(built, args, msg):
    assert msg in refusal(L.lib().vexb_sort, 0, None, *args)


def test_sort_of_fewer_than_two_elements_needs_nothing(built):
    lib = L.lib()
    for n in (0, 1):
        L.check(lib.vexb_sort(0, None, K if n else None, L.F64, None, -1, n, 0, None, 0))
        L.check(lib.vexb_sort(0, None, K, L.I32, V, L.U64, n, 1, None, 0))


def test_merge_refuses_bad_arguments(built):
    lib = L.lib()
    part = (C.c_size_t * 3)(0, 5, 3)
    k = np.zeros(5, dtype=np.int32)
    assert "decrease" in refusal(lib.vexb_sort_merge, 2, part, k.ctypes.data, L.I32, None, -1, 0, k.ctypes.data, None)
    part = (C.c_size_t * 3)(0, 2, 5)
    assert "unknown key dtype" in refusal(lib.vexb_sort_merge, 2, part, k.ctypes.data, 8, None, -1, 0, k.ctypes.data, None)
    assert "without a val_dtype" in refusal(lib.vexb_sort_merge, 2, part, k.ctypes.data, L.I32, k.ctypes.data, -1, 0,
                                            k.ctypes.data, k.ctypes.data)
