"""The numpy restatement of csrc/scan.cu's order of additions (tests/scan_order.py) against np.cumsum and plain loops,
exact for integers and within a tolerance for floats; the workspace sizes; and every argument vexb_scan,
vexb_scan_by_key, vexb_reduce_by_key_count and vexb_reduce_by_key_write refuse before they touch a device.  No GPU
needed."""
import ctypes as C

import numpy as np
import pytest

import scan_order as so

from vexcl_b200 import _lib as L

TILE = so.TILE
SIZES = [0, 1, 2, TILE - 1, TILE, TILE + 1, 5 * TILE - 1, 5 * TILE + 1, 1024 * TILE + 3, 2100 * TILE + 17]
INTS = [np.int32, np.uint32, np.int64, np.uint64]


def loop_scan_by_key(keys, x, exclusive, init):
    out = np.empty_like(x)
    with np.errstate(over="ignore"):
        for i in range(x.size):
            head = i == 0 or not keys[i] == keys[i - 1]
            if exclusive:
                out[i] = x.dtype.type(init) if head else out[i - 1] + x[i - 1]
            else:
                out[i] = x[i] if head else out[i - 1] + x[i]
    return out


@pytest.mark.parametrize("t", INTS, ids=lambda t: np.dtype(t).name)
def test_restatement_is_cumsum_for_integers(t):
    rng = np.random.default_rng(1)
    info = np.iinfo(t)
    for n in SIZES:
        x = rng.integers(info.min, info.max, n, dtype=t, endpoint=True)
        assert np.array_equal(so.scan(x), np.cumsum(x, dtype=t))
        init = t(info.max - 3)
        with np.errstate(over="ignore"):
            want = np.concatenate([[init], init + np.cumsum(x, dtype=t)[:-1]]).astype(t)[:n]
        assert np.array_equal(so.scan(x, True, init), want)


@pytest.mark.parametrize("t", [np.float64, np.float32], ids=lambda t: np.dtype(t).name)
def test_restatement_is_close_to_float64_sums(t):
    rng = np.random.default_rng(2)
    for n in SIZES[1:]:
        x = rng.standard_normal(n).astype(t)
        ref = np.cumsum(x.astype(np.float64))
        tol = (1e-13 if t == np.float64 else 2e-5) * np.cumsum(np.abs(x.astype(np.float64)))
        assert np.all(np.abs(so.scan(x).astype(np.float64) - ref) <= tol)
        ex = so.scan(x, True, 0.5).astype(np.float64)
        assert ex[0] == 0.5 and np.all(np.abs(ex[1:] - (0.5 + ref[:-1])) <= tol[:-1] + 1e-6)


def test_exclusive_keeps_the_bits_of_init():
    x = np.ones(10, np.float32)
    assert np.signbit(so.scan(x, True, -0.0)[0])
    nan = np.array([0x7FC01234], np.uint32).view(np.float32)[0]
    assert so.scan(x, True, nan)[:1].view(np.uint32)[0] == 0x7FC01234


@pytest.mark.parametrize("kt", [np.float64, np.int32, np.uint64])
def test_restatement_by_key_against_a_loop(kt):
    rng = np.random.default_rng(3)
    for n in (1, 2, 100, TILE + 3, 3 * TILE - 1):
        keys = np.sort(rng.integers(0, max(1, n // 7), n)).astype(kt)
        x = rng.integers(-1000, 1000, n).astype(np.int64)
        assert np.array_equal(so.scan_by_key(keys, x), loop_scan_by_key(keys, x, False, 0))
        assert np.array_equal(so.scan_by_key(keys, x, True, 7), loop_scan_by_key(keys, x, True, 7))
        ok, ov = so.reduce_by_key(keys, x)
        u, first = np.unique(keys, return_index=True)
        assert np.array_equal(ok, u) and np.array_equal(ov, np.add.reduceat(x, first))


def test_restatement_of_float_keys():
    keys = np.array([1.0, np.nan, np.nan, -0.0, 0.0, 0.0, 2.0, 2.0])
    x = np.arange(1, 9, dtype=np.int32)
    assert so.scan_by_key(keys, x).tolist() == [1, 2, 3, 4, 9, 15, 7, 15]
    ok, ov = so.reduce_by_key(keys, x)
    assert ov.tolist() == [1, 2, 3, 15, 15] and not np.signbit(ok[3])


def test_restatement_of_parts_counts_init_once():
    x = np.arange(1, 101, dtype=np.int64)
    for sizes in ([100], [40, 60], [0, 50, 0, 50], [33, 33, 34]):
        assert np.array_equal(so.scan_parts(x, sizes, True, 1000), so.scan(x, True, 1000))
        assert np.array_equal(so.scan_parts(x, sizes), np.cumsum(x))


# ------------------------------------------------------------------------------------------- the C ABI
def workspace(n, vdt):
    nb = C.c_size_t()
    L.check(L.lib().vexb_scan_workspace_bytes(n, vdt, C.byref(nb)))
    return nb.value


def test_workspace_bytes(built):
    assert workspace(0, L.F64) == 0
    for n in (1, TILE, TILE + 1, 10 ** 6, (1 << 31) - 1):
        t = -(-n // TILE)
        for vdt, vb in ((L.F32, 4), (L.U64, 8)):
            w = workspace(n, vdt)
            assert w >= t * vb + (t + 1) * 4 and w % 256 == 0 and w < t * vb + (t + 1) * 4 + 512


def refusal(fn, *args):
    code = fn(*args)
    assert code == L.ERR_INVALID, code
    return L.lib().vexb_last_error().decode()


def test_workspace_bytes_refuses(built):
    nb = C.c_size_t()
    assert "unknown value dtype 6" in refusal(L.lib().vexb_scan_workspace_bytes, 10, 6, C.byref(nb))
    assert "bytes is NULL" in refusal(L.lib().vexb_scan_workspace_bytes, 10, L.F64, None)


# Refused before any device call: these run without a GPU.  Pointers are never dereferenced.
K, I, O, O2, WS = (C.c_void_p(a) for a in (0x10000, 0x20000, 0x30000, 0x38000, 0x40000))
BIG = 1 << 30


@pytest.mark.parametrize("args, msg", [
    ((I, O, 6, 10, 0, None, WS, BIG), "unknown value dtype 6"),
    ((None, O, L.F64, 10, 0, None, WS, BIG), "NULL input or output"),
    ((I, None, L.F64, 10, 1, None, WS, BIG), "NULL input or output"),
    ((I, O, L.I64, 1 << 31, 0, None, WS, 1 << 40), "at most 2^31 - 1"),
    ((I, O, L.F64, 10, 0, None, None, BIG), "d_workspace is NULL"),
    ((I, O, L.F64, 5 * TILE, 0, None, WS, 256), "workspace too small"),
])
def test_scan_refuses_bad_arguments(built, args, msg):
    assert msg in refusal(L.lib().vexb_scan, 0, None, *args)


@pytest.mark.parametrize("args, msg", [
    ((K, 7, I, O, L.F64, 10, 0, None, WS, BIG), "unknown key dtype 7"),
    ((K, L.I32, I, O, -1, 10, 0, None, WS, BIG), "unknown value dtype -1"),
    ((None, L.I32, I, O, L.F64, 10, 0, None, WS, BIG), "NULL keys, input or output"),
    ((K, L.I32, I, None, L.F64, 10, 0, None, WS, BIG), "NULL keys, input or output"),
    ((K, L.I32, I, K, L.I32, 10, 0, None, WS, BIG), "keys and ovals are the same buffer"),
    ((K, L.I32, I, O, L.F64, 1 << 31, 0, None, WS, 1 << 40), "at most 2^31 - 1"),
    ((K, L.I32, I, O, L.F64, 10, 1, None, None, BIG), "d_workspace is NULL"),
    ((K, L.I32, I, O, L.F64, 5 * TILE, 1, None, WS, 100), "workspace too small"),
])
def test_scan_by_key_refuses_bad_arguments(built, args, msg):
    assert msg in refusal(L.lib().vexb_scan_by_key, 0, None, *args)


@pytest.mark.parametrize("args, msg", [
    ((K, 9, I, L.F64, 10, WS, BIG), "unknown key dtype 9"),
    ((K, L.F32, I, 9, 10, WS, BIG), "unknown value dtype 9"),
    ((None, L.F32, I, L.F64, 10, WS, BIG), "NULL keys or values"),
    ((K, L.F32, None, L.F64, 10, WS, BIG), "NULL keys or values"),
    ((K, L.F32, I, L.F64, 1 << 31, WS, 1 << 40), "at most 2^31 - 1"),
    ((K, L.F32, I, L.F64, 10, None, BIG), "d_workspace is NULL"),
    ((K, L.F32, I, L.F64, 5 * TILE, WS, 8), "workspace too small"),
])
def test_reduce_by_key_count_refuses_bad_arguments(built, args, msg):
    runs = C.c_size_t()
    assert msg in refusal(L.lib().vexb_reduce_by_key_count, 0, None, *args, C.byref(runs))


def test_reduce_by_key_count_refuses_a_null_count(built):
    assert "nruns is NULL" in refusal(L.lib().vexb_reduce_by_key_count, 0, None, K, L.F32, I, L.F64, 10, WS, BIG, None)


@pytest.mark.parametrize("outs, msg", [
    ((None, O), "NULL keys or values"),
    ((O, None), "NULL keys or values"),
    ((K, O), "apart from each other and from ikeys and ivals"),
    ((O, I), "apart from each other and from ikeys and ivals"),
    ((O, O), "apart from each other and from ikeys and ivals"),
    ((I, O2), "apart from each other and from ikeys and ivals"),
])
def test_reduce_by_key_write_refuses_bad_arguments(built, outs, msg):
    assert msg in refusal(L.lib().vexb_reduce_by_key_write, 0, None, K, L.I64, I, L.F64, 10, *outs, WS, BIG)


def test_empty_input_needs_nothing(built):
    lib = L.lib()
    L.check(lib.vexb_scan(0, None, None, None, L.F64, 0, 1, None, None, 0))
    L.check(lib.vexb_scan_by_key(0, None, None, L.I32, None, None, L.F32, 0, 0, None, None, 0))
    runs = C.c_size_t(5)
    L.check(lib.vexb_reduce_by_key_count(0, None, None, L.I32, None, L.F32, 0, None, 0, C.byref(runs)))
    assert runs.value == 0
    L.check(lib.vexb_reduce_by_key_write(0, None, None, L.I32, None, L.F32, 0, None, None, None, 0))
