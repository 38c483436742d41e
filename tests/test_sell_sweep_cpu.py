"""Host-side ground of the storage-order sweep over a sliced-ELL strip (generated assignment kernels, csrc/jit.cu): the
kernel gives one thread to every stored lane and writes the target at that lane's row, so every element is written exactly
once only if sell_layout puts each of the n rows -- empty ones included -- in exactly one lane.  Checked through
vexb_csr_sell_layout, with the argument checks of vexb_dspmat_sweep_strip.  No device is touched."""
import ctypes as C

import numpy as np
import pytest

from vexcl_b200 import _lib as L


def layout(w, sigma):
    n = len(w)
    row = np.concatenate([[0], np.cumsum(w)]).astype(np.int64)
    ns, slots = C.c_size_t(0), C.c_size_t(0)
    L.check(L.lib().vexb_csr_sell_layout(n, row.ctypes.data, 8, sigma, C.byref(ns), C.byref(slots), None, None))
    perm = np.full(ns.value * 32, -7, np.int32)
    sptr = np.full(ns.value + 1, -7, np.int32)
    L.check(L.lib().vexb_csr_sell_layout(n, row.ctypes.data, 8, sigma, C.byref(ns), C.byref(slots), perm.ctypes.data, sptr.ctypes.data))
    return perm, sptr


@pytest.mark.parametrize("sigma", [32, 256, 1024])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 8 * 1024 + 17])
@pytest.mark.parametrize("rows", ["uneven", "all empty", "empty runs"])
def test_every_row_sits_in_exactly_one_lane(built, n, sigma, rows):
    rng = np.random.default_rng(n + sigma)
    w = rng.integers(0, 40, n)
    if rows == "all empty":
        w[:] = 0
    elif rows == "empty runs":
        w[rng.random(n) < 0.5] = 0
        w[n // 3:n // 2] = 0
    perm, sptr = layout(w, sigma)
    assert perm.size == (n + 31) // 32 * 32
    lanes = perm[perm >= 0]
    assert np.array_equal(np.sort(lanes), np.arange(n))                  # each row once, no other row
    assert np.all(perm[perm < 0] == -1)
    for s in range(perm.size // 32):                                     # and its slice is wide enough for it
        r = perm[32 * s:32 * s + 32]
        assert (sptr[s + 1] - sptr[s]) // 32 >= max([w[i] for i in r if i >= 0], default=0)
        assert (sptr[s + 1] - sptr[s]) % 32 == 0
    # a row's lane lies in the row's own window of sigma rows: what keeps a warp's elementwise accesses close together
    pos = np.empty(n, np.int64)
    pos[lanes] = np.nonzero(perm >= 0)[0]
    assert np.array_equal(pos // sigma, np.arange(n) // sigma)


def test_sweep_strip_argument_checks(built):
    h = C.c_void_p(1)
    assert L.lib().vexb_dspmat_sweep_strip(None, C.byref(h)) == L.ERR_INVALID
    assert b"NULL" in L.lib().vexb_last_error()
