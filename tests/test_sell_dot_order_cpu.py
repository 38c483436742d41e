"""tests/sell_dot_order.py without a device: with lanes in row order it is reduce_order's hybrid-ELL dot, padding lanes
add +0, and on a real sliced-ELL layout the restated dot stays within the error bound of its depth."""
import math

import numpy as np

import reduce_order as ro
import sell_dot_order as so


def test_lanes_in_row_order_give_the_hybrid_ell_dot(built):
    rng = np.random.default_rng(1)
    for n in (1, 255, 256, 257, 8 * 256 * 3 + 5):
        w, y = rng.standard_normal(n), rng.standard_normal(n)
        perm = np.full(-(-n // 32) * 32, -1, np.int32)
        perm[:n] = np.arange(n)
        got = so.dot_partials(w, y, perm)
        want = ro.dot_partials(w, y)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
        assert so.fused_dot(w, y, perm) == ro.fused_dot(w, y)


def test_layout_order_and_padding(built):
    rng = np.random.default_rng(2)
    for n, sigma in ((33, 256), (1025, 256), (9000, 1024)):
        widths = rng.integers(0, 40, n)
        row = np.concatenate([[0], np.cumsum(widths)]).astype(np.int64)
        perm = so.sell_layout(row, sigma)
        assert perm.size == -(-n // 32) * 32 and np.array_equal(np.sort(perm[perm >= 0]), np.arange(n))
        w, y = rng.standard_normal(n), rng.standard_normal(n)
        assert so.dot_partials(w, y, perm).size == so.interior_blocks(perm)
        d = so.fused_dot(w, y, perm)
        assert abs(d - math.fsum(w * y)) <= 40 * 2.0 ** -53 * float(np.sum(np.abs(w * y)))
        for dtype in (np.float64, np.float32):
            assert so.fused_dot(np.zeros(n, dtype), y.astype(dtype), perm) == 0
