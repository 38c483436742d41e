"""Pins tests/stencil_ref.py without a GPU: the shared-memory thresholds of stencil_launch worked out by hand, the operator
restatement against a per-element loop over vexb_stencil_op's literal block windows, and the halo exchange against
`convolve` of the whole vector."""
import numpy as np
import pytest

import oracle
from oracle.stencil import convolve_loop
import stencil_ref as sr

# dtype: widest width accepted, first refused, last at <= 48 KB, last whose two pipe windows fit in 100 KB
THRESHOLDS = {np.float64: (11504, 11505, 2344, 3224), np.float32: (23544, 23545, 5240, 7160)}


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_shared_memory_thresholds(dtype):
    widest, refused, last48, lastpipe = THRESHOLDS[dtype]
    assert sr.accepted(widest, dtype) and not sr.accepted(refused, dtype)
    assert not sr.attribute_path(last48, dtype) and sr.attribute_path(last48 + 1, dtype)
    assert sr.pipe_fits(lastpipe, dtype) and not sr.pipe_fits(lastpipe + 1, dtype)
    # each is the edge: every narrower width passes the same test
    assert all(sr.accepted(w, dtype) for w in range(widest - 64, widest + 1))
    assert all(not sr.attribute_path(w, dtype) for w in range(1, last48 + 1, 97))
    assert all(sr.pipe_fits(w, dtype) for w in range(1, lastpipe + 1, 97))


def test_geometry_by_hand():
    assert [sr.ceil8(w) for w in (1, 7, 8, 9, 16, 17)] == [8, 8, 8, 16, 16, 24]
    assert sr.st_pad(1032) == 1161 and sr.wlen(21) == 1048
    assert sr.smem_bytes(21, np.float64) == (1048 + 131 + 1 + 24) * 8
    assert sr.pipe_smem_bytes(21, np.float32) == (2 * (1048 + 131 + 1) + 24) * 4
    assert sr.tiles(1) == 1 and sr.tiles(1024) == 1 and sr.tiles(1025) == 2
    # 3 * 1024 + 5 outputs, width 33, center 16: the first and the last two tiles clamp, the second loads directly
    assert [sr.tile_inside(t, 3077, 33, 16) for t in range(4)] == [False, True, False, False]
    assert not any(sr.tile_inside(t, 1025, 9, 4) for t in range(2))
    # the pipe kernel needs stencil.kernel = 0, fitting windows and more tiles than resident blocks
    assert sr.uses_pipe(9, 132 * 1024 + 1, np.float64, 0, 1, 132)
    assert not sr.uses_pipe(9, 132 * 1024, np.float64, 0, 1, 132)
    assert not sr.uses_pipe(9, 132 * 1024 + 1, np.float64, 1, 1, 132)
    assert not sr.uses_pipe(3225, 10 ** 7, np.float64, 0, 1, 132)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_convolve_slice_is_convolve_without_halos(dtype):
    rng = np.random.default_rng(3)
    for n, w in ((1, 1), (7, 9), (300, 21), (1030, 64)):
        for c in sorted({0, w // 2, w - 1}):
            s, x, y = (rng.random(m).astype(dtype) for m in (w, n, n))
            assert np.array_equal(sr.convolve_slice(s, c, x), sr.convolve(s, c, x))
            got = sr.convolve_slice(s, c, x, y=y, alpha=0.5, append=True)
            assert got.dtype == dtype
            assert np.array_equal(got, sr.convolve(s, c, x, y=y, alpha=0.5, append=True))
            assert np.array_equal(sr.convolve_slice(s, c, x), convolve_loop(s, c, x))


def _operator_loop(body, width, center, x, left, right, y, alpha, append):
    """vexb_stencil_op one output at a time, from each block's literal window."""
    x = np.asarray(x)
    T, n = x.dtype.type, x.size
    out = np.empty(n, dtype=x.dtype)
    for b in range(-(-n // sr.OP_B)):
        win = sr.op_window(x, b, width, center, left, right)
        for t in range(sr.OP_B):
            i = b * sr.OP_B + t
            if i >= n:
                break
            X = (lambda k, t=t: np.array([win[center + t + k]], dtype=x.dtype))
            v = T(alpha) * sr.BODIES[body][1](X, T, width, center)[0]
            out[i] = y[i] + v if append else v
    return out


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_operator_restatement_against_the_literal_loop(dtype):
    rng = np.random.default_rng(5)
    shapes = {"second_difference": (3, 1), "forward": (4, 0), "backward": (4, 3), "min_max": (3, 1), "sum_squares": (37, 11)}
    for body, (w, c) in shapes.items():
        for n in (1, 2, 255, 257, 300):
            x, y = rng.random(n).astype(dtype), rng.random(n).astype(dtype)
            left, right = (rng.random(max(m, 1)).astype(dtype) + 10 for m in (c, w - 1 - c))
            for lh, rh in ((None, None), (left, None), (None, right), (left, right)):
                for alpha, append in ((1.0, False), (0.5, True)):
                    want = _operator_loop(body, w, c, x, lh, rh, y, alpha, append)
                    got = sr.apply_operator(body, w, c, x, lh, rh, y, alpha, append)
                    assert got.dtype == dtype
                    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (body, n, lh is None, rh is None)


def test_operator_bodies_by_hand():
    x = np.array([1.0, 2.0, 4.0, 8.0])
    # second difference with the ends clamped: [1-2+2, 1-4+4, 2-8+8, 4-16+8]
    assert np.array_equal(sr.apply_operator("second_difference", 3, 1, x), [1.0, 1.0, 2.0, -4.0])
    # halos replace the clamps: [5-2+2, ..., 4-16+7]
    assert np.array_equal(sr.apply_operator("second_difference", 3, 1, x, left=[5.0], right=[7.0]), [5.0, 1.0, 2.0, -5.0])
    assert np.array_equal(sr.apply_operator("sum_squares", 3, 1, x), [6.0, 21.0, 84.0, 144.0])
    # float bodies round in float: 2^24 + 1 is not a float
    xf = np.array([2.0 ** 24, 1.0, 0.0], dtype=np.float32)
    assert sr.apply_operator("sum_squares", 2, 0, xf)[1] == np.float32(1.0)
    assert sr.apply_operator("forward", 4, 0, np.array([2.0 ** 25, 1.0, 1.0, 0.0], dtype=np.float32))[0] == np.float32(-(2.0 ** 24) + 1)


def _bounds(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_halos_against_the_whole_vector(dtype):
    """Two and three slices, with slices of length 0, 1 and shorter than either halo."""
    rng = np.random.default_rng(9)
    slicings = [(20, 20), (1, 39), (39, 1), (0, 40), (40, 0), (3, 37), (16, 0, 24), (16, 1, 23), (0, 0, 40), (2, 1, 37),
                (16, 16, 8), (30, 2, 8), (1, 1, 1), (2, 0, 1)]
    for sizes in slicings:
        n = sum(sizes)
        x, y = rng.random(n).astype(dtype), rng.random(n).astype(dtype)
        for w, c in ((1, 0), (2, 0), (2, 1), (5, 2), (9, 0), (9, 8), (21, 7)):
            s = rng.random(w).astype(dtype)
            b = _bounds(sizes)
            want = sr.convolve(s, c, x)
            assert np.array_equal(sr.convolve_slices(s, c, x, b), want), (sizes, w, c)
            assert np.array_equal(sr.convolve_slices(s, c, x, b, y=y, alpha=0.5, append=True),
                                  sr.convolve(s, c, x, y=y, alpha=0.5, append=True))


def test_halo_contents_by_hand():
    x = np.arange(10.0)
    # width 7, center 4: left halos of 4, right halos of 2; the middle slice [2, 3) has both, padded at the left end
    (l0, r0), (l1, r1), (l2, r2) = sr.slice_halos(x, [0, 2, 3, 10], 4, 7)
    assert l0 is None and list(r0) == [2.0, 3.0]
    assert list(l1) == [0.0, 0.0, 0.0, 1.0] and list(r1) == [3.0, 4.0]
    assert list(l2) == [0.0, 0.0, 1.0, 2.0] and r2 is None
    # an empty slice gets nothing; the right halo of a slice before a short last slice is padded with x[n - 1]
    halos = sr.slice_halos(x, [0, 9, 9, 10], 0, 4)
    assert halos[1] == (None, None) and list(halos[0][1]) == [9.0, 9.0, 9.0]
    # one slice: no halos at all
    assert sr.slice_halos(x, [0, 10], 4, 7) == [(None, None)]


def test_reach_of_one_infinity():
    """What the GPU reach cases assert: an inf at p makes exactly outputs [p - rhalo, p + center] non-finite."""
    s = oracle.uniform_real(4, 9) + 0.5
    for p in (0, 5, 60, 63):
        for c in (0, 4, 8):
            x = np.ones(64)
            x[p] = -np.inf
            bad = ~np.isfinite(sr.convolve(s, c, x))
            lo, hi = max(p - (8 - c), 0), min(p + c, 63)
            assert np.array_equal(np.flatnonzero(bad), np.arange(lo, hi + 1)), (p, c)
