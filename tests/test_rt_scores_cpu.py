"""The oracle's per-candidate score hooks (rt2d_scores, rt2d_scores_tsdf, rt3d_scores) against
the oracle's own Match: reduced by first maximum in generation order, the scores give Match's
result (real_time_correlative_scan_matcher_2d.cc:142-143 std::max_element,
real_time_correlative_scan_matcher_3d.cc:45-48 `score > best_score`).  The device tests in
test_gpu_rt_kernels.py compare the kernels with these scores bit for bit."""
import math

import numpy as np

from benchmarks import synthetic
from tests import worlds
from tests.test_oracle_golden_3d import _rt3d_fixture, rt3d_reference_initial_poses


def _bits(x):
    return np.array(x, np.float32).view(np.uint32)


def _first_max_2d(scores, want, lin_cells):
    w = 2 * lin_cells + 1
    assert len(scores) == want["candidates_scored"] == want["num_scans"] * w * w
    i = int(np.argmax(scores))            # first maximum; -0.0 and +0.0 compare equal
    assert _bits(scores[i]) == _bits(want["score"])
    scan, r = divmod(i, w * w)
    assert (scan, -lin_cells + r // w, -lin_cells + r % w) == (
        want["best_scan_index"], want["best_x_offset"], want["best_y_offset"])


def test_rt2d_scores_reduce_to_match(oracle):
    grid, occ, _, _ = worlds.small_world(501, size_cells=160, beams=181, max_range=5.0)
    og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
    rng = np.random.RandomState(5)
    for lin, ang, w_t, w_r in [(0.1, math.radians(7.0), 0.1, 0.1), (0.0, 0.0, 0.1, 0.1),
                               (0.3, math.radians(3.0), 0.0, 0.0)]:
        pose = synthetic.random_free_pose(occ, grid, rng, margin_cells=10)
        scan = synthetic.cast_scan(occ, grid, pose, beams=241, max_range=5.0, seed=3)
        init = pose + rng.uniform(-1, 1, 3) * [0.05, 0.05, 0.05]
        scores = oracle.rt2d_scores(og, scan, init, lin, ang, w_t, w_r)
        want = oracle.rt2d_match(og, scan, init, lin, ang, w_t, w_r)
        _first_max_2d(scores, want, int(math.ceil(lin / grid.resolution)))


def test_rt2d_tsdf_scores_reduce_to_match(oracle):
    spec, occ = synthetic.make_tsdf2d(502, size_cells=160)
    rng = np.random.RandomState(6)
    g = synthetic.GridSpec(np.zeros_like(spec.tsd_cells), spec.resolution, spec.max_x, spec.max_y)
    pose = synthetic.random_free_pose(occ, g, rng, margin_cells=10)
    scan = synthetic.cast_scan(occ, g, pose, beams=241, max_range=5.0, seed=4)
    args = (spec.tsd_cells, spec.weight_cells, spec.resolution, spec.max_x, spec.max_y,
            spec.truncation_distance, spec.max_weight, scan, pose + [0.03, -0.02, 0.02], 0.1,
            math.radians(5.0), 0.1, 0.1)
    _first_max_2d(oracle.rt2d_scores_tsdf(*args), oracle.rt2d_match_tsdf(*args), 2)


def test_rt2d_tsdf_scores_below_zero(oracle):
    """Truncation 0.35: the largest tsd value decodes to slightly more than the truncation,
    so every weighted cell scores below 0.  With one weight-0 cell, read alone by the
    mid-window candidate, Match returns that candidate with score 0."""
    res, trunc = 0.0625, 0.35
    tsd = np.full((30, 30), 32767, np.uint16)
    wgt = np.full((30, 30), 32767, np.uint16)
    max_xy = 30 * res / 2
    init = [max_xy - 15.5 * res, max_xy - 15.5 * res, 0.0]
    cloud = np.zeros((4, 3), np.float32)
    args = (tsd, wgt, res, max_xy, max_xy, trunc, 10.0, cloud, init, 2 * res, 0.5, 0.1, 0.0)
    scores = oracle.rt2d_scores_tsdf(*args)
    assert (scores < 0).all()
    _first_max_2d(scores, oracle.rt2d_match_tsdf(*args), 2)
    wgt[15, 15] = 0
    scores = oracle.rt2d_scores_tsdf(*args)
    want = oracle.rt2d_match_tsdf(*args)
    assert want["score"] == 0.0 and (want["best_x_offset"], want["best_y_offset"]) == (0, 0)
    assert want["best_scan_index"] == 0 and (scores <= 0).all()
    _first_max_2d(scores, want, 2)


def test_rt3d_scores_reduce_to_match(oracle):
    pts, ogrid, _, _ = _rt3d_fixture(oracle)
    for init in rt3d_reference_initial_poses()[:4]:
        scores = oracle.rt3d_scores(ogrid, pts, init, 0.3, math.radians(1.0), 1e-1, 1.0)
        want = oracle.rt3d_match(ogrid, pts, init, 0.3, math.radians(1.0), 1e-1, 1.0)
        assert len(scores) == want["candidates_scored"]
        i = int(np.argmax(scores))
        assert i == want["best_index"]
        assert _bits(scores[i]) == _bits(want["score"])
