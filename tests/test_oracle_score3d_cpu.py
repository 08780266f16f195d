"""Pins the oracle's 3D ScoreCandidates test hook (score_candidates) against a numpy
evaluation of the reference's per-depth cell formula over the oracle's precomputation
levels, at every depth and full_resolution_depth, with negative offsets.  CPU only."""
import numpy as np
import pytest

from tests import worlds3d

RES = 0.1


def _case(oracle, seed, depth, frd, xy, z, n_hi=200):
    rng = np.random.RandomState(seed)
    hi = worlds3d.random_voxels(rng, 3000, 24, RES)
    lo = worlds3d.random_voxels(rng, 400, 8, 0.45)
    od = worlds3d.fast_options(depth=depth, frd=frd, xy=xy, z=z, angular=0.03)
    om = oracle.FastCorrelativeScanMatcher3D(oracle.HybridGrid(RES, hi.indices, hi.values),
                                             oracle.HybridGrid(0.45, lo.indices, lo.values),
                                             np.zeros(8, np.float32), od)
    node = worlds3d.node_data(worlds3d.random_cloud(rng, n_hi, 2.0),
                              low=worlds3d.random_cloud(rng, 50, 2.0))
    pose = [0.03, -0.02, 0.01, 1, 0, 0, 0]
    return rng, od, om, node, pose


@pytest.mark.parametrize("depth,frd,xy,z", [
    (2, 1, 0.7, 0.3), (3, 1, 0.5, 0.0), (4, 2, 0.9, 0.5), (5, 3, 0.7, 0.3),
    (6, 3, 1.3, 0.5), (6, 8, 0.7, 0.3), (8, 3, 1.1, 0.7)])
def test_score_candidates_hook_equals_numpy(oracle, depth, frd, xy, z):
    rng, od, om, node, pose = _case(oracle, depth * 10 + frd, depth, frd, xy, z)
    wxy, wz = worlds3d.search_window(od, RES)
    cells, _, _ = om.discrete_scans(False, pose, [0, 0, 0, 1, 0, 0, 0], node)
    S, n = cells.shape[:2]
    assert S >= 2
    for d in range(depth):
        # every candidate offset of the window, including negative and odd ones
        m = 300
        cand = np.stack([rng.randint(0, S, m), rng.randint(-wxy, wxy + 1, m),
                         rng.randint(-wxy, wxy + 1, m), rng.randint(-wz, wz + 1, m)], axis=1)
        sums, scores, low = om.score_candidates(
            False, pose, [0, 0, 0, 1, 0, 0, 0], node, d, cand)
        want = worlds3d.numpy_sums(om, cells, d, frd, wxy, wz, cand)
        np.testing.assert_array_equal(sums, want)
        np.testing.assert_array_equal(scores.view(np.uint32),
                                      worlds3d.to_score(want, n).view(np.uint32))
        assert (low is not None) == (d == 0)
        assert sums.max() > 0
        if d == 0:   # a mean of probabilities in [0.1, 0.9], up to float rounding
            assert np.all((low > 0.0999) & (low < 0.9001))


@pytest.mark.parametrize("depth,frd", [(4, 1), (5, 3), (5, 9)])
def test_lowest_resolution_maximum_is_what_match_explores(oracle, depth, frd):
    """The largest lowest-resolution score from the hook is the first candidate Match
    expands: with min_score equal to it Match expands nothing, just below it at least one
    node, and Match scores exactly the hook's lattice."""
    rng, od, om, node, pose = _case(oracle, 77 + depth, depth, frd, 0.6, 0.3, n_hi=80)
    wxy, wz = worlds3d.search_window(od, RES)
    cells, _, _ = om.discrete_scans(False, pose, [0, 0, 0, 1, 0, 0, 0], node)
    S = len(cells)
    step = 1 << (depth - 1)
    xs = np.arange(-wxy, wxy + 1, step)
    zs = np.arange(-wz, wz + 1, step)
    cand = np.array([(s, x, y, zz) for s in range(S) for zz in zs for y in xs for x in xs])
    sums, scores, _ = om.score_candidates(False, pose, [0, 0, 0, 1, 0, 0, 0], node, depth - 1,
                                          cand)
    np.testing.assert_array_equal(
        sums, worlds3d.numpy_sums(om, cells, depth - 1, frd, wxy, wz, cand))
    top = scores.max()
    at = om.match(pose, [0, 0, 0, 1, 0, 0, 0], node, float(top))
    assert not at["found"] and at["nodes_expanded"] == 0
    assert at["lowest_resolution_candidates"] == len(cand)
    below = om.match(pose, [0, 0, 0, 1, 0, 0, 0], node,
                     float(np.nextafter(top, np.float32(-1))))
    assert below["nodes_expanded"] >= 1
    if below["found"]:
        assert below["score"] <= top
