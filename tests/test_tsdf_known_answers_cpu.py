"""The reference's TSDFMatchCostFunction2D known answers (tsdf_match_cost_function_2d_test.cc)
on a grid built by the restated TSDFRangeDataInserter2D (tests/tsdf_inserter.py), and the
restated minimiser of tests/tsdf2d_oracle.py held equal to the C++ oracle's loop."""
import numpy as np
import pytest

from tests import tsdf2d_oracle as T
from tests import tsdf_inserter as I
from tests.test_oracle_golden_ceres2d import smooth_grid


def reference_cost_fixture(insert=True):
    """TSDFSpaceCostFunction2DTest: MapLimits(0.1, (2.05, 2.05), CellLimits(40, 40)),
    truncation 0.3, max weight 1, and InsertPointcloud()."""
    g = T.TSDF2D(40, 40, 0.1, 2.05, 2.05, 0.3, 1.0)
    if not insert:
        return g
    options = I.TSDFInserterOptions2D(
        truncation_distance=0.3, maximum_weight=1.0, update_free_space=False,
        num_normal_samples=2, sample_radius=10.0, project_sdf_distance_to_scan_normal=True,
        update_weight_range_exponent=0,
        update_weight_angle_scan_normal_to_ray_kernel_bandwidth=0.0,
        update_weight_distance_cell_to_hit_kernel_bandwidth=0.0)
    returns = []
    x = np.float32(-0.5)
    while x < np.float32(0.5):   # for (float x = -.5; x < 0.5f; x += 0.1)
        returns.append([x, 1.0, 0.0])
        x = np.float32(float(x) + 0.1)
    return I.insert(g, [-0.5, -0.5], returns, options)


MATCHING_CLOUD = np.array([[0.0, 1.0, 0.0]], np.float32)
# (pose y, residual, Jacobian) of ExactInitialPose and PertubatedInitialPose; None = invalid
# (MatchEmptyTSDF on the empty grid, InvalidInitialPose at y = +-0.4)
KNOWN_ANSWERS = [(0.0, 0.0, (0.0, -1.0, 0.0)), (0.1, -0.1, (0.0, -1.0, 0.0)),
                 (-0.1, 0.1, (0.0, -1.0, 0.0)), (0.4, None, None), (-0.4, None, None)]


def _cost_function(g, cloud, pose):
    # CreateTSDFMatchCostFunction2D(1.f, cloud, tsdf): scaling 1 = occupied_space_weight / sqrt(1)
    r, j, valid = T.evaluate(g, cloud, pose, pose[:2], pose[2], 1.0, 1.0, 1.0)
    return r[0], j[0], valid


def test_match_empty_tsdf():
    g = reference_cost_fixture(insert=False)
    assert not _cost_function(g, np.zeros((1, 3), np.float32), [0.0, 0.0, 0.0])[2]


@pytest.mark.parametrize("y,residual,jacobian", KNOWN_ANSWERS)
def test_reference_cost_function_known_answers(y, residual, jacobian):
    g = reference_cost_fixture()
    r, j, valid = _cost_function(g, MATCHING_CLOUD, [0.0, y, 0.0])
    if residual is None:
        assert not valid
        return
    assert valid
    assert abs(r - residual) < 1e-3
    assert np.allclose(j, jacobian, rtol=0, atol=1e-3)


def test_inserter_fixture_is_a_surface_at_the_returns():
    """The inserted band straddles y = 1 (the returns): tsd falls through zero there."""
    g = reference_cost_fixture()
    iy, ix = np.nonzero(g.weight_cells)
    assert len(ix) > 0
    cx, cy = g.cell_center(ix, iy)
    tsd = g.get_correspondence_cost(ix, iy)
    near = np.abs(cy - 1.0) < 0.06
    assert np.all(np.abs(tsd[near]) < 0.06)
    assert np.all(np.abs(cy[~near] - 1.0) <= 0.35)


def test_ray_to_pixel_mask_covers_the_segment():
    # ray_to_pixel_mask_test.cc: a diagonal ray through three pixels
    assert I.ray_to_pixel_mask((0, 0), (2999, 2999), 1000) == [(0, 0), (1, 1), (2, 2)]
    assert I.ray_to_pixel_mask((2999, 2999), (0, 0), 1000) == [(0, 0), (1, 1), (2, 2)]
    assert I.ray_to_pixel_mask((500, 500), (500, 2500), 1000) == [(0, 0), (0, 1), (0, 2)]


@pytest.mark.parametrize("nonmonotonic", [True, False])
def test_restated_loop_equals_the_cpp_oracle_loop(oracle, nonmonotonic):
    """The Python trust-region loop on the ProbabilityGrid cost of oracle/ gives the C++
    oracle's CeresMatch2D: the two copies of the minimiser cannot drift apart."""
    rng = np.random.RandomState(8)
    grid = smooth_grid(oracle)
    ang = rng.uniform(0, 2 * np.pi, 300)
    rad = rng.uniform(0.02, 0.3, 300)
    cloud = np.stack([rad * np.cos(ang), rad * np.sin(ang), np.zeros(300)], 1).astype(np.float32)
    init = np.array([0.525 + 0.05, -0.125 - 0.04, 0.3])

    def prob_cost(g, xyz, pose, target, angle, ow, tw, rw, jacobian):
        r, j = oracle.ceres2d_evaluate(g, xyz, pose, target, angle, ow, tw, rw, jacobian)
        return r, j, True
    got = T.match(grid, cloud, init[:2], init, 20.0, 10.0, 1.0, nonmonotonic, 15,
                  evaluator=prob_cost)
    want = oracle.ceres2d_match(grid, cloud, init[:2], init, 20.0, 10.0, 1.0, nonmonotonic, 15)
    assert np.allclose(got["pose"], want["pose"], rtol=0, atol=1e-9)
    assert got["iterations"] == want["iterations"]
    assert got["num_successful_steps"] == want["num_successful_steps"]
    assert got["termination"] == want["termination"]
    assert got["initial_cost"] == pytest.approx(want["initial_cost"], rel=1e-12)
    assert got["final_cost"] == pytest.approx(want["final_cost"], rel=1e-9)
