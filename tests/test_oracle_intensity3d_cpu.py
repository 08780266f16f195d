"""Pins the intensity restatement (tests/intensity3d_oracle.py: IntensityHybridGrid,
IntensityCostFunction3D and HuberLoss with Ceres' Corrector) to the reference's known answers
— intensity_cost_function_3d_test.cc and ceres_scan_matcher_3d_test.cc with its intensity
block — checks its derivatives against central differences, and its minimiser loop against
the C++ oracle's on the problem without intensity.  CPU only."""
import math

import numpy as np
import pytest

from tests import intensity3d_oracle as iorc
from tests.test_oracle_golden_3d import is_nearly
from tests.test_oracle_golden_ceres3d import POINTS

# ceres_scan_matcher_3d_test.cc:73-88
FIXTURE_INTENSITY = (0.5, 55.0, 100.0)   # weight, huber_scale, intensity_threshold
FIXTURE_OPTIONS = dict(occupied_space_weights=[1.0], translation_weight=0.01,
                       rotation_weight=0.1, use_nonmonotonic_steps=True, max_num_iterations=10)


def hybrid(oracle, resolution, points):
    idx = np.array([oracle.hybrid_get_cell_index(resolution, p) for p in points], np.int32)
    val = np.full(len(idx), oracle.probability_to_value(1.0), np.uint16)
    return (resolution, idx, val), oracle.HybridGrid(resolution, idx, val)


def intensity_grid(oracle, resolution, points, intensities):
    """IntensityHybridGrid::AddIntensity at each point's cell -> (flat spec, oracle grid)."""
    cells = {}
    for p, v in zip(points, intensities):
        c = oracle.hybrid_get_cell_index(resolution, p)
        s, n = cells.get(c, (np.float32(0), 0))
        cells[c] = (np.float32(s + np.float32(v)), n + 1)
    idx = np.array(list(cells), np.int32).reshape(-1, 3)
    sums = np.array([v[0] for v in cells.values()], np.float32)
    counts = np.array([v[1] for v in cells.values()], np.int32)
    return (resolution, idx, sums, counts), iorc.IntensityHybridGrid(resolution, idx, sums, counts)


def fixture(oracle, rotate=0.0):
    """The reference fixture: grids at the points moved by (-1, 0, 0), intensity 50 each;
    `rotate` turns the cloud about z (FullPoseCorrection)."""
    shifted = POINTS + np.array([-1, 0, 0], np.float32)
    hspec, hgrid = hybrid(oracle, 1.0, shifted)
    ispec, igrid = intensity_grid(oracle, 1.0, shifted, [50.0] * len(POINTS))
    cloud = POINTS
    if rotate:
        c, s = np.float32(math.cos(rotate)), np.float32(math.sin(rotate))
        cloud = np.stack([c * POINTS[:, 0] - s * POINTS[:, 1], s * POINTS[:, 0] + c * POINTS[:, 1],
                          POINTS[:, 2]], 1).astype(np.float32)
    return cloud, np.full(len(POINTS), 50.0, np.float32), hspec, hgrid, ispec, igrid


def plus(x, delta):
    """x (+) delta with QuaternionParameterization::Plus on the rotation."""
    out = np.array(x, np.float64)
    out[:3] += delta[:3]
    d = np.asarray(delta[3:], np.float64)
    nd = np.linalg.norm(d)
    if nd > 0:
        z = np.concatenate([[math.cos(nd)], math.sin(nd) / nd * d])
        w = x[3:]
        out[3:] = [z[0] * w[0] - z[1] * w[1] - z[2] * w[2] - z[3] * w[3],
                   z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2],
                   z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1],
                   z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0]]
    return out


# intensity_cost_function_3d_test.cc:37-61
def test_intensity_cost_function_smoke_test(oracle):
    cloud = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2]], np.float32)
    intensities = np.array([50, 100, 150], np.float32)
    grid = iorc.IntensityHybridGrid(0.3)
    grid.add_intensity(oracle.hybrid_get_cell_index(0.3, [0, 0, 0]), 50.0)
    _, hgrid = hybrid(oracle, 0.3, cloud[:1])
    # scaling_factor = weight / sqrt(n) = 1
    res, _ = iorc.evaluate(
        [(cloud, hgrid, grid, intensities)], [0, 0, 0, 1, 0, 0, 0], [0, 0, 0], [1, 0, 0, 0],
        [(math.sqrt(3.0), 1.0, 100.0)], occupied_space_weights=[1.0])
    assert np.allclose(res[3:6], [0.0, -100.0, 0.0], rtol=0, atol=1e-9)


# ceres_scan_matcher_3d_test.cc:99-131 with the fixture's intensity block
@pytest.mark.parametrize("start,rotate", [((-1.0, 0.0, 0.0), 0.0), ((-0.8, 0.0, 0.0), 0.0),
                                          ((-1.0, 0.0, -0.2), 0.0), ((-0.9, -0.2, 0.2), 0.0),
                                          ((-0.95, -0.05, 0.05), 0.05)])
def test_reference_fixture_with_intensity_block(oracle, start, rotate):
    cloud, intensities, _, hgrid, _, igrid = fixture(oracle, rotate)
    a = 0.05 if rotate else 0.0
    init = list(start) + [math.cos(a / 2), math.sin(a / 2), 0.0, 0.0]
    want = iorc.match([(cloud, hgrid, igrid, intensities)], init[:3], init, [FIXTURE_INTENSITY],
                      **FIXTURE_OPTIONS)
    expected = [-1, 0, 0, math.cos(-rotate / 2), 0, 0, math.sin(-rotate / 2)]
    assert want["final_cost"] <= 1e-2
    assert is_nearly(want["pose"], expected, 3e-2)


def test_interpolated_intensity_equals_voxel_values_at_centres(oracle):
    rng = np.random.RandomState(4)
    pts = rng.uniform(-1.0, 1.0, (60, 3)).astype(np.float32)
    _, igrid = intensity_grid(oracle, 0.25, pts, rng.uniform(1, 200, 60).astype(np.float32))
    res = float(np.float32(0.25))
    for x in np.arange(-1.25, 1.3, res):
        for y in np.arange(-1.25, 1.3, 2 * res):
            for z in (-0.5, 0.0, 0.75):
                c = oracle.hybrid_get_cell_index(0.25, [x, y, z])
                assert iorc.interpolated_intensity(igrid, c[0] * res, c[1] * res, c[2] * res) == \
                    pytest.approx(igrid.get_intensity(*c), abs=1e-4)


def test_get_intensity_is_the_float_mean_and_zero_where_empty(oracle):
    grid = iorc.IntensityHybridGrid(0.5)
    for v in (10.0, 20.0, 31.0):
        grid.add_intensity((1, 2, 3), v)
    assert grid.get_intensity(1, 2, 3) == float(np.float32(61.0) / np.float32(3))
    assert grid.get_intensity(0, 0, 0) == 0.0
    empty = iorc.IntensityHybridGrid(0.5, [[4, 4, 4]], [0.0], [0])
    assert empty.get_intensity(4, 4, 4) == 0.0


def _random_intensity_case(oracle, seed, n=40):
    rng = np.random.RandomState(seed)
    shifted = POINTS + np.array([-1, 0, 0], np.float32)
    _, hgrid = hybrid(oracle, 0.5, shifted)
    surf = shifted[rng.randint(0, 7, 300)] + rng.uniform(-0.4, 0.4, (300, 3))
    _, igrid = intensity_grid(oracle, 0.5, surf.astype(np.float32),
                              rng.uniform(10, 90, 300).astype(np.float32))
    cloud = (POINTS[rng.randint(0, 7, n)] + rng.uniform(-0.3, 0.3, (n, 3))).astype(np.float32)
    intensities = rng.uniform(5, 120, n).astype(np.float32)
    q = np.array([1.0, 0.03, -0.02, 0.05])
    pose = np.concatenate([[-0.93, 0.04, -0.03], q / np.linalg.norm(q)])
    return cloud, intensities, hgrid, igrid, pose


def test_intensity_rows_match_central_differences(oracle):
    cloud, intensities, hgrid, igrid, pose = _random_intensity_case(oracle, 5)
    entries = [(cloud, hgrid, igrid, intensities)]
    io = [(2.0, 1.0, 100.0)]
    tq = [1.0, 0.0, 0.0, 0.0]
    _, jac = iorc.evaluate(entries, pose, pose[:3], tq, io, occupied_space_weights=[1.0])
    n = len(cloud)
    rows = slice(n, 2 * n)
    assert np.abs(jac[rows]).max() > 1.0
    h = 1e-6
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        rp, _ = iorc.evaluate(entries, plus(pose, d), pose[:3], tq, io,
                              occupied_space_weights=[1.0], jacobian=False)
        rm, _ = iorc.evaluate(entries, plus(pose, -d), pose[:3], tq, io,
                              occupied_space_weights=[1.0], jacobian=False)
        fd = (rp[rows] - rm[rows]) / (2 * h)
        assert np.allclose(fd, jac[rows, k], rtol=1e-4, atol=1e-4)
    # returns brighter than the threshold: zero residual and zero row
    bright = intensities > 100.0
    assert bright.any()
    r, _ = iorc.evaluate(entries, pose, pose[:3], tq, io,
                                             occupied_space_weights=[1.0])
    assert np.all(r[rows][bright] == 0.0) and np.all(jac[rows][bright] == 0.0)


@pytest.mark.parametrize("huber_scale", [0.3, 1e4])
def test_huber_corrected_gradient_matches_central_differences(oracle, huber_scale):
    """Both branches of HuberLoss: s_b > a^2 (outliers, a = 0.3) and s_b <= a^2."""
    cloud, intensities, hgrid, igrid, pose = _random_intensity_case(oracle, 6)
    entries = [(cloud, hgrid, igrid, intensities)]
    io = [(2.0, huber_scale, 100.0)]
    tq = [1.0, 0.0, 0.0, 0.0]
    kw = dict(occupied_space_weights=[1.0])
    r, _ = iorc.evaluate(entries, pose, pose[:3], tq, io, jacobian=False, **kw)
    n = len(cloud)
    sb = float(np.sum(r[n:2 * n] ** 2))
    assert (sb > huber_scale ** 2) == (huber_scale == 0.3)
    cost, g, _ = iorc.normal(entries, pose, pose[:3], tq, io, **kw)
    rho = sb if sb <= huber_scale ** 2 else 2 * huber_scale * math.sqrt(sb) - huber_scale ** 2
    plain = float(np.sum(r[:n] ** 2) + np.sum(r[2 * n:] ** 2))
    assert cost == pytest.approx(0.5 * (plain + rho), rel=1e-12)
    h = 1e-6
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        cp = iorc.normal(entries, plus(pose, d), pose[:3], tq, io, **kw)[0]
        cm = iorc.normal(entries, plus(pose, -d), pose[:3], tq, io, **kw)[0]
        assert (cp - cm) / (2 * h) == pytest.approx(g[k], rel=1e-4, abs=1e-5)


def test_block_above_the_threshold_contributes_nothing(oracle):
    cloud, intensities, hgrid, igrid, pose = _random_intensity_case(oracle, 7)
    tq = [1.0, 0.0, 0.0, 0.0]
    kw = dict(occupied_space_weights=[1.0])
    bright = np.full(len(cloud), 150.0, np.float32)
    with_block = iorc.normal([(cloud, hgrid, igrid, bright)], pose, pose[:3],
                                                 tq, [(2.0, 0.3, 100.0)], **kw)
    without = iorc.normal([(cloud, hgrid)], pose, pose[:3], tq, [None], **kw)
    assert with_block[0] == without[0]
    assert np.array_equal(with_block[1], without[1]) and np.array_equal(with_block[2], without[2])


@pytest.mark.parametrize("seed,nonmonotonic", [(8, True), (9, False)])
def test_minimiser_loop_equals_the_cpp_oracle_without_intensity(oracle, seed, nonmonotonic):
    """The restated loop on the problem without intensity blocks is the C++ oracle's loop
    (sums over points are numpy's here, so to 1e-9 rather than bit for bit)."""
    cloud, intensities, hgrid, igrid, pose = _random_intensity_case(oracle, seed, n=300)
    init = list(pose)
    opts = dict(FIXTURE_OPTIONS, use_nonmonotonic_steps=nonmonotonic, max_num_iterations=12)
    want = oracle.ceres3d_match([(cloud, hgrid)], init[:3], init, **opts)
    got = iorc.match([(cloud, hgrid, None, intensities)], init[:3], init, [None], **opts)
    assert np.allclose(got["pose"], want["pose"], rtol=0, atol=1e-9)
    assert got["initial_cost"] == pytest.approx(want["initial_cost"], rel=1e-12)
    assert got["final_cost"] == pytest.approx(want["final_cost"], rel=1e-9)
    for k in ("iterations", "num_successful_steps", "termination"):
        assert got[k] == want[k]
