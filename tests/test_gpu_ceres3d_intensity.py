"""Device CeresScanMatcher3D with intensity blocks (csm_intensity_grid3d,
csm_ceres_match3d_intensity_batch, csm_ceres_evaluate3d_intensity) against the reference's
known answers (intensity_cost_function_3d_test.cc, ceres_scan_matcher_3d_test.cc with its
intensity block) and the intensity restatement (tests/intensity3d_oracle.py).  Tolerances as in test_gpu_ceres3d.py:
uncorrected residuals and rows to 1e-12, solved poses to 1e-7."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic
from cartographer_b200 import scan_matching as sm
from cartographer_b200._lib import CsmError, lib, ptr
from tests import intensity3d_oracle as iorc
from tests.test_gpu_ceres3d import _same_solution
from tests.test_oracle_golden_3d import is_nearly
from tests.test_oracle_intensity3d_cpu import FIXTURE_INTENSITY, fixture

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-7


def _fixture_matcher():
    return sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
        occupied_space_weight_0=1.0, translation_weight=0.01, rotation_weight=0.1,
        use_nonmonotonic_steps=True, max_num_iterations=10,
        intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(*FIXTURE_INTENSITY)))


def _device(hspec, ispec):
    return (sm.DeviceHybridGrid(synthetic.HybridGridSpec(*hspec)),
            sm.DeviceIntensityGrid(sm.IntensityGridSpec(*ispec)))


# intensity_cost_function_3d_test.cc:37-61
def test_intensity_cost_function_smoke_test_on_device(oracle):
    cloud = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2]], np.float32)
    intensities = np.array([50, 100, 150], np.float32)
    idx = np.array([oracle.hybrid_get_cell_index(0.3, [0, 0, 0])], np.int32)
    dint = sm.DeviceIntensityGrid(sm.IntensityGridSpec(0.3, idx, [50.0], [1]))
    dhi = sm.DeviceHybridGrid(synthetic.HybridGridSpec(0.3, idx, [oracle.probability_to_value(1.0)]))
    m = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
        occupied_space_weight_0=1.0,
        intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(
            math.sqrt(3.0), 1.0, 100.0)))                 # scaling_factor = 1
    res, _ = m.Evaluate([(cloud, dhi, dint, intensities)], [0, 0, 0, 1, 0, 0, 0], [0, 0, 0],
                        [1, 0, 0, 0])
    assert np.allclose(res[3:6], [0.0, -100.0, 0.0], rtol=0, atol=1e-9)
    dint.close()
    dhi.close()


# ceres_scan_matcher_3d_test.cc:99-131 with the fixture's intensity block
@pytest.mark.parametrize("start,rotate", [((-1.0, 0.0, 0.0), 0.0), ((-0.8, 0.0, 0.0), 0.0),
                                          ((-1.0, 0.0, -0.2), 0.0), ((-0.9, -0.2, 0.2), 0.0),
                                          ((-0.95, -0.05, 0.05), 0.05)])
def test_reference_fixture_with_intensity_on_device(oracle, start, rotate):
    cloud, intensities, hspec, hgrid, ispec, igrid = fixture(oracle, rotate)
    dhi, dint = _device(hspec, ispec)
    a = 0.05 if rotate else 0.0
    init = list(start) + [math.cos(a / 2), math.sin(a / 2), 0.0, 0.0]
    pose, summary = _fixture_matcher().Match(init[:3], init, [(cloud, dhi, dint, intensities)])
    assert summary["final_cost"] <= 1e-2
    assert is_nearly(pose, [-1, 0, 0, math.cos(-rotate / 2), 0, 0, math.sin(-rotate / 2)], 3e-2)
    _same_solution(pose, summary, iorc.match(
        [(cloud, hgrid, igrid, intensities)], init[:3], init, [FIXTURE_INTENSITY],
        occupied_space_weights=[1.0], translation_weight=0.01, rotation_weight=0.1,
        use_nonmonotonic_steps=True, max_num_iterations=10))
    dhi.close()
    dint.close()


@pytest.fixture(scope="module")
def config5(oracle):
    """BASELINE config-5 size: 64 rings x 1024 azimuths (~64 k points) against the 10 cm /
    45 cm grids of a 40 m building, with an intensity grid over the 10 cm voxels."""
    hi, lo, _, world = synthetic.make_submap3d(41, 40.0, 64, 1024, 20.0)
    rng = np.random.RandomState(541)
    node = synthetic.make_node3d(world, rng, 64, 1024, 20.0, seed=7100, jitter=0.15)
    inten = synthetic.node_intensities(world, node, 7100)
    ispec = synthetic.make_intensity_grid3d(hi, world, 41)
    dev = (sm.DeviceHybridGrid(hi), sm.DeviceHybridGrid(lo), sm.DeviceIntensityGrid(ispec))
    orc = (oracle.HybridGrid(hi.resolution, hi.indices, hi.values),
           oracle.HybridGrid(lo.resolution, lo.indices, lo.values),
           iorc.IntensityHybridGrid(ispec.resolution, ispec.indices, ispec.sums, ispec.counts))
    yield node, inten, dev, orc
    for d in dev:
        d.close()


def _opts(huber_scale, **kw):
    return sm.CeresScanMatcherOptions3D(
        intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(0.5, huber_scale, 100.0),
        **kw)


@pytest.mark.parametrize("huber_scale", [0.3, 55.0])
def test_config5_residuals_and_rows_equal_the_oracle(oracle, config5, huber_scale):
    node, inten, (dhi, dlo, dint), (ohi, olo, oint) = config5
    assert len(node["cloud"]) > 40000 and (inten > 100.0).any()
    q = np.array([math.cos(0.03), 0.01, -0.02, math.sin(0.03)])
    pose = np.concatenate([node["pose"][:3] + [0.04, -0.03, 0.02], q / np.linalg.norm(q)])
    m = sm.CeresScanMatcher3D(_opts(huber_scale))
    for with_jac in (True, False):
        got_r, got_j = m.Evaluate([(node["cloud"], dhi, dint, inten), (node["low"], dlo)], pose,
                                  node["pose"][:3], node["pose"][3:], jacobian=with_jac)
        want_r, want_j = iorc.evaluate(
            [(node["cloud"], ohi, oint, inten), (node["low"], olo)], pose, node["pose"][:3],
            node["pose"][3:], [(0.5, huber_scale, 100.0), None], jacobian=with_jac)
        n = len(node["cloud"])
        assert got_r.shape == want_r.shape == (2 * n + len(node["low"]) + 6,)
        assert np.allclose(got_r, want_r, rtol=0, atol=1e-12)
        assert np.abs(want_r[n:2 * n]).max() > 0.01
        if with_jac:
            assert np.allclose(got_j, want_j, rtol=0, atol=1e-12)


@pytest.mark.parametrize("huber_scale,nonmonotonic", [(0.3, False), (0.3, True), (55.0, False)])
def test_config5_match_equals_the_oracle(oracle, config5, huber_scale, nonmonotonic):
    node, inten, (dhi, dlo, dint), (ohi, olo, oint) = config5
    m = sm.CeresScanMatcher3D(_opts(huber_scale, use_nonmonotonic_steps=nonmonotonic,
                                    max_num_iterations=12))
    rng = np.random.RandomState(int(huber_scale) + nonmonotonic)
    init = node["pose"].copy()
    init[:3] += rng.uniform(-0.05, 0.05, 3)
    yaw = 2 * math.atan2(node["pose"][6], node["pose"][3]) + rng.uniform(-0.01, 0.01)
    init[3:] = [math.cos(yaw / 2), 0, 0, math.sin(yaw / 2)]
    pose, summary = m.Match(init[:3], init, [(node["cloud"], dhi, dint, inten),
                                             (node["low"], dlo)])
    want = iorc.match(
        [(node["cloud"], ohi, oint, inten), (node["low"], olo)], init[:3], init,
        [(0.5, huber_scale, 100.0), None], use_nonmonotonic_steps=nonmonotonic,
        max_num_iterations=12)
    _same_solution(pose, summary, want)
    assert summary["final_cost"] <= summary["initial_cost"]


def test_mixed_batch_equals_single_calls(oracle, config5):
    """Jobs with and without intensity blocks (on either cloud) in one launch; the jobs without
    one also equal csm_ceres_match3d_batch bit for bit."""
    node, inten, (dhi, dlo, dint), _ = config5
    low_inten = np.random.RandomState(3).uniform(5, 120, len(node["low"])).astype(np.float32)
    opts = _opts(0.3)
    opts.intensity_cost_function_options_1 = sm.IntensityCostFunctionOptions(2.0, 1.0, 100.0)
    m = sm.CeresScanMatcher3D(opts)
    entries = [[(node["cloud"], dhi, dint, inten), (node["low"], dlo)],
               [(node["cloud"], dhi), (node["low"], dlo)],
               [(node["cloud"], dhi), (node["low"], dlo, dint, low_inten)],
               [(node["cloud"], dhi, None, inten), (node["low"], dlo)]]
    inits = []
    for k in range(len(entries)):
        init = node["pose"].copy()
        init[:3] += [0.03 * (k - 1), -0.02 * k, 0.01 * k]
        inits.append(init)
    poses, sums = m.MatchBatch([i[:3] for i in inits], inits, entries)
    assert m.last_stats["host_syncs"] == 1
    for init, e, p, s in zip(inits, entries, poses, sums):
        p1, s1 = m.Match(init[:3], init, e)
        assert np.array_equal(p, p1) and s == s1
    plain = [1, 3]
    pp, ps = sm.CeresScanMatcher3D(opts).MatchBatch(
        [inits[k][:3] for k in plain], [inits[k] for k in plain],
        [[(e[0], e[1]) for e in entries[k]] for k in plain])
    for i, k in enumerate(plain):
        assert np.array_equal(pp[i], poses[k]) and ps[i] == sums[k]
    assert not np.array_equal(poses[0], poses[1])


def test_empty_intensity_grid_reads_zero(oracle):
    cloud, intensities, hspec, _, _, _ = fixture(oracle)
    dhi = sm.DeviceHybridGrid(synthetic.HybridGridSpec(*hspec))
    empty = sm.DeviceIntensityGrid(sm.IntensityGridSpec(1.0, np.zeros((0, 3), np.int32), [], []))
    m = _fixture_matcher()
    pose = [-0.9, 0.1, 0.0, 1.0, 0.0, 0.0, 0.0]
    res, _ = m.Evaluate([(cloud, dhi, empty, intensities)], pose, pose[:3], pose[3:])
    n = len(cloud)
    assert np.array_equal(res[n:2 * n], 0.5 / math.sqrt(n) * (0.0 - intensities.astype(np.float64)))
    dhi.close()
    empty.close()


def test_invalid_intensity_options_are_rejected(oracle):
    cloud, intensities, hspec, _, ispec, _ = fixture(oracle)
    dhi, dint = _device(hspec, ispec)
    init = [-1.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    for bad in ((0.0, 55.0, 100.0), (0.5, 0.0, 100.0), (0.5, 55.0, 0.0), (0.5, -1.0, 100.0)):
        m = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
            occupied_space_weight_0=1.0,
            intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(*bad)))
        with pytest.raises(CsmError) as e:
            m.Match(init[:3], init, [(cloud, dhi, dint, intensities)])
        assert e.value.status == 1
    # options of a cloud without an intensity grid are not read
    m = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
        occupied_space_weight_0=1.0,
        intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(*FIXTURE_INTENSITY)))
    m.Match(init[:3], init, [(cloud, dhi, dint, intensities), (cloud, dhi)])
    # a grid without intensities
    xyz = np.ascontiguousarray(cloud, np.float32)
    job, ijob = sm.CsmCeresJob3D(), sm.CsmCeresIntensityJob3D()
    job.num_clouds, job.grid[0], job.xyz[0], job.num_points[0] = 1, dhi._h, ptr(xyz, C.c_float), 7
    for k in range(7):
        job.initial_pose[k] = init[k]
    ijob.intensity_grid[0] = dint._h
    opt, iopt = m.options._c(), m.options._c_intensity()
    res = sm.CsmCeresResult3D()
    assert lib().csm_ceres_match3d_intensity_batch(C.byref(job), C.byref(ijob), 1, C.byref(opt),
                                                   C.byref(iopt), C.byref(res), None) == 1
    assert lib().csm_ceres_match3d_intensity_batch(C.byref(job), None, 1, C.byref(opt),
                                                   C.byref(iopt), C.byref(res), None) == 1
    dhi.close()
    dint.close()
