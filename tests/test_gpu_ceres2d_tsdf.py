"""CeresScanMatcher2D on TSDF2D submaps (TSDFMatchCostFunction2D) on the device, against the
CPU restatement tests/tsdf2d_oracle.py; and the TSDF2D device grid handle."""
import numpy as np
import pytest

from benchmarks import synthetic
from tests import tsdf2d_oracle as T
from tests.test_tsdf_known_answers_cpu import (KNOWN_ANSWERS, MATCHING_CLOUD,
                                              reference_cost_fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _world(seed, size_cells=200, beams=181, max_range=8.0, scans=3):
    spec, occ = synthetic.make_tsdf2d(seed, size_cells=size_cells)
    rng = np.random.RandomState(seed)
    out = []
    for k in range(scans):
        pose = synthetic.random_free_pose(occ, spec, rng, margin_cells=20)
        out.append((pose, synthetic.cast_scan(occ, spec, pose, beams=beams, max_range=max_range,
                                              seed=seed + k)))
    return spec, occ, out


def _same_summary(got, want, atol=1e-7):
    pose, s = got
    assert np.allclose(pose, want["pose"], rtol=0, atol=atol), (pose, want)
    assert s["termination"] == want["termination"]
    assert s["iterations"] == want["iterations"]
    assert s["num_successful_steps"] == want["num_successful_steps"]
    if want["termination"] != "EVALUATION_FAILED" or want["initial_cost"] != -1.0:
        assert s["initial_cost"] == pytest.approx(want["initial_cost"], rel=1e-12)
        assert s["final_cost"] == pytest.approx(want["final_cost"], rel=1e-7, abs=1e-15)
    else:
        assert s["initial_cost"] == -1.0 and s["final_cost"] == -1.0


def test_residuals_and_jacobian_equal_the_oracle(sm):
    spec, _, scans = _world(3)
    g = T.TSDF2D.from_spec(spec)
    dev = sm.RealTimeGrid2D(spec)
    m = sm.CeresScanMatcher2D()
    try:
        for pose, scan in scans:
            x = pose + np.array([0.02, -0.01, 0.015])
            r, j, valid = m.EvaluateChecked(dev, scan, x, x[:2] + 0.01, x[2] - 0.02)
            rw, jw, vw = T.evaluate(g, scan, x, x[:2] + 0.01, x[2] - 0.02)
            assert valid and vw
            assert np.allclose(r, rw, rtol=1e-12, atol=1e-12 * np.abs(rw).max())
            assert np.allclose(j, jw, rtol=1e-10, atol=1e-10 * np.abs(jw).max())
            r2, j2, valid2 = m.EvaluateChecked(dev, scan, x, x[:2], x[2], jacobian=False)
            rw2, _, _ = T.evaluate(g, scan, x, x[:2], x[2], jacobian=False)
            assert valid2 and j2 is None
            assert np.allclose(r2, rw2, rtol=1e-12, atol=1e-12 * np.abs(rw2).max())
        # the scan far outside the grid: the cost function fails
        far = np.array([500.0, 500.0, 0.0])
        _, _, valid = m.EvaluateChecked(dev, scans[0][1], far, far[:2], 0.0)
        assert not valid and not T.evaluate(g, scans[0][1], far, far[:2], 0.0)[2]
    finally:
        dev.close()


def _device_grid(sm, g):
    return sm.RealTimeGrid2D(sm.TSDF2DSpec(g.tsd_cells, g.weight_cells, g.resolution, g.max_x,
                                           g.max_y, g.truncation_distance, g.max_weight))


@pytest.mark.parametrize("y,residual,jacobian", KNOWN_ANSWERS)
def test_reference_cost_function_known_answers_on_the_device(sm, y, residual, jacobian):
    """tsdf_match_cost_function_2d_test.cc on the grid the restated TSDFRangeDataInserter2D
    builds (ExactInitialPose, PertubatedInitialPose, InvalidInitialPose), through
    csm_ceres_evaluate2d_checked with scaling 1."""
    dev = _device_grid(sm, reference_cost_fixture())
    m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(occupied_space_weight=1.0))
    try:
        pose = [0.0, y, 0.0]
        r, j, valid = m.EvaluateChecked(dev, MATCHING_CLOUD, pose, pose[:2], 0.0)
        if residual is None:
            assert not valid
            return
        assert valid
        assert abs(r[0] - residual) < 1e-3
        assert np.allclose(j[0], jacobian, rtol=0, atol=1e-3)
    finally:
        dev.close()


def test_match_empty_tsdf_on_the_device(sm):
    dev = _device_grid(sm, reference_cost_fixture(insert=False))
    m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(occupied_space_weight=1.0))
    try:
        _, _, valid = m.EvaluateChecked(dev, np.zeros((1, 3), np.float32), [0.0, 0.0, 0.0],
                                        [0.0, 0.0], 0.0)
        assert not valid
        pose, s = m.Match([0.0, 0.0], [0.1, 0.2, 0.05], MATCHING_CLOUD, dev)
        assert s["termination"] == "EVALUATION_FAILED"
        assert np.array_equal(pose, [0.1, 0.2, 0.05])
    finally:
        dev.close()


def test_probability_update_refuses_a_tsdf_handle(sm):
    """csm_rt_grid2d_update would leave the weight cells stale: it refuses TSDF handles."""
    from cartographer_b200._lib import CsmError, lib, ptr
    import ctypes as C
    g = reference_cost_fixture()
    dev = _device_grid(sm, g)
    try:
        cells = np.ascontiguousarray(g.tsd_cells)
        with pytest.raises(CsmError):
            sm.check(lib().csm_rt_grid2d_update(dev._h, ptr(cells, C.c_uint16)))
        with pytest.raises(ValueError):
            dev.update(g.tsd_cells)
    finally:
        dev.close()


@pytest.mark.parametrize("nonmonotonic", [True, False])
def test_solved_poses_equal_the_oracle(sm, nonmonotonic):
    spec, _, scans = _world(7, scans=4)
    g = T.TSDF2D.from_spec(spec)
    dev = sm.RealTimeGrid2D(spec)
    opts = sm.CeresScanMatcherOptions2D(use_nonmonotonic_steps=nonmonotonic,
                                        max_num_iterations=20)
    m = sm.CeresScanMatcher2D(opts)
    rng = np.random.RandomState(11)
    try:
        for pose, scan in scans:
            init = pose + np.array([rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05),
                                    rng.uniform(-0.02, 0.02)])
            got = m.Match(init[:2], init, scan, dev)
            want = T.match(g, scan, init[:2], init, 20.0, 10.0, 1.0, nonmonotonic, 20)
            _same_summary(got, want)
    finally:
        dev.close()


def test_mixed_batch_equals_single_calls(sm):
    devs, jobs = [], []
    rng = np.random.RandomState(5)
    try:
        for s in range(3):
            tspec, occ, tscans = _world(20 + s, scans=2)
            pgrid, pocc = synthetic.make_grid2d(30 + s, size_cells=200)
            tdev, pdev = sm.RealTimeGrid2D(tspec), sm.RealTimeGrid2D(pgrid)
            devs += [tdev, pdev]
            ppose = synthetic.random_free_pose(pocc, pgrid, rng, margin_cells=20)
            pscan = synthetic.cast_scan(pocc, pgrid, ppose, beams=181, max_range=8.0, seed=s)
            for pose, scan in tscans:
                jobs.append((tdev, scan, pose + np.array([0.03, -0.02, 0.01])))
            jobs.append((pdev, pscan, ppose + np.array([-0.02, 0.03, -0.01])))
        jobs.append((devs[0], jobs[0][1], np.array([500.0, 500.0, 0.0])))   # fails at the start
        m = sm.CeresScanMatcher2D()
        poses, sums = m.MatchBatch([j[2][:2] for j in jobs], [j[2] for j in jobs],
                                   [j[1] for j in jobs], [j[0] for j in jobs])
        for k, (dev, scan, init) in enumerate(jobs):
            p1, s1 = m.Match(init[:2], init, scan, dev)
            assert np.array_equal(poses[k], p1)
            assert sums[k] == s1
        assert sums[-1]["termination"] == "EVALUATION_FAILED"
    finally:
        for d in devs:
            d.close()


def test_baseline_size_tsdf(sm):
    spec, occ = synthetic.make_tsdf2d(900, size_cells=1000)
    g = T.TSDF2D.from_spec(spec)
    rng = np.random.RandomState(900)
    dev = sm.RealTimeGrid2D(spec)
    m = sm.CeresScanMatcher2D()
    try:
        for k in range(2):
            pose = synthetic.random_free_pose(occ, spec, rng, margin_cells=40)
            scan = synthetic.cast_scan(occ, spec, pose, beams=1081, seed=k)
            init = pose + np.array([0.03, -0.04, 0.01])
            _same_summary(m.Match(init[:2], init, scan, dev),
                          T.match(g, scan, init[:2], init))
    finally:
        dev.close()


def test_rt_batch_on_a_tsdf_handle_equals_the_per_call_form(sm):
    spec, occ, scans = _world(41, scans=4)
    rt = sm.RealTimeCorrelativeScanMatcher2D(
        sm.RealTimeCorrelativeScanMatcherOptions(0.1, 0.12, 0.1, 0.1))
    dev = sm.RealTimeGrid2D(spec)
    try:
        inits = [p + np.array([0.04, -0.03, 0.02]) for p, _ in scans]
        sb, pb, _ = rt.MatchBatch(inits, [s for _, s in scans], dev)
        for k, (_, scan) in enumerate(scans):
            s1, p1 = rt.MatchTSDF(inits[k], scan, spec)
            assert sb[k] == s1 and np.array_equal(pb[k], p1)
        # update(): the handle follows new cells
        spec2, _ = synthetic.make_tsdf2d(42, size_cells=200)
        dev.update(spec2.tsd_cells, spec2.weight_cells)
        sb2, pb2, _ = rt.MatchBatch(inits[:1], [scans[0][1]], dev)
        s2, p2 = rt.MatchTSDF(inits[0], scans[0][1], spec2)
        assert sb2[0] == s2 and np.array_equal(pb2[0], p2)
    finally:
        dev.close()
