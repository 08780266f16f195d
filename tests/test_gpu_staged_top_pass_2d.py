"""A MatchFullSubmap batch is staged in groups of jobs (each group's rotation tables,
discretisation and tile-form lowest-resolution pass before the next group's tables).  A
batch of 16 such searches forms three groups; job for job it returns what each search
returns alone, in a batch of one group."""
import math

import numpy as np
import pytest

from benchmarks import synthetic

pytestmark = pytest.mark.gpu


def test_staged_full_submap_batch_equals_single_jobs():
    from cartographer_b200 import scan_matching as sm
    grid, occ = synthetic.make_grid2d(0, 1000)
    rng = np.random.RandomState(5)
    scans = []
    for i in range(16):
        pose = synthetic.random_free_pose(occ, grid, rng)
        scans.append(synthetic.cast_scan(occ, grid, pose, seed=300 + i))
    lin, ang, depth, min_score = 7.0, math.radians(30.0), 7, 0.6
    m = sm.FastCorrelativeScanMatcher2D(grid, sm.FastCorrelativeScanMatcherOptions2D(lin, ang, depth))
    clouds = [sm.DeviceCloud(s) for s in scans]
    jobs = np.zeros(len(scans), sm.JOB2D_DTYPE)
    jobs["cloud_index"] = np.arange(len(scans))
    jobs["full_submap"] = 1
    jobs["min_score"] = min_score
    res, _ = sm.match_batch([m], clouds, jobs, lin, ang)
    assert res["found"].sum() >= 1
    rotations = []
    for k in range(len(scans)):
        one, st1 = sm.match_batch([m], [clouds[k]], jobs[:1], lin, ang)
        rotations.append(st1["num_scans"])
        for name in res.dtype.names:
            np.testing.assert_array_equal(res[k][name], one[0][name], err_msg="%d %s" % (k, name))
    # groups start at >= 4096 rotations and grow 4x: with these sizes the batch has three
    # groups, and a single search (< 4096 rotations) has one
    assert max(rotations) < 4096 and sum(rotations) > 5 * 4096, rotations
    for c in clouds:
        c.close()
    m.close()
