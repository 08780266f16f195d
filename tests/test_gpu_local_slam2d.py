"""LocalTrajectoryBuilder2D on the device against the recipe: the same scans through the
existing public calls (voxel_filter_batch, adaptive_voxel_filter_batch,
RealTimeCorrelativeScanMatcher2D.MatchBatch, CeresScanMatcher2D.Match, MotionFilter,
ActiveSubmaps2D.InsertRangeData) with the per-point transforms of the float32 restatement."""
import math

import numpy as np
import pytest

from benchmarks.local_slam2d_recipe import _quat_yaw, run
from cartographer_b200 import local_slam as L
from cartographer_b200 import scan_matching as sm
from cartographer_b200._lib import CsmError
from tests import local_slam2d_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("online,accumulate", [(False, 1), (True, 1), (False, 2), (True, 2)])
def test_builder_equals_recipe(online, accumulate):
    o = L.LocalTrajectoryBuilderOptions2D(min_range=0.2, num_accumulated_range_data=accumulate,
                                          use_online_correlative_scan_matching=online)
    o.submaps_options = sm.SubmapsOptions2D(num_range_data=10)
    o.motion_filter_options = L.MotionFilterOptions(max_distance_meters=0.15)
    b, matched, dropped, inserted = run(o, 300 if accumulate == 1 else 60)
    assert matched > 0 and inserted > 0
    if accumulate == 1:
        assert any(s.insertion_finished for s in b.active_submaps.submaps()) or \
            inserted >= 20
    b.close()


def test_dropped_and_miss_only_scans():
    o = L.LocalTrajectoryBuilderOptions2D(min_range=0.2)
    o.submaps_options = sm.SubmapsOptions2D(num_range_data=10)

    def tweak(k, hw):
        hw = hw.copy()
        if k == 5:
            hw[:, 2] = 5.0            # wholly above max_z: dropped
        if k == 8:
            hw[:, :3] *= 50.0         # every hit beyond max_range: misses only, dropped
        return hw
    b, matched, dropped, inserted = run(o, 12, tweak)
    assert dropped == 2 and matched == 10
    b.close()


def test_hooks_and_refusals():
    o = L.LocalTrajectoryBuilderOptions2D(min_range=0.2)
    slam = L.LocalSlam2D(o)
    pose = L.rigid3f((1.0, 2.0, 0.0), L._quatd_mul(_quat_yaw(0.3), (1, 0, 0, 0)))
    hits = np.array([[0.2, 0, 0], [30, 0, 0], [np.nextafter(np.float32(30), np.float32(31)), 0, 0],
                     [0.1, 0, 0], [3, 4, 1]], np.float32)
    origins = np.array([[0, 0, 0], [0.1, 0, 0]], np.float32)
    oi = np.array([0, 0, 0, 0, 1], np.int32)
    st = slam.accumulate(hits, origins, oi, L._flat(pose)[None], np.zeros(5, np.int32))
    assert st["host_syncs"] == 0
    r, m = O.accumulate(hits, origins, oi, [pose], [0] * 5, 0.2, 30.0, 5.0)
    assert np.array_equal(slam.read(L.ACCUMULATED_RETURNS), r)
    assert np.array_equal(slam.read(L.ACCUMULATED_MISSES), m)
    before = slam.read(L.ACCUMULATED_RETURNS)
    bad = hits.copy()
    bad[0, 0] = np.nan
    for args in [(bad, origins, oi, L._flat(pose)[None], np.zeros(5, np.int32)),
                 (hits, origins, oi + 5, L._flat(pose)[None], np.zeros(5, np.int32)),
                 (hits, origins, oi, L._flat(pose)[None], np.ones(5, np.int32))]:
        with pytest.raises(CsmError) as e:
            slam.accumulate(*args)
        assert e.value.status == 1
    assert np.array_equal(slam.read(L.ACCUMULATED_RETURNS), before)
    T = L.rigid3f((0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))
    res, st = slam.match(L._flat(T), (1, 2, 0), (0, 0, 0), None)
    assert res.status == L.MATCHED and st["host_syncs"] == 2
    assert np.array_equal(slam.read(L.CROPPED_RETURNS), O.crop(O.transform(r, T), -0.8, 2.0))
    with pytest.raises(CsmError):
        slam.match(L._flat(T), (1, 2, 0), (0, 0, 0), None)   # nothing accumulated
    g = sm.RealTimeGrid2D.empty(*sm.create_grid_limits((1, 2), 0.05))
    org, st = slam.insert(L._flat(L.embed3d_f((0.1, 0.2, 0.3))), [g])
    assert st["host_syncs"] == 2
    with pytest.raises(CsmError):
        slam.insert(L._flat(L.embed3d_f((0.1, 0.2, 0.3))), [g])   # inserted already
    g.close()
    slam.close()


def test_loop_closes_on_finished_submap():
    o = L.LocalTrajectoryBuilderOptions2D(min_range=0.2)
    o.submaps_options = sm.SubmapsOptions2D(num_range_data=5)
    o.motion_filter_options = L.MotionFilterOptions(max_distance_meters=0.0)
    b, matched, dropped, inserted = run(o, 10)   # the first submap finishes at its 10th scan
    finished = [s for s in b.active_submaps.submaps() if s.insertion_finished]
    assert finished
    sub = finished[0].constraint_builder_submap()
    stack = sm.FastCorrelativeScanMatcher2D(sub.grid.read(), sm.FastCorrelativeScanMatcherOptions2D(
        7.0, math.radians(30.0), 7))
    cloud = b.slam.read(L.FILTERED)
    found, score, _ = stack.MatchFullSubmap(cloud, 0.2)
    assert found and score > 0.2
    stack.close()
    b.close()


def test_accumulation_past_one_launch_of_capped_blocks():
    """More than 2^24 crop entries (2 x 9 M accumulated points) and a 9 M-hit scan: every
    entry is transformed, cropped and compacted, in order."""
    o = L.LocalTrajectoryBuilderOptions2D(min_range=0.0, max_range=30.0)
    slam = L.LocalSlam2D(o)
    n = 9_000_000
    i = np.arange(n)
    hits = np.zeros((n, 3), np.float32)
    hits[:, 0] = np.float32(1.0) + (i % 1000).astype(np.float32) * np.float32(0.001)
    hits[:, 1] = 0.5
    hits[i % 3 == 1, 0] = 40.0                         # beyond max_range: misses
    hits[:, 2] = np.where(i % 2 == 0, 0.25, 5.0)       # every other point above max_z
    ident = L.rigid3f((0, 0, 0), (1, 0, 0, 0))
    slam.accumulate(hits, np.zeros((1, 3), np.float32), np.zeros(n, np.int32),
                    L._flat(ident)[None], np.zeros(n, np.int32))
    ret_mask = i % 3 != 1
    assert len(slam.read(L.ACCUMULATED_RETURNS)) == ret_mask.sum()
    res, st = slam.match(L._flat(ident), (0, 0, 0), (0, 0, 0), None)
    assert res.status == L.MATCHED and st["host_syncs"] == 2
    cr = slam.read(L.CROPPED_RETURNS)
    assert cr.tobytes() == hits[ret_mask & (hits[:, 2] <= 2.0)].tobytes()
    cm = slam.read(L.CROPPED_MISSES)
    # a miss lies 5 m along its ray, so even a hit above max_z leaves a miss below it
    assert len(cm) == (~ret_mask).sum() and (cm[:, 2] <= np.float32(2.0)).all()
    slam.close()


def test_refusals_leave_the_builder_unchanged():
    o = L.LocalTrajectoryBuilderOptions2D(min_range=0.2)
    slam = L.LocalSlam2D(o)
    ident = L.rigid3f((0, 0, 0), (1, 0, 0, 0))
    hits = np.array([[1, 0, 0], [0, 2, 0], [3, 3, 0]], np.float32)
    slam.accumulate(hits, np.zeros((1, 3), np.float32), np.zeros(3, np.int32),
                    L._flat(ident)[None], np.zeros(3, np.int32))
    before = slam.read(L.ACCUMULATED_RETURNS)
    tsdf = sm.RealTimeGrid2D.empty_tsdf(0.05, 2.5, 2.5, 0.3, 10.0)
    with pytest.raises(CsmError) as e:
        slam.match(L._flat(ident), (0, 0, 0), (0, 0, 0), tsdf)
    assert e.value.status == 1
    bad = L._flat(ident)
    bad[3] = np.inf
    with pytest.raises(CsmError):
        slam.match(bad, (0, 0, 0), (0, 0, 0), None)
    assert slam.read(L.ACCUMULATED_RETURNS).tobytes() == before.tobytes()
    res, _ = slam.match(L._flat(ident), (0, 0, 0), (0, 0, 0), None)
    assert res.status == L.MATCHED
    g = sm.RealTimeGrid2D.empty(*sm.create_grid_limits((0, 0), 0.05))
    info = g.read()
    for grids in ([tsdf], [g, g]):
        with pytest.raises(CsmError):
            slam.insert(L._flat(L.embed3d_f((0.0, 0.0, 0.1))), grids)
    far = L.embed3d_f((2000.0, 0.0, 0.1))                # would grow past 30000 cells
    with pytest.raises(CsmError):
        slam.insert(L._flat(far), [g])
    after = g.read()
    assert after.cells.tobytes() == info.cells.tobytes() and after.max_x == info.max_x
    org, st = slam.insert(L._flat(L.embed3d_f((0.0, 0.0, 0.1))), [g])   # still insertable
    assert st["host_syncs"] == 2 and len(slam.read(L.LOCAL_RETURNS)) == 3
    tsdf.close()
    g.close()
    slam.close()
