"""Submap3D::InsertData into the active submaps on the device (csm_range_inserter3d_insert_submaps
and scan_matching.ActiveSubmaps3D) against two references after every scan: the same sequence
driven through the single-grid call (csm_range_inserter3d_insert) on data transformed and
filtered by the host restatement tests/submap_insert3d_oracle.cc, and the CPU inserter
tests/insert3d_oracle.py.  Every handle's dense box, voxels, intensity sums, counts and means
bit for bit; the lifecycle; the histograms; the refusals; ConstraintBuilder3D on a finished
submap."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from tests import insert3d_oracle as O
from tests.test_gpu_insert3d import assert_grid_equal, assert_igrid_equal

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
LUA = dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
           intensity_threshold=40.0)   # trajectory_builder_3d.lua submaps.range_data_inserter


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("submap_insert3d") / "libsubmap_insert3d_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                           os.path.join(ROOT, "tests", "submap_insert3d_oracle.cc"), "-o", so])
    return C.CDLL(so)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def host_transform(host, pose, origin, pts, max_range):
    pts = np.ascontiguousarray(pts, F).reshape(-1, 3)
    out_o, out_p = np.zeros(3, F), np.zeros_like(pts)
    kept = np.zeros(len(pts), np.uint8)
    host.submap_transform(_p(np.asarray(pose, np.float64), C.c_double),
                          _p(np.asarray(origin, F), C.c_float), _p(pts, C.c_float), len(pts),
                          C.c_float(max_range), _p(out_o, C.c_float), _p(out_p, C.c_float),
                          _p(kept, C.c_uint8))
    return out_o, out_p, kept.astype(bool)


class RefSubmap:
    """One submap inserted today's way: host transform and filter, then two single-grid calls
    on device handles, and the same into the CPU inserter's grids."""

    def __init__(self, sm, pose, hi_res=0.1, lo_res=0.45, intensity=True):
        self.pose = pose
        self.hi = (sm.DeviceHybridGrid.empty(hi_res), O.HybridGrid(hi_res))
        self.lo = (sm.DeviceHybridGrid.empty(lo_res), O.HybridGrid(lo_res))
        self.ig = ((sm.DeviceIntensityGrid.empty(hi_res), O.IntensityHybridGrid(hi_res))
                   if intensity else None)

    def insert(self, host, ins, origin, pts, inten, max_range):
        dev, ora = ins
        o, p, kept = host_transform(host, self.pose, origin, pts, max_range)
        ki = None if inten is None else np.asarray(inten, F)[kept]
        ig = self.ig
        dev.Insert(o, p[kept], ki, self.hi[0], None if ig is None else ig[0])
        ora.insert(o, p[kept], ki, self.hi[1], None if ig is None else ig[1])
        dev.Insert(o, p, None, self.lo[0])
        ora.insert(o, p, None, self.lo[1])


def assert_same(dev, ref, intensity=True):
    """dev: DeviceHybridGrid / DeviceIntensityGrid from the new call; ref: (device, oracle)."""
    if intensity:
        a, b = dev.read(), ref[0].read()
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x.view(np.uint32) if x.dtype == F else x,
                                          y.view(np.uint32) if y.dtype == F else y)
        assert_igrid_equal(dev, ref[1])
    else:
        (la, va), (lb, vb) = dev.read(), ref[0].read()
        np.testing.assert_array_equal(la, lb)
        np.testing.assert_array_equal(va, vb)
        assert_grid_equal(dev, ref[1])


def assert_submap_equal(sub, ref):
    assert_same(sub.high_resolution_hybrid_grid, ref.hi, False)
    assert_same(sub.low_resolution_hybrid_grid, ref.lo, False)
    if ref.ig is not None:
        assert_same(sub.high_resolution_intensity_hybrid_grid, ref.ig)


def _world():
    from benchmarks import synthetic
    return synthetic, synthetic.make_building(4, size_m=40.0)


def _tilt(rng):
    a = rng.normal(scale=0.05, size=3)
    a[2] = rng.uniform(-math.pi, math.pi)
    h = np.linalg.norm(a) / 2
    q = np.concatenate([[math.cos(h)], a / max(np.linalg.norm(a), 1e-12) * math.sin(h)])
    return q / np.linalg.norm(q)


# ---- 1. 50 config-5-like scans through ActiveSubmaps3D, every handle after every scan ----
def test_active_submaps_every_scan(sm, host):
    synthetic, (occ, cell, origin) = _world()
    rng = np.random.RandomState(21)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng) for _ in range(3)]
    clouds = [synthetic.cast_lidar_3d(occ, cell, origin, p, rings=64, azimuths=1024,
                                      max_range=20.0, seed=i) for i, p in enumerate(poses)]
    options = sm.SubmapsOptions3D(high_resolution=0.10, high_resolution_max_range=20.0,
                                  low_resolution=0.45, num_range_data=10,
                                  range_data_inserter_options=sm.RangeDataInserterOptions3D(**LUA))
    active = sm.ActiveSubmaps3D(options)
    ins = (sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**LUA)), O.RangeDataInserter3D(**LUA))
    refs, ref_count, ref_hist = [], [], []
    added, finished_seen = 0, 0
    held = None
    for k in range(50):
        base = poses[k % 3]
        pose = base + np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), 0, rng.uniform(-1, 1)])
        c, s = math.cos(pose[3]), math.sin(pose[3])
        # the local frame: the sensor scan placed at the pose, and 5 % of it pushed past 20 m
        pts = (clouds[k % 3].astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T
               + pose[:3]).astype(F)
        far = rng.rand(len(pts)) < 0.05
        pts[far] = (pose[:3] + (pts[far] - pose[:3]) * 1.6).astype(F)
        inten = synthetic.surface_intensity((occ, cell, origin), pts, seed=k)
        inten[::7] = F(40.0)   # on the threshold: kept
        q = _tilt(rng)
        hist = rng.uniform(0, 30, 120).astype(F)
        # the reference's lifecycle, restated
        if not refs or ref_count[-1] == options.num_range_data:
            if len(refs) >= 2:
                refs.pop(0), ref_count.pop(0), ref_hist.pop(0)
            refs.append(RefSubmap(sm, [*F(pose[:3]).astype(np.float64).tolist(), *q]))
            ref_count.append(0)
            ref_hist.append(np.zeros(120, F))
            added += 1
        subs = active.InsertData(pose[:3].astype(F), pts, inten, q, hist)
        assert active.range_data_inserter.last_stats["host_syncs"] <= 2
        for r, i in zip(refs, range(len(refs))):
            r.insert(host, ins, pose[:3].astype(F), pts, inten, 20.0)
            ref_count[i] += 1
            ref_hist[i] = ref_hist[i] + sm.rotate_histogram(
                hist, sm.yaw_in_submap_from_gravity(r.pose, q))
        assert len(subs) == len(refs)
        for sub, r, n, h in zip(subs, refs, ref_count, ref_hist):
            np.testing.assert_array_equal(np.asarray(sub.local_pose), np.asarray(r.pose))
            assert sub.num_range_data == n
            assert sub.insertion_finished == (n == 2 * options.num_range_data)
            np.testing.assert_array_equal(sub.rotational_scan_matcher_histogram.view(np.uint32),
                                          h.view(np.uint32))
            assert_submap_equal(sub, r)
        if subs[0].insertion_finished and held is None:
            held = (subs[0], refs[0])   # the pose graph keeps it past its eviction
        finished_seen += subs[0].insertion_finished
    assert added == 5 and finished_seen >= 3
    # evicted: the intensity grid is forgotten, the grids stay readable while held
    sub, ref = held
    assert sub not in active.submaps() and sub.high_resolution_intensity_hybrid_grid is None
    assert_same(sub.high_resolution_hybrid_grid, ref.hi, False)
    assert_same(sub.low_resolution_hybrid_grid, ref.lo, False)


# ---- 2. edge cases of one call ----
def _call(sm, host, ins, entries, refs, origin, pts, inten, max_range=20.0):
    sm_ins, ora, single = ins
    sm_ins.insert_submaps([(r.pose, *e) for r, e in zip(refs, entries)], origin, pts, inten,
                          max_range)
    assert sm_ins.last_stats["host_syncs"] <= 2
    for r in refs:
        r.insert(host, (single, ora), origin, pts, inten, max_range)
    for e, r in zip(entries, refs):
        assert_same(e[0], r.hi, False)
        assert_same(e[1], r.lo, False)
        if r.ig is not None:
            assert_same(e[2], r.ig)


def _entries(sm, refs):
    return [(sm.DeviceHybridGrid.empty(r.hi[1].resolution),
             sm.DeviceHybridGrid.empty(r.lo[1].resolution),
             None if r.ig is None else sm.DeviceIntensityGrid.empty(r.ig[1].resolution))
            for r in refs]


def _scan(rng, n, centre, spread):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (centre + d * rng.uniform(0.2, spread, n)[:, None]).astype(F)


@pytest.mark.parametrize("num", [1, 3])
def test_edge_cases(sm, host, num):
    rng = np.random.RandomState(30 + num)
    opts = sm.RangeDataInserterOptions3D(**LUA)
    ins = (sm.RangeDataInserter3D(opts), O.RangeDataInserter3D(**LUA), sm.RangeDataInserter3D(opts))
    poses = [[0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0],
             [1.5, -0.5, 0.25, *_tilt(rng)],
             [-2.0, 3.0, -0.75, math.cos(0.4), 0.0, 0.0, math.sin(0.4)]][:num]
    refs = [RefSubmap(sm, p, 0.1, 0.45, intensity=(i != 1)) for i, p in enumerate(poses)]
    entries = _entries(sm, refs)   # the first call finds every handle empty
    o = F([0.3, -0.2, 0.1])
    cases = []
    pts = _scan(rng, 3000, o, 6.0)
    cases.append((pts, rng.uniform(0, 60, len(pts)).astype(F)))              # growth of all
    pts = _scan(rng, 500, o, 3.0)
    cases.append((pts, np.full(len(pts), 40.5, F)))                          # all too bright
    far = _scan(rng, 400, o, 3.0)
    far = (o + (far - o) / np.linalg.norm(far - o, axis=1, keepdims=True) *
           rng.uniform(4.5, 6.0, (len(far), 1))).astype(F)
    cases.append((far, np.full(len(far), 5.0, F)))                           # all beyond 4 m
    cases.append((np.zeros((0, 3), F), np.zeros(0, F)))                      # no returns
    pts = _scan(rng, 800, o + 20.0, 4.0)
    cases.append((pts, None))                                                # no intensities
    cases.append((_scan(rng, 1000, o - 15.0, 8.0), np.full(1000, 40.0, F)))  # on the threshold
    for pts, inten in cases:
        max_range = 4.0 if pts is far else 20.0
        _call(sm, host, ins, entries, refs, o, pts, inten, max_range)


def test_no_returns_leave_handles_unchanged(sm, host):
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**LUA))
    hi, lo, ig = (sm.DeviceHybridGrid.empty(0.1), sm.DeviceHybridGrid.empty(0.45),
                  sm.DeviceIntensityGrid.empty(0.1))
    pose = [5.0, 5.0, 1.0, 1.0, 0.0, 0.0, 0.0]
    ins.insert_submaps([(pose, hi, lo, ig)], [100.0, 0.0, 0.0], np.zeros((0, 3), F),
                       np.zeros(0, F), 20.0)
    # nothing inserted: the boxes stay the fresh handles' one voxel at the origin
    assert hi.read()[0].tolist() == [0, 0, 0] and not hi.read()[1].any()
    assert lo.read()[0].tolist() == [0, 0, 0] and ig.read()[0].tolist() == [0, 0, 0]
    # the origin is still checked
    with pytest.raises(Exception) as e:
        ins.insert_submaps([(pose, hi, lo, ig)], [1e6, 0.0, 0.0], np.zeros((0, 3), F), None, 20.0)
    assert e.value.status == 1


# ---- 3. refusals change no handle ----
def test_refusals_change_nothing(sm):
    from cartographer_b200._lib import CsmError
    rng = np.random.RandomState(5)
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**LUA))
    pose_a = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    pose_b = [3.0, 1.0, 0.0, math.cos(0.3), 0.0, 0.0, math.sin(0.3)]
    grids = [(sm.DeviceHybridGrid.empty(0.1), sm.DeviceHybridGrid.empty(0.45),
              sm.DeviceIntensityGrid.empty(0.1)) for _ in range(2)]
    entries = [(pose_a, *grids[0]), (pose_b, *grids[1])]
    pts = _scan(rng, 2000, 0, 5.0)
    ins.insert_submaps(entries, [0, 0, 0], pts, np.full(len(pts), 5, F), 20.0)

    def snapshot():
        return [x.copy() for g in grids for h in g for x in h.read()]

    before = snapshot()
    bad = []
    p = pts.copy()
    p[1000] = [1e9, 0, 0]                  # outside the cube in the low-resolution grid
    bad.append((entries, [0, 0, 0], p))
    p = pts.copy()
    p[7] = [np.nan, 0, 0]                  # non-finite
    bad.append((entries, [0, 0, 0], p))
    bad.append((entries, [0, 0, -1e9], pts))   # origin outside the cube
    bad.append(([(pose_a, *grids[0]), (pose_b, grids[1][0], grids[0][1], grids[1][2])],
                [0, 0, 0], pts))           # a handle twice
    bad.append(([(pose_a, grids[0][0], grids[0][0], None)], [0, 0, 0], pts))
    for ent, org, p in bad:
        with pytest.raises(CsmError) as e:
            ins.insert_submaps(ent, org, p, np.full(len(p), 5, F), 20.0)
        assert e.value.status == 1
        for a, b in zip(before, snapshot()):
            np.testing.assert_array_equal(a, b)
    # num_samples >= 2^15 cannot happen inside the cube (cells at most 16383 apart): the
    # farthest pair of cells along an axis is accepted
    g = (sm.DeviceHybridGrid.empty(0.1), sm.DeviceHybridGrid.empty(0.1))
    ins.insert_submaps([(pose_a, *g, None)], [-819.1, 0.0, 0.0], np.float32([[819.0, 0.0, 0.0]]),
                       None, 1e9)
    assert g[0].read()[1].any() and g[1].read()[1].any()


def test_refuses_another_device(sm):
    if sm.device_count() < 2:
        pytest.skip("one device")
    from cartographer_b200._lib import CsmError
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**LUA))
    a, b = sm.DeviceHybridGrid.empty(0.1), sm.DeviceHybridGrid.empty(0.45, device=1)
    with pytest.raises(CsmError):
        ins.insert_submaps([([0, 0, 0, 1, 0, 0, 0], a, b, None)], [0, 0, 0],
                           np.float32([[1, 0, 0]]), None, 20.0)
    assert not a.read()[1].any()


# ---- 4. ConstraintBuilder3D on a finished submap ----
def test_constraint_builder_on_finished_submap(sm, host):
    from cartographer_b200 import constraint_builder as cb
    synthetic, (occ, cell, origin) = _world()
    rng = np.random.RandomState(8)
    options = sm.SubmapsOptions3D(num_range_data=3, range_data_inserter_options=
                                  sm.RangeDataInserterOptions3D(**LUA))
    active = sm.ActiveSubmaps3D(options)
    ins = (sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**LUA)), O.RangeDataInserter3D(**LUA))
    base = synthetic.random_free_pose_3d(occ, cell, origin, rng)
    cloud = synthetic.cast_lidar_3d(occ, cell, origin, base, rings=32, azimuths=1024,
                                    max_range=20.0, seed=3)
    ref = None
    hist = np.ones(24, F)
    for k in range(6):
        pose = base + np.array([0.2 * k, -0.1 * k, 0, 0.02 * k])
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T +
               pose[:3]).astype(F)
        subs = active.InsertData(pose[:3].astype(F), pts, None, [1, 0, 0, 0], hist)
        if ref is None:
            ref = RefSubmap(sm, subs[0].local_pose, intensity=False)
        ref.insert(host, ins, pose[:3].astype(F), pts, None, 20.0)
    sub = subs[0]
    assert sub.insertion_finished
    levels = []
    for hi, lo in ((sub.high_resolution_hybrid_grid, sub.low_resolution_hybrid_grid),
                   (ref.hi[0], ref.lo[0])):
        m = sm.FastCorrelativeScanMatcher3D.from_device_grids(
            hi, lo, sub.rotational_scan_matcher_histogram,
            sm.FastCorrelativeScanMatcherOptions3D(branch_and_bound_depth=5,
                                                   full_resolution_depth=3))
        levels.append([(lv[0].tolist(), lv[1].tobytes())
                       for lv in (m.precomputation_grid(d) for d in range(5))])
        m.close()
    assert levels[0] == levels[1]
    opts = cb.ConstraintBuilderOptions3D(
        sampling_ratio=1.0, min_score=0.2, global_localization_min_score=0.2,
        branch_and_bound_depth=5, full_resolution_depth=3, min_rotational_score=0.0,
        min_low_resolution_score=0.1, linear_xy_search_window=0.5, linear_z_search_window=0.3,
        angular_search_window=0.05)
    records = []
    for hi, lo in ((sub.high_resolution_hybrid_grid, sub.low_resolution_hybrid_grid),
                   (ref.hi[0], ref.lo[0])):
        builder = cb.ConstraintBuilder3D(opts)
        view = (sub.constraint_builder_submap() if hi is sub.high_resolution_hybrid_grid
                else cb.Submap3D(hi, lo, sub.rotational_scan_matcher_histogram))
        node = sm.TrajectoryNodeData3D(cloud[::3], synthetic.voxel_downsample(cloud, 0.45), hist)
        npose = synthetic.yaw_pose7(base[0] + 0.1, base[1] - 0.05, base[2], base[3])
        builder.MaybeAddConstraint((0, 0), view, (1, 0), node, npose, list(sub.local_pose))
        builder.MaybeAddGlobalConstraint((0, 0), view, (1, 1), node, list(npose[3:]),
                                         list(sub.local_pose[3:]))
        builder.NotifyEndOfNode()
        builder.WhenDone(lambda r: None)
        records.append(builder.last_records.copy())
        for sid in list(builder.executor.matchers):
            builder.executor.delete_matcher(sid)
    assert records[0].tobytes() == records[1].tobytes()
    assert records[0]["found"].sum() >= 1
