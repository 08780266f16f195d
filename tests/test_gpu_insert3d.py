"""RangeDataInserter3D on the device (csrc/insert3d.cu) against the CPU restatement in
tests/insert3d_oracle.py: every voxel of the dense boxes — occupancy values, intensity sums,
counts and means — bit for bit, after every insert."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import insert3d_oracle as O

pytestmark = pytest.mark.gpu

REF = dict(hit_probability=0.7, miss_probability=0.4, num_free_space_voxels=1000,
           intensity_threshold=100.0)   # range_data_inserter_3d_test.cc:33-38
REF_RETURNS = np.array([[-3, -1, 4], [-2, 0, 4], [-1, 1, 4], [0, 2, 4]], np.float32)


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _pair(sm, opts):
    return (sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**opts)),
            O.RangeDataInserter3D(**opts))


def _grid(sm, resolution, indices=None, values=None):
    if indices is None:
        return sm.DeviceHybridGrid.empty(resolution), O.HybridGrid(resolution)
    from benchmarks.synthetic import HybridGridSpec
    return (sm.DeviceHybridGrid(HybridGridSpec(resolution, indices, values)),
            O.HybridGrid(resolution, indices, values))


def _igrid(sm, resolution, indices=None, sums=None, counts=None):
    if indices is None:
        return sm.DeviceIntensityGrid.empty(resolution), O.IntensityHybridGrid(resolution)
    return (sm.DeviceIntensityGrid(sm.IntensityGridSpec(resolution, indices, sums, counts)),
            O.IntensityHybridGrid(resolution, indices, sums, counts))


def _contains(lo, shape, keys):
    idx = O.unpack(keys) - lo
    return bool(np.all((idx >= 0) & (idx < np.asarray(shape[::-1]))))


def assert_grid_equal(dev, ora):
    lo, vol = dev.read()
    assert _contains(lo, vol.shape, ora.keys[ora.values != 0]), "a voxel outside the box"
    np.testing.assert_array_equal(vol, ora.dense(lo, vol.shape[::-1]))
    return lo, vol.shape[::-1]


def assert_igrid_equal(dev, ora):
    lo, mean, sums, counts = dev.read()
    assert _contains(lo, mean.shape, ora.keys[ora.counts != 0]), "a voxel outside the box"
    dims = mean.shape[::-1]
    np.testing.assert_array_equal(counts, ora.dense(lo, dims, 1))
    np.testing.assert_array_equal(sums.view(np.uint32), ora.dense(lo, dims, 0).view(np.uint32))
    np.testing.assert_array_equal(mean.view(np.uint32), ora.dense_mean(lo, dims).view(np.uint32))
    return lo, dims


def _insert(pair, origin, returns, intensities, g, ig=None):
    dev, ora = pair
    dev.Insert(origin, returns, intensities, g[0], None if ig is None else ig[0])
    ora.insert(origin, returns, intensities, g[1], None if ig is None else ig[1])


# ---- 1. the reference's cases (range_data_inserter_3d_test.cc) on the device ----
def test_reference_cases(sm):
    ins = _pair(sm, REF)
    g, ig = _grid(sm, 1.0), _igrid(sm, 1.0)
    _insert(ins, [0, 0, -4], REF_RETURNS, [7, 8, 9, 10], g, ig)
    assert_grid_equal(*g)
    assert_igrid_equal(*ig)
    lo, vol = g[0].read()
    prob = lambda c: O.value_to_probability(vol[c[2] - lo[2], c[1] - lo[1], c[0] - lo[0]])  # noqa
    for c in ([0, 0, -4], [0, 0, -3], [0, 0, -2], [-2, 0, 3]):
        assert abs(prob(c) - 0.4) < 1e-4
    _, mean, _, _ = ig[0].read()
    ilo = ig[0].read()[0]
    for x in range(-4, 5):
        for y in range(-4, 5):
            on = -3 <= x <= 0 and y == x + 2
            z = 4 - lo[2]
            inside = 0 <= x - lo[0] < vol.shape[2] and 0 <= y - lo[1] < vol.shape[1]
            v = vol[z, y - lo[1], x - lo[0]] if inside else 0
            if on:
                assert abs(prob([x, y, 4]) - 0.7) < 1e-4
                assert mean[4 - ilo[2], y - ilo[1], x - ilo[0]] == 10 + x
            else:
                assert v == 0
    for _ in range(1000):   # ProbabilityProgression
        _insert(ins, [0, 0, -4], REF_RETURNS, None, g)
    assert_grid_equal(*g)
    lo, vol = g[0].read()
    assert abs(prob([-2, 0, 4]) - 0.9) < 1e-3
    assert abs(prob([-2, 0, 3]) - 0.1) < 1e-3 and abs(prob([0, 0, -3]) - 0.1) < 1e-3
    assert ins[0].last_stats["host_syncs"] == 1


# ---- 2. seeded scans, every insert checked ----
def _scan(rng, n, centre, spread):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = rng.uniform(0.2, spread, n)[:, None]
    return (centre + d * r).astype(np.float32)


@pytest.mark.parametrize("start", ["empty", "voxel_list"])
def test_seeded_scans_every_insert(sm, start):
    rng = np.random.RandomState(7 if start == "empty" else 8)
    ins = _pair(sm, dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=3,
                         intensity_threshold=40.0))
    if start == "empty":
        g, ig = _grid(sm, 0.1), _igrid(sm, 0.25)
    else:
        idx = np.unique(rng.randint(-30, 30, size=(400, 3)), axis=0).astype(np.int32)
        g = _grid(sm, 0.1, idx, rng.randint(1, 32768, len(idx)).astype(np.uint16))
        iidx = np.unique(rng.randint(-10, 10, size=(200, 3)), axis=0).astype(np.int32)
        cnt = rng.randint(0, 4, len(iidx)).astype(np.int32)
        ig = _igrid(sm, 0.25, iidx, (rng.uniform(0, 40, len(iidx)) * cnt).astype(np.float32),
                    cnt)
        assert_grid_equal(*g)
        assert_igrid_equal(*ig)
    boxes = set()
    for k in range(50):
        origin = rng.uniform(-1.5, 1.5, 3).astype(np.float32) * (1 + k / 10)
        pts = _scan(rng, rng.randint(1, 3000), origin, 1.0 + k / 8)
        inten = rng.uniform(0, 60, len(pts)).astype(np.float32)
        inten[::7] = 40.0   # on the threshold: kept
        _insert(ins, origin, pts, inten, g, ig)
        boxes.add(tuple(np.concatenate(assert_grid_equal(*g))))
        assert_igrid_equal(*ig)
        assert ins[0].last_stats["host_syncs"] == 1
    assert len(boxes) > 3   # the box grew along the way


# ---- 3. edge cases ----
def test_edge_cases(sm):
    rng = np.random.RandomState(3)
    for nfsv in (0, 1, 2, 5, 200):   # 200 > every num_samples below
        ins = _pair(sm, dict(REF, num_free_space_voxels=nfsv))
        g, ig = _grid(sm, 0.5), _igrid(sm, 0.3)   # intensity resolution differs
        o = np.float32([0.1, -0.2, 0.05])
        cases = [
            np.float32([[2, 2, 2], [2, 2, 2], [2.1, 2, 2]]),            # duplicates in one cell
            np.float32([[3, 0, 0], [6, 0, 0]]),                          # hit crossed by a ray
            np.float32([[6, 0, 0], [3, 0, 0]]),                          # ... other order
            np.float32([[0.1, -0.2, 0.05], [0.2, 0, 0]]),                # returns in the origin cell
            np.float32([[-4, -3, -5], [-4, 3, -5], [4, -3, 5], [-1, 7, -2]]),  # negative / mixed
            np.float32([[0.25, -0.25, 0.75], [-0.75, 1.25, -1.25]]),    # half-voxel boundaries
            np.zeros((0, 3), np.float32),                                # no returns
        ]
        for pts in cases:
            inten = np.float32([100.0, 100.5, 7.0, 50.0][:len(pts)] +
                               [3.0] * max(0, len(pts) - 4))
            _insert(ins, o, pts, inten, g, ig)
            assert_grid_equal(*g)
            assert_igrid_equal(*ig)
            _insert(ins, o, pts, None, g, ig)   # NULL intensities: the intensity grid is untouched
            assert_grid_equal(*g)
            assert_igrid_equal(*ig)
    # growth through each of the six faces, from a non-empty box
    ins = _pair(sm, dict(REF, num_free_space_voxels=2))
    g = _grid(sm, 0.1, np.zeros((1, 3), np.int32), np.uint16([20000]))
    ig = _igrid(sm, 0.1, np.zeros((1, 3), np.int32), np.float32([5]), np.int32([1]))
    last = None
    for axis in range(3):
        for sign in (-1, 1):
            p = np.zeros((1, 3), np.float32)
            p[0, axis] = sign * rng.uniform(2.0, 4.0)
            _insert(ins, [0, 0, 0], p, [1.0], g, ig)
            lo, dims = assert_grid_equal(*g)
            assert_igrid_equal(*ig)
            box = (tuple(lo), tuple(dims))
            assert box != last
            last = box


# ---- 4. errors leave every handle unchanged ----
def test_invalid_calls_change_nothing(sm):
    from cartographer_b200._lib import lib, ptr, CsmError
    lib_ = lib()
    out = C.c_void_p()
    for bad in (dict(REF, hit_probability=0.5), dict(REF, miss_probability=0.5),
                dict(REF, num_free_space_voxels=-1), dict(REF, hit_probability=1.0)):
        o = sm.RangeDataInserterOptions3D(**bad)._c()
        assert lib_.csm_range_inserter3d_create(C.byref(o), 0, C.byref(out)) == 1
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**REF))
    g = sm.DeviceHybridGrid.empty(0.1)
    ig = sm.DeviceIntensityGrid.empty(0.05)
    ins.Insert([0, 0, 0], _scan(np.random.RandomState(1), 100, 0, 2.0),
               np.full(100, 5, np.float32), g, ig)
    before = g.read(), ig.read()
    far = np.float32([[819.0, 0, 0]])   # cell 8190 at 0.1 m, 16380 at 0.05 m
    for origin, pts, inten in (([0, 0, 0], np.float32([[1e9, 0, 0]]), None),
                               ([0, 0, -1e9], np.float32([[1, 0, 0]]), None),
                               ([0, 0, 0], np.float32([[np.nan, 0, 0]]), None),
                               ([0, 0, 0], far, np.float32([1.0]))):      # intensity cell only
        with pytest.raises(CsmError) as e:
            ins.Insert(origin, pts, inten, g, ig)
        assert e.value.status == 1
    after = g.read(), ig.read()
    for a, b in zip(before[0] + before[1], after[0] + after[1]):
        np.testing.assert_array_equal(a, b)
    # null grid
    org = np.zeros(3, np.float32)
    assert lib_.csm_range_inserter3d_insert(ins._h, ptr(org, C.c_float), None, None, 0, None,
                                            None, None) == 1


# ---- 5. the matchers read inserted handles as they read created ones ----
def test_matchers_on_inserted_handles(sm):
    from benchmarks import synthetic
    rng = np.random.RandomState(5)
    hi_ins, lo_ins = _pair(sm, {**REF, "num_free_space_voxels": 2}), \
        _pair(sm, {**REF, "num_free_space_voxels": 2})
    hi, lo, ig = _grid(sm, 0.1), _grid(sm, 0.45), _igrid(sm, 0.1)
    occ, cell, origin = synthetic.make_building(2, size_m=16.0)
    for k in range(6):
        pose = synthetic.random_free_pose_3d(occ, cell, origin, rng, margin_m=3.0)
        cloud = synthetic.cast_lidar_3d(occ, cell, origin, pose, rings=16, azimuths=512,
                                        max_range=10.0, seed=k)
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T +
               pose[:3]).astype(np.float32)
        inten = synthetic.surface_intensity((occ, cell, origin), pts, seed=k)
        _insert(hi_ins, pose[:3], pts, inten, hi, ig)
        _insert(lo_ins, pose[:3], pts, None, lo)
    assert_grid_equal(*hi)
    assert_grid_equal(*lo)
    assert_igrid_equal(*ig)
    spec = synthetic.HybridGridSpec
    hi_c = sm.DeviceHybridGrid(spec(0.1, hi[1].indices(), hi[1].values))
    lo_c = sm.DeviceHybridGrid(spec(0.45, lo[1].indices(), lo[1].values))
    ig_c = sm.DeviceIntensityGrid(sm.IntensityGridSpec(0.1, ig[1].indices(), ig[1].sums,
                                                       ig[1].counts))
    node = cloud[::4]
    start = synthetic.yaw_pose7(pose[0] + 0.05, pose[1] - 0.04, pose[2], pose[3] + 0.02)
    rt = sm.RealTimeCorrelativeScanMatcher3D(
        sm.RealTimeCorrelativeScanMatcherOptions(0.15, 0.02, 0.1, 0.1))
    a = rt.Match(start, node, hi[0])
    b = rt.Match(start, node, hi_c)
    assert a[0] == b[0] and np.array_equal(a[1], b[1])
    opts = sm.CeresScanMatcherOptions3D(
        occupied_space_weight_0=1.0, occupied_space_weight_1=6.0, translation_weight=5.0,
        rotation_weight=4e2, use_nonmonotonic_steps=False,
        intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(0.5, 0.3, 40.0))
    cm = sm.CeresScanMatcher3D(opts)
    inten = synthetic.surface_intensity((occ, cell, origin), pts, seed=99)[::4]
    pa, sa = cm.Match(start[:3], start, [(node, hi[0], ig[0], inten), (node[::3], lo[0])])
    pb, sb = cm.Match(start[:3], start, [(node, hi_c, ig_c, inten), (node[::3], lo_c)])
    assert np.array_equal(pa, pb)
    for k in ("initial_cost", "final_cost", "iterations", "termination"):
        assert sa[k] == sb[k] or (isinstance(sa[k], float) and np.array_equal(sa[k], sb[k]))


# ---- 6. config-5 size: 65,536-point scans ----
def test_config5_size_scans(sm):
    from benchmarks import synthetic
    rng = np.random.RandomState(11)
    occ, cell, origin = synthetic.make_building(4, size_m=40.0)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng) for _ in range(3)]
    clouds = [synthetic.cast_lidar_3d(occ, cell, origin, p, rings=64, azimuths=1024,
                                      max_range=20.0, seed=i) for i, p in enumerate(poses)]
    hi_ins, lo_ins = _pair(sm, dict(REF, num_free_space_voxels=2)), \
        _pair(sm, dict(REF, num_free_space_voxels=2))
    hi, lo, ig = _grid(sm, 0.1), _grid(sm, 0.45), _igrid(sm, 0.1)
    tight = {0.1: None, 0.45: None}
    reallocs = {0.1: 0, 0.45: 0}
    boxes = {0.1: None, 0.45: None}
    for k in range(20):
        base = poses[k % 3]
        pose = base + np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), 0, rng.uniform(-1, 1)])
        cloud = clouds[k % 3]
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T +
               pose[:3]).astype(np.float32)
        inten = synthetic.surface_intensity((occ, cell, origin), pts, seed=k)
        near = np.linalg.norm(pts - pose[:3], axis=1) <= 20.0
        _insert(hi_ins, pose[:3], pts[near], inten[near], hi, ig)
        _insert(lo_ins, pose[:3], pts, None, lo)
        for res, (dev, ora) in ((0.1, hi), (0.45, lo)):
            lo_, dims = assert_grid_equal(dev, ora)
            cells = np.concatenate([O.cell_index(res, pose[:3].astype(np.float32)),
                                    O.cell_index(res, pts[near] if res == 0.1 else pts)])
            t = np.stack([cells.min(0), cells.max(0)])
            if tight[res] is not None:
                t = np.stack([np.minimum(t[0], tight[res][0]), np.maximum(t[1], tight[res][1])])
            tight[res] = t
            vol = np.prod(np.asarray(dims, np.float64))
            assert vol <= 2 * np.prod((t[1] - t[0] + 1).astype(np.float64))
            box = (tuple(lo_), tuple(dims))
            reallocs[res] += box != boxes[res]
            boxes[res] = box
        assert_igrid_equal(*ig)
        assert hi_ins[0].last_stats["host_syncs"] == 1
    # slack of extent / 8 per side: after the first few scans the box stops moving
    assert reallocs[0.1] <= 10 and reallocs[0.45] <= 10, reallocs
