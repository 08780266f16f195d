"""FastCorrelativeScanMatcher3D built from device-resident grids
(csm_matcher3d_create_from_grid3d) against the same matcher built from the grids' non-zero
voxels (csm_matcher3d_create) and against the CPU oracle: every precomputation level box and
byte, the derived grid size, every field of every result, independence from later inserts,
batches, refusals, and ConstraintBuilder3D on device submaps."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import insert3d_oracle as O
from tests import worlds3d

pytestmark = pytest.mark.gpu

INSERT = dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
              intensity_threshold=40.0)   # trajectory_builder_3d.lua


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _opts(sm, od):
    return sm.FastCorrelativeScanMatcherOptions3D(
        od["branch_and_bound_depth"], od["full_resolution_depth"], od["min_rotational_score"],
        od["min_low_resolution_score"], od["linear_xy_search_window"],
        od["linear_z_search_window"], od["angular_search_window"])


def _spec(resolution, ora):
    """The non-zero voxels of an oracle grid, in the flat form."""
    keep = ora.values != 0
    return synthetic.HybridGridSpec(resolution, ora.indices()[keep], ora.values[keep])


def _device_spec(grid):
    """The non-zero voxels of a DeviceHybridGrid, read back."""
    lo, vol = grid.read()
    z, y, x = np.nonzero(vol)
    idx = (np.stack([x, y, z], 1) + lo).astype(np.int32)
    return synthetic.HybridGridSpec(grid.resolution, idx, vol[z, y, x])


def _scan(occ, cell, origin, pose, rings, azimuths, max_range, seed):
    cloud = synthetic.cast_lidar_3d(occ, cell, origin, pose, rings=rings, azimuths=azimuths,
                                    max_range=max_range, seed=seed)
    c, s = math.cos(pose[3]), math.sin(pose[3])
    world = (cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T +
             pose[:3]).astype(np.float32)
    return cloud, world


class _Submap:
    """A high (0.10 m) and a low (0.45 m) resolution grid on the device, filled by
    RangeDataInserter3D, with the CPU restatement's grids beside them (asserted equal)."""

    def __init__(self, sm, seed, scans, from_voxels=False, rings=8, azimuths=256):
        self.sm = sm
        self.world = synthetic.make_building(seed, size_m=16.0)
        occ, cell, origin = self.world
        self.rng = np.random.RandomState(seed)
        if from_voxels:   # handles created from voxel lists (csm_grid3d_create), then grown
            vox = worlds3d.random_voxels(self.rng, 200, 12, 0.1)
            lvox = worlds3d.random_voxels(self.rng, 60, 4, 0.45)
            self.hi = (sm.DeviceHybridGrid(vox), O.HybridGrid(0.1, vox.indices, vox.values))
            self.lo = (sm.DeviceHybridGrid(lvox), O.HybridGrid(0.45, lvox.indices, lvox.values))
        else:
            self.hi = (sm.DeviceHybridGrid.empty(0.1), O.HybridGrid(0.1))
            self.lo = (sm.DeviceHybridGrid.empty(0.45), O.HybridGrid(0.45))
        self.ins = (sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**INSERT)),
                    O.RangeDataInserter3D(**INSERT))
        self.poses = [synthetic.random_free_pose_3d(occ, cell, origin, self.rng, margin_m=3.0)
                      for _ in range(3)]
        self.last = None
        self.insert(scans, rings, azimuths)

    def insert(self, scans, rings=8, azimuths=256):
        occ, cell, origin = self.world
        for k in range(scans):
            pose = self.poses[k % len(self.poses)] + np.array(
                [self.rng.uniform(-0.5, 0.5), self.rng.uniform(-0.5, 0.5), 0.0,
                 self.rng.uniform(-0.3, 0.3)])
            cloud, pts = _scan(occ, cell, origin, pose, rings, azimuths, 10.0,
                               int(self.rng.randint(1 << 30)))
            org = pose[:3].astype(np.float32)
            for g in (self.hi, self.lo):
                self.ins[0].Insert(org, pts, None, g[0])
                self.ins[1].insert(org, pts, None, g[1])
            self.last = (pose, cloud)
        for g in (self.hi, self.lo):
            lo, vol = g[0].read()
            np.testing.assert_array_equal(vol, g[1].dense(lo, vol.shape[::-1]))

    def specs(self):
        return _spec(0.1, self.hi[1]), _spec(0.45, self.lo[1])

    def close(self):
        for h in (self.hi[0], self.lo[0], self.ins[0]):
            h.close()


def _both(sm, hi_dev, lo_dev, hi_spec, lo_spec, od, hist, grid_size=0):
    """(from the handles, from the voxel lists)."""
    o = _opts(sm, od)
    a = sm.FastCorrelativeScanMatcher3D.from_device_grids(hi_dev, lo_dev, hist, o,
                                                          grid_size_in_voxels=grid_size)
    b = sm.FastCorrelativeScanMatcher3D(hi_spec, lo_spec, hist, o, grid_size_in_voxels=grid_size)
    return a, b


def _assert_levels_equal(a, b, depth):
    for d in range(depth):
        la, va = a.precomputation_grid(d)
        lb, vb = b.precomputation_grid(d)
        np.testing.assert_array_equal(la, lb)
        assert va.shape == vb.shape
        np.testing.assert_array_equal(va, vb)


def _levels(m, depth):
    return [m.precomputation_grid(d) for d in range(depth)]


def _node(sm, cloud, hist=None):
    low = synthetic.voxel_downsample(cloud, 0.45)
    hist = np.zeros(10, np.float32) if hist is None else hist
    return sm.TrajectoryNodeData3D(cloud, low, hist)


def _odict(node):
    return dict(gravity_alignment=node.gravity_alignment,
                high_resolution_point_cloud=node.high_resolution_point_cloud,
                low_resolution_point_cloud=node.low_resolution_point_cloud,
                rotational_scan_matcher_histogram=node.rotational_scan_matcher_histogram)


def _assert_oracle(want, got):
    assert (got is not None) == want["found"]
    if got is not None:
        assert np.float32(got["score"]).view(np.uint32) == np.float32(want["score"]).view(np.uint32)
        np.testing.assert_array_equal(got["pose_estimate"], want["pose"])


def _assert_same_result(ra, rb):
    assert (ra is None) == (rb is None)
    if ra is None:
        return
    assert ra.keys() == rb.keys()
    for k in ra:
        if isinstance(ra[k], np.ndarray):
            np.testing.assert_array_equal(ra[k], rb[k])
        elif isinstance(ra[k], np.floating):
            assert np.float32(ra[k]).view(np.uint32) == np.float32(rb[k]).view(np.uint32), k
        else:
            assert ra[k] == rb[k], k


# ---- 1. every level, from empty handles and from handles created from voxels ----
@pytest.fixture(scope="module", params=[False, True], ids=["empty", "from_voxels"])
def inserted(sm, request):
    s = _Submap(sm, 3, 4, from_voxels=request.param)
    yield s
    s.close()


@pytest.mark.parametrize("depth,frd", [(1, 1), (1, 2), (1, 3), (3, 1), (3, 3), (3, 4), (8, 1),
                                       (8, 3), (8, 8), (8, 9)])
def test_every_level(sm, inserted, depth, frd):
    od = worlds3d.fast_options(depth=depth, frd=frd)
    hs, ls = inserted.specs()
    a, b = _both(sm, inserted.hi[0], inserted.lo[0], hs, ls, od, np.zeros(10, np.float32))
    _assert_levels_equal(a, b, depth)
    a.close()
    b.close()


# ---- 2. geometry edges ----
def _handle(sm, resolution, idx, val):
    return sm.DeviceHybridGrid(synthetic.HybridGridSpec(resolution, np.asarray(idx, np.int32),
                                                        np.asarray(val, np.uint16)))


def _nonzero(idx, val, resolution):
    idx, val = np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(val, np.uint16)
    return synthetic.HybridGridSpec(resolution, idx[val != 0], val[val != 0])


def _lattice(m, node, full=True):
    q = [1.0, 0.0, 0.0, 0.0]
    return m.score_top(full, [0, 0, 0] + q, [0, 0, 0] + q, node, 0.0)


CORNERS = [[x, y, z] for x in (-5, 6) for y in (-3, 4) for z in (-2, 2)]
GEOMETRY = {
    # zero margins around the non-zero cells: explicit zero voxels widen the handle's box
    "zero_margins": ([[-9, -9, -9], [0, 0, 0], [1, 2, 0], [9, 9, 9]], [0, 30000, 2000, 0]),
    "single_voxel": ([[3, -4, 5]], [17000]),
    "faces_and_corners": (CORNERS + [[0, -3, 0], [6, 0, 0], [0, 0, 2]],
                          list(range(1000, 1000 + 500 * 11, 500))),
    "explicit_zeros": ([[-2, 0, 1], [4, 5, 6]], [0, 0]),
    "cube_edges": ([[-8192, 0, 0], [8191, 1, -1], [0, 0, 0]], [32767, 1, 9000]),
    "marker_bit_only": ([[1, 1, 1], [2, 2, 2]], [0x8000, 0x8000 | 20000]),
}


@pytest.mark.parametrize("case", sorted(GEOMETRY))
@pytest.mark.parametrize("depth,frd", [(3, 1), (8, 3)])
def test_geometry_edges(sm, case, depth, frd):
    idx, val = GEOMETRY[case]
    od = worlds3d.fast_options(depth=depth, frd=frd)
    hi = _handle(sm, 0.1, idx, val)
    lo = _handle(sm, 0.45, idx, val)
    a, b = _both(sm, hi, lo, _nonzero(idx, val, 0.1), _nonzero(idx, val, 0.45), od,
                 np.zeros(10, np.float32))
    _assert_levels_equal(a, b, depth)
    for m in (a, b, hi, lo):
        m.close()


def test_empty_handles(sm):
    od = worlds3d.fast_options(depth=3, frd=2)
    hi, lo = sm.DeviceHybridGrid.empty(0.1), sm.DeviceHybridGrid.empty(0.45)
    empty = synthetic.HybridGridSpec(0.1, np.zeros((0, 3), np.int32), np.zeros(0, np.uint16))
    a, b = _both(sm, hi, lo, empty, empty, od, np.zeros(10, np.float32))
    _assert_levels_equal(a, b, 3)
    node = _node(sm, worlds3d.random_cloud(np.random.RandomState(1), 30, 0.4))
    assert _lattice(a, node)["nxc"] == _lattice(b, node)["nxc"]
    # every candidate ties on an empty grid; a local window keeps the ties within the engine's
    # capacity (MatchFullSubmap's would not be)
    ident = [0, 0, 0, 1, 0, 0, 0]
    _assert_same_result(a.Match(ident, ident, node, 0.0), b.Match(ident, ident, node, 0.0))
    for m in (a, b, hi, lo):
        m.close()


# non-zero boxes on both sides of +-64 * 2^k: the derived grid size (64 << bits) follows the
# non-zero cells, not the zero cells the handle's box also holds
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("side", ["low", "high"])
def test_derived_grid_size(sm, oracle, k, side):
    edge = 64 << (k - 1)   # grid_size 128 << (k - 1) holds [-edge, edge)
    inside = -edge if side == "low" else edge - 1
    outside = inside - 1 if side == "low" else inside + 1
    zero = outside - 3 if side == "low" else outside + 3   # beyond `outside`, value 0
    od = worlds3d.fast_options(depth=5, frd=3)
    node = _node(sm, worlds3d.random_cloud(np.random.RandomState(k), 40, 0.4))
    lattices = []
    for far in (inside, outside):
        idx = [[0, 0, 0], [far, 1, 0], [1, 2, 1], [zero, 0, 0]]
        val = [20000, 25000, 15000, 0]
        hi, lo = _handle(sm, 0.1, idx, val), _handle(sm, 0.45, idx, val)
        hs, ls = _nonzero(idx, val, 0.1), _nonzero(idx, val, 0.45)
        a, b = _both(sm, hi, lo, hs, ls, od, np.zeros(10, np.float32))
        _assert_levels_equal(a, b, 5)
        ta, tb = _lattice(a, node), _lattice(b, node)
        assert (ta["nxc"], ta["nzc"]) == (tb["nxc"], tb["nzc"])
        np.testing.assert_array_equal(ta["sums"], tb["sums"])
        q = [1.0, 0.0, 0.0, 0.0]
        ra, rb = a.MatchFullSubmap(q, q, node, 0.0), b.MatchFullSubmap(q, q, node, 0.0)
        _assert_same_result(ra, rb)
        om = oracle.FastCorrelativeScanMatcher3D(
            oracle.HybridGrid(0.1, hs.indices, hs.values),
            oracle.HybridGrid(0.45, ls.indices, ls.values), np.zeros(10, np.float32), od)
        _assert_oracle(om.match_full_submap(q, q, _odict(node), 0.0), ra)
        lattices.append(ta["nxc"])
        for m in (a, b, hi, lo):
            m.close()
    assert lattices[1] > lattices[0], "the grid size did not follow the non-zero box"


def test_explicit_grid_size(sm):
    idx, val = [[0, 0, 0], [5, 1, 0], [1, 2, 1]], [20000, 25000, 15000]
    od = worlds3d.fast_options(depth=5, frd=3)
    node = _node(sm, worlds3d.random_cloud(np.random.RandomState(3), 40, 0.4))
    hi, lo = _handle(sm, 0.1, idx, val), _handle(sm, 0.45, idx, val)
    lat = {}
    for gs in (0, 512):
        a, b = _both(sm, hi, lo, _nonzero(idx, val, 0.1), _nonzero(idx, val, 0.45), od,
                     np.zeros(10, np.float32), grid_size=gs)
        ta, tb = _lattice(a, node), _lattice(b, node)
        assert ta["nxc"] == tb["nxc"]
        lat[gs] = ta["nxc"]
        a.close()
        b.close()
    assert lat[512] > lat[0]


# ---- 3. results: Match and MatchFullSubmap, against the list path and the oracle ----
def _oracle_matcher(oracle, hs, ls, hist, od):
    return oracle.FastCorrelativeScanMatcher3D(oracle.HybridGrid(0.1, hs.indices, hs.values),
                                               oracle.HybridGrid(0.45, ls.indices, ls.values),
                                               hist, od)


def test_results(sm, oracle):
    s = _Submap(sm, 7, 6)
    hs, ls = s.specs()
    hist = np.ones(24, np.float32)
    od = worlds3d.fast_options(depth=5, frd=3, xy=0.6, z=0.3, angular=0.05)
    a, b = _both(sm, s.hi[0], s.lo[0], hs, ls, od, hist)
    om = _oracle_matcher(oracle, hs, ls, hist, od)
    rng = np.random.RandomState(2)
    pose, cloud = s.last
    found = 0
    for k in range(4):
        node = _node(sm, cloud[k::5], hist)
        npose = synthetic.yaw_pose7(pose[0] + rng.uniform(-0.2, 0.2),
                                    pose[1] + rng.uniform(-0.2, 0.2), pose[2],
                                    pose[3] + rng.uniform(-0.03, 0.03))
        ident = [0, 0, 0, 1, 0, 0, 0]
        ra, rb = a.Match(npose, ident, node, 0.3), b.Match(npose, ident, node, 0.3)
        _assert_same_result(ra, rb)
        _assert_oracle(om.match(npose, ident, _odict(node), 0.3), ra)
        found += ra is not None
        # MatchFullSubmap's angular step shrinks with the node's range: the points within
        # 4 m keep the oracle's search small
        near = cloud[k::3][np.linalg.norm(cloud[k::3], axis=1) < 4.0][:80]
        fnode = _node(sm, near if len(near) >= 10 else cloud[k::5][:80], hist)
        q = list(npose[3:])
        fa = a.MatchFullSubmap(q, [1, 0, 0, 0], fnode, 0.3)
        _assert_same_result(fa, b.MatchFullSubmap(q, [1, 0, 0, 0], fnode, 0.3))
        _assert_oracle(om.match_full_submap(q, [1, 0, 0, 0], _odict(fnode), 0.3), fa)
    assert found >= 1
    # the low-resolution gate rejects the best leaf: min_low_resolution_score just above it
    node = _node(sm, cloud[::5], hist)
    npose = synthetic.yaw_pose7(pose[0] + 0.1, pose[1] - 0.1, pose[2], pose[3])
    best = a.Match(npose, [0, 0, 0, 1, 0, 0, 0], node, 0.3)
    assert best is not None
    gate = dict(od, min_low_resolution_score=float(np.nextafter(best["low_resolution_score"],
                                                                np.float32(1))))
    ga, gb = _both(sm, s.hi[0], s.lo[0], hs, ls, gate, hist)
    ra = ga.Match(npose, [0, 0, 0, 1, 0, 0, 0], node, 0.3)
    _assert_same_result(ra, gb.Match(npose, [0, 0, 0, 1, 0, 0, 0], node, 0.3))
    _assert_oracle(_oracle_matcher(oracle, hs, ls, hist, gate).match(
        npose, [0, 0, 0, 1, 0, 0, 0], _odict(node), 0.3), ra)
    assert ra is None or ra["best_offset"] != best["best_offset"] or \
        ra["best_scan_index"] != best["best_scan_index"]
    for m in (a, b, ga, gb):
        m.close()
    s.close()


def test_config5_node(sm, oracle):
    """A 65,536-point config-5 node on a submap of 20 config-5 scans (64 x 1024)."""
    occ, cell, origin = synthetic.make_building(4, size_m=40.0)
    rng = np.random.RandomState(11)
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**INSERT))
    hi, lo = sm.DeviceHybridGrid.empty(0.1), sm.DeviceHybridGrid.empty(0.45)
    base = synthetic.random_free_pose_3d(occ, cell, origin, rng)
    for k in range(20):
        pose = base + np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), 0.0,
                                rng.uniform(-0.3, 0.3)])
        _, pts = _scan(occ, cell, origin, pose, 64, 1024, 20.0, k)
        ins.Insert(pose[:3].astype(np.float32), pts, None, hi)
        ins.Insert(pose[:3].astype(np.float32), pts, None, lo)
    hs, ls = _device_spec(hi), _device_spec(lo)
    od = dict(worlds3d.fast_options(depth=8, frd=3, xy=1.0, z=0.5, angular=0.05),
              min_rotational_score=0.0, min_low_resolution_score=0.3)
    hist = np.ones(24, np.float32)
    a, b = _both(sm, hi, lo, hs, ls, od, hist)
    _assert_levels_equal(a, b, 8)
    cloud = synthetic.cast_lidar_3d(occ, cell, origin, base, rings=64, azimuths=1024,
                                    max_range=20.0, seed=99)
    cloud = cloud[np.resize(np.arange(len(cloud)), 65536)]
    node = _node(sm, cloud, hist)
    npose = synthetic.yaw_pose7(base[0] + 0.3, base[1] - 0.2, base[2], base[3] + 0.02)
    ident = [0, 0, 0, 1, 0, 0, 0]
    ra = a.Match(npose, ident, node, 0.3)
    _assert_same_result(ra, b.Match(npose, ident, node, 0.3))
    assert ra is not None
    _assert_oracle(_oracle_matcher(oracle, hs, ls, hist, od).match(npose, ident, _odict(node),
                                                                   0.3), ra)
    for m in (a, b, hi, lo, ins):
        m.close()


# ---- 4. independence from later inserts and from the handles' destruction ----
def test_independent_of_handles(sm):
    s = _Submap(sm, 5, 3)
    od = worlds3d.fast_options(depth=5, frd=2, xy=0.5, z=0.3, angular=0.05)
    hist = np.ones(24, np.float32)
    a = sm.FastCorrelativeScanMatcher3D.from_device_grids(s.hi[0], s.lo[0], hist, _opts(sm, od))
    pose, cloud = s.last
    node = _node(sm, cloud[::3], hist)
    npose = synthetic.yaw_pose7(pose[0] + 0.1, pose[1], pose[2], pose[3])
    ident = [0, 0, 0, 1, 0, 0, 0]
    before = (a.Match(npose, ident, node, 0.2), _levels(a, 5))
    s.insert(3)
    s.close()
    after = (a.Match(npose, ident, node, 0.2), _levels(a, 5))
    _assert_same_result(before[0], after[0])
    for (la, va), (lb, vb) in zip(before[1], after[1]):
        np.testing.assert_array_equal(la, lb)
        np.testing.assert_array_equal(va, vb)
    a.close()


# ---- 5. a batch mixing matchers from both entry points ----
def test_batch_mixes_both_entry_points(sm):
    subs = [_Submap(sm, 20 + i, 3) for i in range(2)]
    od = worlds3d.fast_options(depth=5, frd=3, xy=0.5, z=0.3, angular=0.05)
    hist = np.ones(24, np.float32)
    ms = []
    for s in subs:
        hs, ls = s.specs()
        ms += list(_both(sm, s.hi[0], s.lo[0], hs, ls, od, hist))
    nodes, jobs = [], []
    for i, s in enumerate(subs):
        pose, cloud = s.last
        nodes.append(_node(sm, cloud[::3], hist))
        npose = synthetic.yaw_pose7(pose[0] + 0.1, pose[1] - 0.05, pose[2], pose[3])
        for m in (2 * i, 2 * i + 1):
            jobs.append((m, i, False, npose, [0, 0, 0, 1, 0, 0, 0], 0.2))
            jobs.append((m, i, True, [0, 0, 0] + list(npose[3:]), [0, 0, 0, 1, 0, 0, 0], 0.2))
    got, _ = sm.match_batch3d(ms, nodes, jobs, max_concurrency=4)
    for (mi, ni, full, npose, spose, min_score), r in zip(jobs, got):
        single = ms[mi].match_raw(full, npose, spose, nodes[ni], min_score)[0]
        _assert_same_result(r, single)
    assert any(r is not None for r in got)
    for i in range(2):   # the device-built matcher's jobs == the list-built matcher's
        _assert_same_result(got[4 * i], got[4 * i + 2])
        _assert_same_result(got[4 * i + 1], got[4 * i + 3])
    for m in ms:
        m.close()
    for s in subs:
        s.close()


# ---- 6. refusals ----
def _create(sm, hi, lo, o, out):
    from cartographer_b200._lib import lib
    hist = np.zeros(4, np.float32)
    return lib().csm_matcher3d_create_from_grid3d(
        hi, C.c_int32(0), lo, hist.ctypes.data_as(C.POINTER(C.c_float)), C.c_int32(4),
        None if o is None else C.byref(o), out)


@pytest.mark.parametrize("case", ["null_hi", "null_lo", "null_options", "null_out", "depth0",
                                  "depth13", "frd0"])
def test_refusals(sm, case):
    g = _handle(sm, 0.1, [[0, 0, 0]], [20000])
    od = dict(worlds3d.fast_options(depth=3, frd=2))
    if case == "depth0":
        od["branch_and_bound_depth"] = 0
    if case == "depth13":
        od["branch_and_bound_depth"] = 13
    if case == "frd0":
        od["full_resolution_depth"] = 0
    o = sm.CsmOptions3D(od["branch_and_bound_depth"], od["full_resolution_depth"], 0.0, 0.0,
                        0.5, 0.3, 0.05)
    sentinel = C.c_void_p(0x1234)
    rc = _create(sm, None if case == "null_hi" else g._h, None if case == "null_lo" else g._h,
                 None if case == "null_options" else o,
                 None if case == "null_out" else C.byref(sentinel))
    assert rc == 1   # CSM_E_INVALID
    assert sentinel.value == 0x1234
    g.close()


def test_refuses_handles_on_two_devices(sm):
    if sm.device_count() < 2:
        pytest.skip("one GPU")
    a = sm.DeviceHybridGrid(synthetic.HybridGridSpec(0.1, np.zeros((1, 3), np.int32),
                                                     np.array([20000], np.uint16)), device=0)
    b = sm.DeviceHybridGrid(synthetic.HybridGridSpec(0.45, np.zeros((1, 3), np.int32),
                                                     np.array([20000], np.uint16)), device=1)
    o = sm.CsmOptions3D(3, 2, 0.0, 0.0, 0.5, 0.3, 0.05)
    sentinel = C.c_void_p(0x1234)
    assert _create(sm, a._h, b._h, o, C.byref(sentinel)) == 1
    assert sentinel.value == 0x1234
    a.close()
    b.close()


# ---- 7. ConstraintBuilder3D on device submaps ----
@pytest.mark.parametrize("refine", [False, True])
def test_constraint_builder_on_device_submaps(sm, refine):
    from cartographer_b200 import constraint_builder as cb
    subs = [_Submap(sm, 30 + i, 3) for i in range(2)]
    hist = np.ones(24, np.float32)
    opts = cb.ConstraintBuilderOptions3D(
        sampling_ratio=1.0, min_score=0.2, global_localization_min_score=0.2,
        branch_and_bound_depth=5, full_resolution_depth=3, min_rotational_score=0.0,
        min_low_resolution_score=0.1, linear_xy_search_window=0.5, linear_z_search_window=0.3,
        angular_search_window=0.05,
        ceres_scan_matcher_options_3d=sm.CeresScanMatcherOptions3D(
            occupied_space_weight_0=1.0, occupied_space_weight_1=6.0, translation_weight=5.0,
            rotation_weight=4e2) if refine else None)
    records = []
    executors = []
    for device_side in (True, False):
        builder = cb.ConstraintBuilder3D(opts)
        executors.append(builder.executor)
        for i, s in enumerate(subs):
            if device_side:
                sub = cb.Submap3D(s.hi[0], s.lo[0], hist)
            else:
                hs, ls = s.specs()
                sub = cb.Submap3D(hs, ls, hist)
            pose, cloud = s.last
            node = _node(sm, cloud[::3], hist)
            npose = synthetic.yaw_pose7(pose[0] + 0.1, pose[1] - 0.05, pose[2], pose[3])
            builder.MaybeAddConstraint((0, i), sub, (1, i), node, npose, [0, 0, 0, 1, 0, 0, 0])
            builder.MaybeAddGlobalConstraint((0, i), sub, (1, 10 + i), node, list(npose[3:]),
                                             [1, 0, 0, 0])
        builder.NotifyEndOfNode()
        builder.WhenDone(lambda r: None)
        records.append(builder.last_records.copy())
        if device_side:
            assert executors[0].grids == {}
    assert records[0].tobytes() == records[1].tobytes()
    assert records[0]["found"].sum() >= 2
    if refine:
        assert executors[0].stats["refined"] > 0 and len(executors[1].grids) > 0
    for e in executors:
        for sid in list(e.matchers):
            e.delete_matcher(sid)
    for s in subs:
        s.close()
