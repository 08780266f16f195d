"""Saving device-resident grids (csm_grid3d_voxels, csm_grid3d_to_proto, csm_rt_grid2d_to_proto)
against the test-side references: the voxel set of the CPU insert restatement in the order of the
HybridGrid walk restatement (tests/hybrid_grid_walk.cc), the Grid2D / HybridGrid encoders of
tests/grid_proto_ref.py byte for byte, round trips through the existing loaders, edge cases and
refusals."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

from benchmarks import synthetic
from tests import grid_proto_ref as R
from tests import insert3d_oracle as O
from tests import protowire as pw
from tests import worlds3d

pytestmark = pytest.mark.gpu

INSERT3D = dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
                intensity_threshold=40.0)   # trajectory_builder_3d.lua
CSM_E_CAPACITY = 3


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


@pytest.fixture(scope="module")
def lib():
    from cartographer_b200._lib import lib as L
    return L()


def _ordered(ora):
    """The non-zero voxels of an insert-oracle grid in the walk restatement's order."""
    keep = ora.values != 0
    idx, val, _ = R.walk((ora.indices()[keep], ora.values[keep]))
    return idx, val


def _assert_saved(grid, idx, val):
    got_idx, got_val = grid.voxels()
    np.testing.assert_array_equal(got_idx, idx)
    np.testing.assert_array_equal(got_val, val)
    assert grid.to_proto() == R.hybrid_grid_message(grid.resolution, idx, val)


# ---- 3D: after every insert, from empty handles and from handles made from lists ----
@pytest.mark.parametrize("from_voxels", [False, True], ids=["empty", "from_voxels"])
def test_voxels_and_proto_after_every_insert(sm, from_voxels):
    rng = np.random.RandomState(11 + from_voxels)
    occ, cell, origin = synthetic.make_building(4, size_m=40.0)
    if from_voxels:
        vox = worlds3d.random_voxels(rng, 300, 16, 0.1)
        lvox = worlds3d.random_voxels(rng, 80, 5, 0.45)
        pairs = [(sm.DeviceHybridGrid(vox), O.HybridGrid(0.1, vox.indices, vox.values)),
                 (sm.DeviceHybridGrid(lvox), O.HybridGrid(0.45, lvox.indices, lvox.values))]
    else:
        pairs = [(sm.DeviceHybridGrid.empty(0.1), O.HybridGrid(0.1)),
                 (sm.DeviceHybridGrid.empty(0.45), O.HybridGrid(0.45))]
    dev_ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**INSERT3D))
    ora_ins = O.RangeDataInserter3D(**INSERT3D)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng, margin_m=3.0) for _ in range(4)]
    for k in range(50):
        pose = poses[k % len(poses)] + np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), 0.0,
                                                 rng.uniform(-0.5, 0.5)])
        cloud = synthetic.cast_lidar_3d(occ, cell, origin, pose, rings=64, azimuths=1024,
                                        max_range=20.0, seed=int(rng.randint(1 << 30)))
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T +
               pose[:3]).astype(np.float32)
        org = pose[:3].astype(np.float32)
        for dev, ora in pairs:
            dev_ins.Insert(org, pts, None, dev)
            ora_ins.insert(org, pts, None, ora)
            idx, val = _ordered(ora)
            _assert_saved(dev, idx, val)
    # the last messages once more through protowire.hybrid_grid itself (hybrid_grid_message is
    # its vectorised form, tests/test_grid_to_proto_cpu.py)
    for dev, ora in pairs:
        idx, val = _ordered(ora)
        assert dev.to_proto() == pw.hybrid_grid(dev.resolution, idx, val)
    # the dense boxes carry growth slack beyond the non-zero voxels
    lo, vol = pairs[0][0].read()
    idx, _ = pairs[0][0].voxels()
    assert (np.array(vol.shape[::-1]) > idx.max(0) - idx.min(0) + 1).any()
    # round trips: a handle made from voxels() holds the same cells; the matcher from the two
    # messages equals the matcher from the two handles, level by level and match by match
    for dev, _ in pairs:
        idx, val = dev.voxels()
        again = sm.DeviceHybridGrid(synthetic.HybridGridSpec(dev.resolution, idx, val))
        a_idx, a_val = again.voxels()
        np.testing.assert_array_equal(a_idx, idx)
        np.testing.assert_array_equal(a_val, val)
        again.close()
    od = worlds3d.fast_options(depth=8, frd=3)
    o = sm.FastCorrelativeScanMatcherOptions3D(
        od["branch_and_bound_depth"], od["full_resolution_depth"], od["min_rotational_score"],
        od["min_low_resolution_score"], od["linear_xy_search_window"],
        od["linear_z_search_window"], od["angular_search_window"])
    hist = np.zeros(10, np.float32)
    hi, lo_grid = pairs[0][0], pairs[1][0]
    a = sm.FastCorrelativeScanMatcher3D.from_proto(hi.to_proto(), lo_grid.to_proto(), hist, o)
    b = sm.FastCorrelativeScanMatcher3D.from_device_grids(hi, lo_grid, hist, o)
    for d in range(od["branch_and_bound_depth"]):
        la, va = a.precomputation_grid(d)
        lb, vb = b.precomputation_grid(d)
        np.testing.assert_array_equal(la, lb)
        np.testing.assert_array_equal(va, vb)
    low = synthetic.voxel_downsample(cloud, 0.45)
    node = sm.TrajectoryNodeData3D(cloud, low, hist)
    q = [math.cos(pose[3] / 2), 0.0, 0.0, math.sin(pose[3] / 2)]
    node_pose = list(pose[:3] + np.array([0.3, -0.2, 0.1])) + q
    ra = a.Match(node_pose, [0, 0, 0, 1, 0, 0, 0], node, 0.5)
    rb = b.Match(node_pose, [0, 0, 0, 1, 0, 0, 0], node, 0.5)
    assert (ra is None) == (rb is None)
    if ra is not None:
        for key in ra:
            np.testing.assert_array_equal(np.asarray(ra[key]), np.asarray(rb[key]))
    for m in (a, b):
        m.close()
    for dev, _ in pairs:
        dev.close()
    dev_ins.close()


def _handle(sm, idx, val, resolution=0.1):
    return sm.DeviceHybridGrid(synthetic.HybridGridSpec(
        resolution, np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(val, np.uint16)))


def _box_not_multiple(rng):
    idx = np.unique(np.stack([rng.randint(-37, 51, 400), rng.randint(-70, -3, 400),
                              rng.randint(5, 14, 400)], 1), axis=0)
    return idx, rng.randint(1, 32768, len(idx))


EDGES = (-65, -64, -9, -8, -1, 0, 7, 8, 63, 64)
CASES = {
    "one_voxel": lambda rng: ([[3, -4, 5]], [7]),
    "cube_low_faces": lambda rng: ([[-8192, -8192, -8192], [-8150, -8192, -8120],
                                    [-8192, -8100, -8170], [-8180, -8130, -8192]], [1, 2, 3, 4]),
    "cube_high_faces": lambda rng: ([[8191, 8191, 8191], [8150, 8191, 8120], [8191, 8100, 8170],
                                     [8180, 8130, 8191]], [1, 2, 3, 4]),
    "edges_both_signs": lambda rng: (
        np.array(np.meshgrid(EDGES, EDGES, EDGES, indexing="ij")).reshape(3, -1).T,
        rng.randint(1, 32768, 1000)),
    "box_not_multiple_of_8_or_64": _box_not_multiple,
    "zero_entries_skipped": lambda rng: ([[0, 0, 0], [1, 2, 3], [-5, 9, 2], [100, 0, 0]],
                                         [0, 9, 0, 32767]),
    "value_32767": lambda rng: ([[-1, -1, -1], [0, 0, 0]], [32767, 32767]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_edge_cases_3d(sm, case):
    rng = np.random.RandomState(3)
    idx, val = CASES[case](rng)
    idx, val = np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(val, np.uint16)
    g = _handle(sm, idx, val)
    before = g.read()
    keep = val != 0
    want_idx, want_val, _ = R.walk((idx[keep], val[keep]))
    _assert_saved(g, want_idx, want_val)
    lo, vol = g.read()
    np.testing.assert_array_equal(lo, before[0])
    np.testing.assert_array_equal(vol, before[1])
    g.close()


def test_empty_handle(sm):
    for g in (sm.DeviceHybridGrid.empty(0.1), _handle(sm, [[4, 4, 4]], [0])):
        idx, val = g.voxels()
        assert idx.shape == (0, 3) and val.shape == (0,)
        assert g.to_proto() == b"\x0d" + struct.pack("<f", 0.1)
        g.close()


def test_too_small_capacity_writes_nothing(sm, lib):
    g = _handle(sm, [[1, 2, 3], [4, 5, 6], [-7, 8, 9]], [10, 20, 30])
    idx = np.full((3, 3), -99, np.int32)
    val = np.full(3, 99, np.uint16)
    n = C.c_int64()
    p32, p16 = idx.ctypes.data_as(C.c_void_p), val.ctypes.data_as(C.c_void_p)
    assert lib.csm_grid3d_voxels(g._h, p32, p16, C.c_int64(2), C.byref(n)) == CSM_E_CAPACITY
    assert n.value == 3
    assert (idx == -99).all() and (val == 99).all()
    assert lib.csm_grid3d_voxels(g._h, p32, None, C.c_int64(3), C.byref(n)) == 1
    msg = g.to_proto()
    buf = np.full(len(msg), 0xAB, np.uint8)
    size = C.c_int64()
    assert lib.csm_grid3d_to_proto(g._h, buf.ctypes.data_as(C.c_void_p), C.c_int64(len(msg) - 1),
                                   C.byref(size)) == CSM_E_CAPACITY
    assert size.value == len(msg) and (buf == 0xAB).all()
    assert lib.csm_grid3d_to_proto(g._h, None, C.c_int64(0), C.byref(size)) == 0
    assert size.value == len(msg)
    g.close()


# ---- 2D ----
def _world_scan(occ, spec, pose, seed, beams=541, max_range=8.0):
    pts = synthetic.cast_scan(occ, spec, pose, beams=beams, max_range=max_range, seed=seed)
    c, s = math.cos(pose[2]), math.sin(pose[2])
    w = np.stack([c * pts[:, 0] - s * pts[:, 1] + pose[0], s * pts[:, 0] + c * pts[:, 1] + pose[1],
                  np.zeros(len(pts))], 1).astype(np.float32)
    far = np.hypot(pts[:, 0], pts[:, 1]) >= max_range - 0.05
    return np.float32([pose[0], pose[1], 0]), w[~far], w[far]


@pytest.fixture(scope="module")
def world():
    spec, occ = synthetic.make_grid2d(21, size_cells=600)
    rng = np.random.RandomState(5)
    poses = [synthetic.random_free_pose(occ, spec, rng, margin_cells=40) for _ in range(8)]
    return spec, occ, poses


def _want2d(grid, tsdf=None):
    st = grid.read()
    if tsdf is None:
        return R.grid2d_message(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box)
    return R.grid2d_message(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box,
                            st.weight_cells, *tsdf)


class Grid2DInfo(C.Structure):   # csm_grid2d_info
    _fields_ = [("num_x_cells", C.c_int32), ("num_y_cells", C.c_int32),
                ("resolution", C.c_double), ("max_x", C.c_double), ("max_y", C.c_double),
                ("min_correspondence_cost", C.c_float), ("max_correspondence_cost", C.c_float),
                ("is_tsdf", C.c_int32), ("reserved", C.c_int32)]


def _decode(lib, blob):
    info = Grid2DInfo()
    buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
    assert lib.csm_grid2d_proto_decode(buf, C.c_int64(len(blob)), C.byref(info), None,
                                       C.c_int64(0)) == 0
    cells = np.zeros(info.num_x_cells * info.num_y_cells, np.uint16)
    assert lib.csm_grid2d_proto_decode(buf, C.c_int64(len(blob)), C.byref(info),
                                       cells.ctypes.data_as(C.POINTER(C.c_uint16)),
                                       C.c_int64(cells.size)) == 0
    return info, cells.reshape(info.num_y_cells, info.num_x_cells)


def _check_loaders(sm, lib, grid):
    """Decode gives back the limits and cells; the stack from the message equals the stack from
    the handle level by level."""
    blob = grid.to_proto()
    st = grid.read()
    info, cells = _decode(lib, blob)
    np.testing.assert_array_equal(cells, st.cells)
    assert (info.resolution, info.max_x, info.max_y) == (st.resolution, st.max_x, st.max_y)
    opts = sm.FastCorrelativeScanMatcherOptions2D(7.0, 0.5, 4)
    a = sm.FastCorrelativeScanMatcher2D.from_proto(blob, opts)
    b = sm.FastCorrelativeScanMatcher2D.from_device_grid(grid, opts)
    for level in range(4):
        np.testing.assert_array_equal(a.precomputation_grid(level), b.precomputation_grid(level))
    a.close()
    b.close()


def test_probability_grid_inserts_and_crops(sm, lib, world):
    spec, occ, poses = world
    ins = sm.ProbabilityGridRangeDataInserter2D()
    g = sm.RealTimeGrid2D.empty(0.05, poses[0][0] + 2.5, poses[0][1] + 2.5)
    assert g.read().known_cells_box is None and g.to_proto() == _want2d(g)   # no box field
    for k, pose in enumerate(poses):
        origin, returns, misses = _world_scan(occ, spec, pose, 100 + k)
        ins.Insert(origin, returns, g, misses)
        assert g.to_proto() == _want2d(g)
        crop = g.ComputeCroppedGrid()
        assert crop.read().known_cells_box[:2] == (0, 0)   # a box with zero coordinates
        assert crop.to_proto() == _want2d(crop)
        if k in (0, len(poses) - 1):
            _check_loaders(sm, lib, crop)
            _check_loaders(sm, lib, g)
        crop.close()
    g.close()
    empty = sm.RealTimeGrid2D.empty(0.05, 1.0, 1.0, 10, 10)
    one = empty.ComputeCroppedGrid()   # an empty known-cells box crops to 1 x 1
    assert one.shape == (1, 1) and one.to_proto() == _want2d(one)
    for h in (one, empty, ins):
        h.close()


def test_pitched_handle_and_negative_zero(sm, lib):
    rng = np.random.RandomState(2)
    cells = rng.randint(0, 32768, (23, 37)).astype(np.uint16)
    cells[:3] = 0
    g = sm.RealTimeGrid2D(synthetic.GridSpec(cells, 0.05, -0.0, 3.0))
    blob = g.to_proto()
    assert blob == _want2d(g)
    assert struct.pack("<d", -0.0) in blob      # -0.0 is written
    _check_loaders(sm, lib, g)
    before = g.read()
    g.to_proto()
    after = g.read()
    np.testing.assert_array_equal(before.cells, after.cells)
    assert before.known_cells_box == after.known_cells_box
    buf = np.full(len(blob), 0xAB, np.uint8)
    size = C.c_int64()
    assert lib.csm_rt_grid2d_to_proto(g._h, buf.ctypes.data_as(C.c_void_p),
                                      C.c_int64(len(blob) - 1), C.byref(size)) == CSM_E_CAPACITY
    assert size.value == len(blob) and (buf == 0xAB).all()
    g.close()


def test_tsdf_inserts(sm, lib, world):
    spec, occ, poses = world
    opts = sm.TSDFRangeDataInserterOptions2D()
    ins = sm.TSDFRangeDataInserter2D(opts)
    g = sm.RealTimeGrid2D.empty_tsdf(0.05, poses[0][0] + 2.5, poses[0][1] + 2.5,
                                     opts.truncation_distance, opts.maximum_weight)
    tsdf = (opts.truncation_distance, opts.maximum_weight)
    assert g.to_proto() == _want2d(g, tsdf)
    for k, pose in enumerate(poses[:5]):
        origin, returns, _ = _world_scan(occ, spec, pose, 200 + k)
        ins.Insert(origin, returns, g)
        blob = g.to_proto()
        assert blob == _want2d(g, tsdf)
    info, cells = _decode(lib, blob)
    assert info.is_tsdf == 1
    np.testing.assert_array_equal(cells, g.read().cells)
    g.close()
    ins.close()
