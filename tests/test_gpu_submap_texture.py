"""Submap textures from device-resident grids (csm_grid3d_to_texture, csm_rt_grid2d_to_texture)
against the CPU restatement (tests/submap_texture_oracle.cc): decompressed cells, width, height,
resolution and the slice pose's bits, after 3D and 2D inserts, under rotated and tilted poses,
at the edges (a long column whose float sum depends on its order, a single voxel, empty grids,
the 2 x 2 wrap, 1 x 1 crops, all 32768 cell values), repeated calls and refusals."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import grid_proto_ref as R
from tests import insert3d_oracle as O3
from tests import submap_texture_oracle as T

pytestmark = pytest.mark.gpu

INSERT3D = dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
                intensity_threshold=40.0)   # trajectory_builder_3d.lua
CSM_E_INVALID, CSM_E_CAPACITY = 1, 3


def _quat(roll, pitch, yaw):
    """Quaterniond of RollPitchYaw (transform.h: yaw * pitch * roll), as (w, x, y, z)."""
    cr, sr = math.cos(roll / 2), math.sin(roll / 2)
    cp, sp = math.cos(pitch / 2), math.sin(pitch / 2)
    cy, sy = math.cos(yaw / 2), math.sin(yaw / 2)
    return (cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy,
            cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy)


def _pose(t, roll=0.0, pitch=0.0, yaw=0.0):
    return tuple(t) + _quat(roll, pitch, yaw)


POSES = {
    "identity": (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0),
    "yaw30": _pose((3.2, -1.7, 0.4), yaw=math.radians(30)),
    "yaw45": _pose((-12.5, 4.05, 1.0), yaw=math.radians(45)),
    "yaw90": _pose((0.05, 0.0, -0.3), yaw=math.radians(90)),
    "tilted": _pose((1.0, 2.0, 0.5), roll=0.03, pitch=-0.02, yaw=math.radians(-70)),
}


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


@pytest.fixture(scope="module")
def lib():
    from cartographer_b200._lib import lib as L
    return L()


def _assert_texture(msg, want):
    got = T.parse(msg)
    assert got["gzipped"][:10] == T.GZIP_HEADER
    assert got["cells"] == want["cells"]
    assert (got["width"], got["height"]) == (want["width"], want["height"])
    assert T.same_bits((got["resolution"],), (want["resolution"],))
    assert T.same_bits(got["slice_pose"], want["slice_pose"]), (got["slice_pose"],
                                                                 want["slice_pose"])
    assert msg == T.message(want, gzipped=got["gzipped"])   # the framing, byte for byte


def _ordered(ora):
    keep = ora.values != 0
    idx, val, _ = R.walk((ora.indices()[keep], ora.values[keep]))
    return idx, val


def _handle(sm, idx, val, resolution=0.1):
    return sm.DeviceHybridGrid(synthetic.HybridGridSpec(
        resolution, np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(val, np.uint16)))


def _check3d(grid, idx, val, pose):
    before = grid.read()
    msg = grid.to_texture(pose)
    _assert_texture(msg, T.texture3d(idx, val, grid.resolution, pose))
    assert grid.to_texture(pose) == msg   # repeated calls give identical bytes
    after = grid.read()
    np.testing.assert_array_equal(before[0], after[0])
    np.testing.assert_array_equal(before[1], after[1])
    return msg


# ---- 3D: after every config-5-size insert, both grids, every pose ----
def test_textures_after_every_insert(sm):
    rng = np.random.RandomState(17)
    occ, cell, origin = synthetic.make_building(4, size_m=40.0)
    pairs = [(sm.DeviceHybridGrid.empty(0.1), O3.HybridGrid(0.1)),
             (sm.DeviceHybridGrid.empty(0.45), O3.HybridGrid(0.45))]
    dev_ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**INSERT3D))
    ora_ins = O3.RangeDataInserter3D(**INSERT3D)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng, margin_m=3.0) for _ in range(4)]
    names = sorted(POSES)
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
            # every pose on the first and last inserts, one pose in turn in between
            for name in (names if k in (0, 49) else [names[k % len(names)]]):
                _check3d(dev, idx, val, POSES[name])
    for dev, _ in pairs:
        dev.close()
    dev_ins.close()


def test_long_column_sums_in_iteration_order(sm):
    """Thousands of voxels in one pixel, in several 64^3 blocks: the float probability sum of
    the iteration order differs from the sum in list order and in sorted order, and the device
    gives the iteration order's texture."""
    rng = np.random.RandomState(9)
    z = np.arange(-1500, 1500)
    idx = np.stack([np.full(z.size, 3), np.full(z.size, -70), z], 1).astype(np.int32)
    # a second column in other 64^3 blocks of x and y
    idx2 = idx.copy()
    idx2[:, 0], idx2[:, 1] = 130, 40
    idx = np.concatenate([idx, idx2])
    val = rng.randint(16400, 32768, len(idx)).astype(np.uint16)
    perm = rng.permutation(len(idx))
    idx, val = idx[perm], val[perm]
    g = _handle(sm, idx, val)
    w_idx, w_val = R.walk((idx, val))[:2]
    p = (np.float32(w_val) * np.float32((0.9 - 0.1) / 32766) +
         np.float32(np.float32(0.1) - np.float32((0.9 - 0.1) / 32766)))
    col = w_idx[:, 0] == 3
    sums = set()
    for order in (np.arange(col.sum()), np.argsort(p[col]), np.argsort(-p[col])):
        acc = np.float32(0)
        for v in p[col][order]:
            acc = np.float32(acc + v)
        sums.add(float(acc))
    assert len(sums) > 1   # the order matters for this column
    for name in sorted(POSES):
        _check3d(g, w_idx, w_val, POSES[name])
    g.close()


def test_single_voxel_empty_and_below_limit(sm):
    one = _handle(sm, [[3, -4, 5]], [30000])
    for name in sorted(POSES):
        _check3d(one, np.array([[3, -4, 5]], np.int32), np.array([30000], np.uint16),
                 POSES[name])
    one.close()
    # a column of 4 voxels: z_difference 3 draws the pixel
    col = _handle(sm, [[0, 0, 0], [0, 0, 3], [0, 0, 1], [0, 0, 2]], [30000, 20000, 16400, 32767])
    idx, val = col.voxels()
    msg = _check3d(col, idx, val, POSES["identity"])
    assert T.parse(msg)["cells"] != b"\0\0"
    col.close()
    empty = sm.DeviceHybridGrid.empty(0.1)
    below = _handle(sm, [[1, 2, 3], [4, 5, 6], [0, 0, 0]], [1, 16383, 16000])   # p < 0.501
    for g in (empty, below):
        idx, val = g.voxels()
        for name in sorted(POSES):
            msg = _check3d(g, idx, val, POSES[name])
            t = T.parse(msg)
            assert (t["width"], t["height"]) == (2, 2) and t["cells"] == bytes(8)
        g.close()


def test_refusals_3d(sm, lib):
    g = _handle(sm, [[0, 0, 0], [0, 0, 5]], [30000, 30000])
    before = g.read()
    msg = g.to_texture(POSES["yaw30"])
    size = C.c_int64(-7)
    buf = np.full(len(msg), 0xAB, np.uint8)
    pose = np.array(POSES["yaw30"], np.float64)
    pp = pose.ctypes.data_as(C.c_void_p)
    bp = buf.ctypes.data_as(C.c_void_p)
    assert lib.csm_grid3d_to_texture(g._h, pp, bp, C.c_int64(len(msg) - 1),
                                     C.byref(size)) == CSM_E_CAPACITY
    assert size.value == len(msg) and (buf == 0xAB).all()
    assert lib.csm_grid3d_to_texture(g._h, pp, None, C.c_int64(0), C.byref(size)) == 0
    assert size.value == len(msg)
    for bad in (np.nan, np.inf):
        p2 = pose.copy()
        p2[4] = bad
        size.value = -7
        assert lib.csm_grid3d_to_texture(g._h, p2.ctypes.data_as(C.c_void_p), bp,
                                         C.c_int64(buf.size), C.byref(size)) == CSM_E_INVALID
        assert size.value == -7 and (buf == 0xAB).all()
    assert lib.csm_grid3d_to_texture(g._h, None, bp, C.c_int64(buf.size),
                                     C.byref(size)) == CSM_E_INVALID
    after = g.read()
    np.testing.assert_array_equal(before[1], after[1])
    assert g.to_texture(POSES["yaw30"]) == msg
    g.close()


# ---- 2D ----
def _world_scan(occ, spec, pose, seed, beams=1081, max_range=8.0):
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


LOCAL = _pose((0.4, -2.25, 0.0), yaw=math.radians(30))


def _check2d(grid, pose=LOCAL, tsdf=None):
    st = grid.read()
    msg = grid.to_texture(pose)
    if tsdf is None:
        want = T.texture2d(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box, pose)
    else:
        want = T.texture2d(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box, pose,
                           st.weight_cells, *tsdf)
    _assert_texture(msg, want)
    assert grid.to_texture(pose) == msg
    after = grid.read()
    np.testing.assert_array_equal(st.cells, after.cells)
    assert st.known_cells_box == after.known_cells_box
    return msg


def test_probability_grid_inserts_and_crops(sm, world):
    spec, occ, poses = world
    ins = sm.ProbabilityGridRangeDataInserter2D()
    g = sm.RealTimeGrid2D.empty(0.05, poses[0][0] + 2.5, poses[0][1] + 2.5)
    t = T.parse(_check2d(g))   # an empty known-cells box: 1 x 1 at offset 0
    assert (t["width"], t["height"], t["cells"]) == (1, 1, b"\0\0")
    for k, pose in enumerate(poses):
        origin, returns, misses = _world_scan(occ, spec, pose, 100 + k)
        ins.Insert(origin, returns, g, misses)
        _check2d(g, POSES["identity"] if k % 2 else LOCAL)
        crop = g.ComputeCroppedGrid()
        _check2d(crop)
        crop.close()
    g.close()
    empty = sm.RealTimeGrid2D.empty(0.05, 1.0, 1.0, 10, 10)
    one = empty.ComputeCroppedGrid()   # an empty known-cells box crops to 1 x 1
    assert one.shape == (1, 1)
    _check2d(one)
    _check2d(empty, POSES["tilted"])
    for h in (one, empty, ins):
        h.close()


def test_every_cell_value(sm):
    """A pitched handle made from cells that holds each of the 32768 values once (value 0
    unknown), and its 1 x 1 crops."""
    rng = np.random.RandomState(4)
    cells = rng.permutation(32768).astype(np.uint16).reshape(128, 256)
    big = np.zeros((130, 261), np.uint16)   # 261 is not a multiple of 8: a pitched handle
    big[1:129, 3:259] = cells
    g = sm.RealTimeGrid2D(synthetic.GridSpec(big, 0.05, 3.0, -2.0))
    for name in sorted(POSES):
        _check2d(g, POSES[name])
    g.close()
    single = np.zeros((5, 7), np.uint16)
    single[3, 2] = 12345
    g = sm.RealTimeGrid2D(synthetic.GridSpec(single, 0.05, 0.0, 0.0))
    crop = g.ComputeCroppedGrid()
    assert crop.shape == (1, 1)
    for h in (g, crop):
        _check2d(h)
        h.close()


def test_tsdf_inserts(sm, world):
    spec, occ, poses = world
    opts = sm.TSDFRangeDataInserterOptions2D()
    ins = sm.TSDFRangeDataInserter2D(opts)
    g = sm.RealTimeGrid2D.empty_tsdf(0.05, poses[0][0] + 2.5, poses[0][1] + 2.5,
                                     opts.truncation_distance, opts.maximum_weight)
    tsdf = (opts.truncation_distance, opts.maximum_weight)
    _check2d(g, tsdf=tsdf)
    for k, pose in enumerate(poses[:5]):
        origin, returns, _ = _world_scan(occ, spec, pose, 200 + k)
        ins.Insert(origin, returns, g)
        _check2d(g, POSES["yaw45"] if k % 2 else LOCAL, tsdf=tsdf)
    g.close()
    ins.close()


def test_refusals_2d(sm, lib):
    rng = np.random.RandomState(2)
    cells = rng.randint(0, 32768, (23, 37)).astype(np.uint16)
    g = sm.RealTimeGrid2D(synthetic.GridSpec(cells, 0.05, -0.0, 3.0))
    msg = _check2d(g)
    size = C.c_int64(-7)
    buf = np.full(len(msg), 0xAB, np.uint8)
    pose = np.array(LOCAL, np.float64)
    pp, bp = pose.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p)
    assert lib.csm_rt_grid2d_to_texture(g._h, pp, bp, C.c_int64(len(msg) - 1),
                                        C.byref(size)) == CSM_E_CAPACITY
    assert size.value == len(msg) and (buf == 0xAB).all()
    assert lib.csm_rt_grid2d_to_texture(g._h, pp, None, C.c_int64(0), C.byref(size)) == 0
    assert size.value == len(msg)
    p2 = pose.copy()
    p2[0] = np.nan
    size.value = -7
    assert lib.csm_rt_grid2d_to_texture(g._h, p2.ctypes.data_as(C.c_void_p), bp,
                                        C.c_int64(buf.size), C.byref(size)) == CSM_E_INVALID
    assert size.value == -7 and (buf == 0xAB).all()
    np.testing.assert_array_equal(g.read().cells, cells)
    assert g.to_texture(LOCAL) == msg
    g.close()
