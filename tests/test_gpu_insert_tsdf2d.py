"""TSDFRangeDataInserter2D with normal estimation and grid growth on the device
(csrc/insert_tsdf2d.cu) against the CPU restatement in tests/insert_tsdf2d_oracle.cc: every tsd cell,
weight cell, limit and the known-cells box bit for bit after every insert, one synchronisation
per insert; refusals that leave the handle unchanged; the real-time matcher and the refinement on
an inserted handle against the same on restated cells."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import insert_tsdf2d_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _pair(sm, **kw):
    opts = sm.TSDFRangeDataInserterOptions2D(**kw)
    return sm.TSDFRangeDataInserter2D(opts), O.TsdfInserter(opts)


def _empty(sm, origin, resolution=0.05, truncation=0.3, max_weight=10.0):
    """ActiveSubmaps2D::CreateGrid for GridType::TSDF on both sides."""
    ora = O.TsdfGrid.create_grid(origin, resolution, truncation, max_weight)
    res, max_x, max_y, nx, ny = ora.limits
    return sm.RealTimeGrid2D.empty_tsdf(res, max_x, max_y, truncation, max_weight, nx, ny), ora


def _from_spec(sm, spec):
    ny, nx = spec.tsd_cells.shape
    ora = O.TsdfGrid(spec.resolution, spec.max_x, spec.max_y, nx, ny, spec.truncation_distance,
                     spec.max_weight, spec.tsd_cells, spec.weight_cells)
    return sm.RealTimeGrid2D(spec), ora


def assert_grid_equal(dev, ora):
    st = dev.read()
    res, max_x, max_y, nx, ny = ora.limits
    assert (st.resolution, st.max_x, st.max_y) == (res, max_x, max_y)
    assert st.cells.shape == (ny, nx) and dev.shape == (ny, nx)
    tsd, weight = ora.arrays()
    np.testing.assert_array_equal(st.cells, tsd)
    np.testing.assert_array_equal(st.weight_cells, weight)
    assert st.known_cells_box == ora.known_box
    return st


def _insert(pair, grids, origin, returns):
    """One insert on both sides; where the restatement refuses, the device must refuse too."""
    from cartographer_b200._lib import CsmError
    dev_ins, ora_ins = pair
    dev, ora = grids
    if ora_ins.insert(origin, returns, ora):
        dev_ins.Insert(origin, returns, dev)
        assert dev_ins.last_stats["host_syncs"] == 1
        return True
    with pytest.raises(CsmError) as e:
        dev_ins.Insert(origin, returns, dev)
    assert e.value.status == 1
    return False


def _world_scan(occ, spec, pose, seed, beams=1081, max_range=8.0):
    """The returns of a scan cast in the synthetic world, in the world frame."""
    pts = synthetic.cast_scan(occ, spec, pose, beams=beams, max_range=max_range, seed=seed)
    c, s = math.cos(pose[2]), math.sin(pose[2])
    w = np.stack([c * pts[:, 0] - s * pts[:, 1] + pose[0], s * pts[:, 0] + c * pts[:, 1] + pose[1],
                  np.zeros(len(pts))], 1).astype(np.float32)
    far = np.hypot(pts[:, 0], pts[:, 1]) >= max_range - 0.05
    return np.float32([pose[0], pose[1], 0]), w[~far]


@pytest.fixture(scope="module")
def world():
    spec, occ = synthetic.make_grid2d(21, size_cells=600)
    rng = np.random.RandomState(5)
    poses = [synthetic.random_free_pose(occ, spec, rng, margin_cells=40) for _ in range(50)]
    return spec, occ, poses


# ---- tsdf_range_data_inserter_2d_test.cc on the device ----
REF = dict(truncation_distance=2.0, maximum_weight=10.0, update_free_space=False,
           num_normal_samples=2, sample_radius=10.0, project_sdf_distance_to_scan_normal=False,
           update_weight_range_exponent=0,
           update_weight_angle_scan_normal_to_ray_kernel_bandwidth=0.0,
           update_weight_distance_cell_to_hit_kernel_bandwidth=0.0)
ORIGIN = np.float32([-0.5, -0.5, 0])
POINT = np.float32([[-0.5, 3.5, 0]])
TWO = np.float32([[-0.5, 3.5, 0], [5.5, 3.5, 0]])


def _ref_grids(sm):
    """MapLimits(1., (1., 7.), CellLimits(8, 1)), truncation 2, maximum weight 10."""
    return (sm.RealTimeGrid2D.empty_tsdf(1.0, 1.0, 7.0, 2.0, 10.0, 8, 1),
            O.TsdfGrid(1.0, 1.0, 7.0, 8, 1, 2.0, 10.0))


@pytest.mark.parametrize("case,options,returns,repeat", [
    ("InsertPoint", {}, POINT, 1001),
    ("InsertPointWithFreeSpaceUpdate", dict(update_free_space=True), POINT, 1001),
    ("InsertPointLinearWeight", dict(update_weight_range_exponent=1), POINT, 1),
    ("InsertPointQuadraticWeight", dict(update_weight_range_exponent=2), POINT, 1),
    ("InsertSmallAnglePointWithoutNormalProjection", {},
     np.float32([[-0.5, 3.5, 0], [5.5, 3.5, 0], [10.5, 3.5, 0]]), 1),
    ("InsertSmallAnglePointWitNormalProjection",
     dict(project_sdf_distance_to_scan_normal=True), TWO, 1),
    ("InsertPointsWithAngleScanNormalToRayWeight",
     dict(update_weight_angle_scan_normal_to_ray_kernel_bandwidth=10.0), TWO, 1),
    ("InsertPointsWithDistanceCellToHit",
     dict(update_weight_distance_cell_to_hit_kernel_bandwidth=10.0), POINT, 1),
])
def test_reference_cases(sm, case, options, returns, repeat):
    pair = _pair(sm, **dict(REF, **options))
    grids = _ref_grids(sm)
    for k in range(repeat):
        assert _insert(pair, grids, ORIGIN, returns)
        if k in (0, repeat - 1):
            assert_grid_equal(*grids)
    assert grids[0].shape[1] > 8   # grew out of the 8 x 1 grid
    if repeat > 1:   # saturated at the maximum weight
        ora = grids[1]
        assert ora.get(*ora.cell_index(-0.5, 2.5))[2] == pytest.approx(10.0, abs=1e-2)


# ---- seeded local-SLAM sequences ----
VARIANTS = {"lua": {}, "free_space": dict(update_free_space=True),
            "unsorted": dict(project_sdf_distance_to_scan_normal=False,
                             update_weight_angle_scan_normal_to_ray_kernel_bandwidth=0.0)}


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("start", ["empty", "cells"])
def test_fifty_seeded_inserts(sm, world, start, variant):
    spec, occ, poses = world
    pair = _pair(sm, **VARIANTS[variant])
    if start == "empty":
        grids = _empty(sm, poses[0][:2])
    else:
        tsdf, _ = synthetic.make_tsdf2d(21, size_cells=600)
        grids = _from_spec(sm, tsdf)
    for k, pose in enumerate(poses):
        origin, returns = _world_scan(occ, spec, pose, seed=k)
        assert _insert(pair, grids, origin, returns)
        assert_grid_equal(*grids)


def test_weights_that_underflow_claim_no_cell(sm, world):
    """A distance kernel so narrow that the band's outer cells get a weight of exactly 0.f: they
    stay unknown, and a later ray may still write them."""
    spec, occ, poses = world
    pair = _pair(sm, update_weight_distance_cell_to_hit_kernel_bandwidth=0.004)
    grids = _empty(sm, poses[3][:2])
    for k in range(4):
        origin, returns = _world_scan(occ, spec, poses[3 + k], seed=30 + k)
        assert _insert(pair, grids, origin, returns)
        st = assert_grid_equal(*grids)
    wide = _empty(sm, poses[3][:2])
    wide_pair = _pair(sm)
    for k in range(4):
        origin, returns = _world_scan(occ, spec, poses[3 + k], seed=30 + k)
        assert _insert(wide_pair, wide, origin, returns)
    assert 0 < np.count_nonzero(st.cells) < np.count_nonzero(wide[0].read().cells)


# ---- edges ----
def test_special_returns(sm):
    """Identical directions (sort ties), returns closer than the truncation distance, z != 0,
    returns on cell borders and exact corners, from a cell corner and from a cell centre."""
    r = 0.05
    for options in ({}, dict(update_free_space=True), VARIANTS["unsorted"]):
        pair = _pair(sm, **options)
        grids = _empty(sm, [0.0, 0.0], r)
        _, max_x, max_y, _, _ = grids[1].limits
        border = lambda k: float(np.float32(max_x - k * r))  # noqa: E731
        o = np.float32([border(50), border(50), 0])   # the origin on a cell corner
        pts = [[o[0] + 1.0, o[1] + 0.5, 0], [o[0] + 2.0, o[1] + 1.0, 0],     # same direction
               [o[0] + 1.5, o[1] + 0.75, 0], [o[0] - 1.0, o[1] - 1.0, 0],
               [o[0] - 2.0, o[1] - 2.0, 0],
               [o[0] + 0.1, o[1] + 0.1, 0], [o[0] - 0.2, o[1], 0],           # closer than 0.3
               [o[0], o[1] + 1.0, 0], [o[0], o[1] - 1.3, 0], [o[0] + 0.8, o[1], 0],
               [o[0] - 0.9, o[1], 0], [o[0] + 0.75, o[1] - 0.75, 0],          # corners
               [o[0] - 0.5, o[1] + 1.0, 0.4], [o[0] + 1.2, o[1] - 0.3, -0.6],  # z != 0
               [border(30), border(62), 0], [border(71), border(40), 0], [border(44), border(44), 0]]
        ret = np.float32(pts)
        assert _insert(pair, grids, o, ret)
        assert_grid_equal(*grids)
        assert _insert(pair, grids, o + np.float32([r / 2, r / 2, 0.2]), ret[::-1].copy())
        assert_grid_equal(*grids)


def test_growth_on_every_side_and_several_doublings(sm):
    for options in ({}, dict(update_free_space=True)):
        pair = _pair(sm, **options)
        grids = _empty(sm, [0.0, 0.0])
        assert _insert(pair, grids, [0, 0, 0], np.float32([[0.3, 0.2, 0], [-0.5, 0.4, 0]]))
        for far in ([-20.0, 0.1], [0.2, 25.0], [31.0, -0.3], [0.4, -33.0]):
            arc = [[far[0] + 0.05 * k * (far[1] != 0.1), far[1] + 0.05 * k, 0] for k in range(5)]
            assert _insert(pair, grids, [0, 0, 0], np.float32(arc))
            assert_grid_equal(*grids)
        assert grids[0].shape[0] >= 800   # several doublings in one insert


def _leaving_return(limits, origin, z=40.0):
    """A steep return whose 2D truncation band ends 0.4 cells past max_x, heading to -y: the
    growth (along the 3D ray) does not reach that far, and RayToPixelMask then walks to cell
    index -1 (its pixel division truncates, its walk does not)."""
    res, max_x, max_y, nx, ny = limits
    d = np.array([math.cos(-0.5), math.sin(-0.5)])
    t_end = (max_x + 0.4 * res - float(origin[0])) / d[0]
    hit = np.asarray(origin[:2], np.float64) + (t_end - 0.3) * d
    return np.float32([[hit[0], hit[1], z]])


def test_refused_calls_leave_the_handle_unchanged(sm, world):
    spec, occ, poses = world
    pair = _pair(sm)
    grids = _empty(sm, poses[2][:2])
    origin, returns = _world_scan(occ, spec, poses[2], seed=2)
    assert _insert(pair, grids, origin, returns)
    before = grids[0].read()
    lib = sm.lib()
    ins = pair[0]._h
    p = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    bad = returns.copy()
    bad[7, 1] = np.nan
    res, max_x, max_y, nx, ny = grids[1].limits
    steep = np.float32([[max_x - 0.1, origin[1], 40.0]])   # the 2D band leaves the 3D growth
    leaving = _leaving_return(grids[1].limits, origin)      # ... by less than a cell
    for ret in (bad, np.float32([[1.0e4, 0, 0]]), steep, leaving):
        assert lib.csm_tsdf_inserter2d_insert(ins, p(origin), p(ret), len(ret), grids[0]._h,
                                              None) == 1
    assert lib.csm_tsdf_inserter2d_insert(ins, None, p(returns), len(returns), grids[0]._h,
                                          None) == 1
    assert lib.csm_tsdf_inserter2d_insert(ins, p(origin), None, 3, grids[0]._h, None) == 1
    for ret in (steep, leaving):   # the restatement refuses them too
        assert not pair[1].insert(origin, ret, grids[1])
    pg = sm.RealTimeGrid2D.empty(res, max_x, max_y, nx, ny)
    assert lib.csm_tsdf_inserter2d_insert(ins, p(origin), p(returns), len(returns), pg._h,
                                          None) == 1
    pg.close()
    after = grids[0].read()
    np.testing.assert_array_equal(after.cells, before.cells)
    np.testing.assert_array_equal(after.weight_cells, before.weight_cells)
    assert (after.resolution, after.max_x, after.max_y, after.known_cells_box) == \
        (before.resolution, before.max_x, before.max_y, before.known_cells_box)
    assert _insert(pair, grids, origin, returns)   # still usable
    assert_grid_equal(*grids)
    # a growing insert refused on the device keeps the old limits and arrays
    far = np.float32([[origin[0] + 12.0, origin[1] + 0.5, 0]])
    probe = O.TsdfGrid(*grids[1].limits, 0.3, 10.0)
    assert pair[1].insert(origin, far, probe)
    assert probe.limits[3] > nx
    grown = np.concatenate([returns, far, _leaving_return(probe.limits, origin)])
    before = grids[0].read()
    assert not _insert(pair, grids, origin, grown)
    after = grids[0].read()
    assert after.cells.shape == before.cells.shape and after.max_x == before.max_x
    np.testing.assert_array_equal(after.cells, before.cells)
    np.testing.assert_array_equal(after.weight_cells, before.weight_cells)


def test_a_marked_cell_on_a_ray_is_refused(sm):
    tsdf, _ = synthetic.make_tsdf2d(4, size_cells=120)
    tsd = tsdf.tsd_cells.copy()
    weight = tsdf.weight_cells.copy()
    ny, nx = tsd.shape
    origin = np.float32([tsdf.max_x - 0.5 * ny * tsdf.resolution,
                         tsdf.max_y - 0.5 * nx * tsdf.resolution, 0])
    ret = np.float32([[origin[0] + 1.0, origin[1] + 0.02, 0]])
    cx, cy = (int(v) for v in O.TsdfGrid(tsdf.resolution, tsdf.max_x, tsdf.max_y, nx, ny, 0.3,
                                         10.0).cell_index(ret[0, 0], ret[0, 1]))
    tsd[cy, cx] = 20000 | 0x8000
    dev = sm.RealTimeGrid2D(sm.TSDF2DSpec(tsd, weight, tsdf.resolution, tsdf.max_x, tsdf.max_y,
                                          0.3, 10.0))
    ins = sm.TSDFRangeDataInserter2D()
    from cartographer_b200._lib import CsmError
    with pytest.raises(CsmError):
        ins.Insert(origin, ret, dev)
    st = dev.read()
    np.testing.assert_array_equal(st.cells, tsd)
    np.testing.assert_array_equal(st.weight_cells, weight)


# ---- readers of an inserted handle ----
def test_matchers_read_an_inserted_handle_as_restated_cells(sm, world):
    spec, occ, poses = world
    pair = _pair(sm)
    dev, ora = grids = _empty(sm, poses[0][:2])
    for k in range(20):
        origin, returns = _world_scan(occ, spec, poses[k % 3] + np.array([0.02 * k, 0, 0]),
                                      seed=100 + k)
        assert _insert(pair, grids, origin, returns)
    st = assert_grid_equal(*grids)
    tsd, weight = ora.arrays()
    twin = sm.RealTimeGrid2D(sm.TSDF2DSpec(tsd, weight, st.resolution, st.max_x, st.max_y, 0.3,
                                           10.0))
    rt = sm.RealTimeCorrelativeScanMatcher2D(
        sm.RealTimeCorrelativeScanMatcherOptions(0.1, 0.12, 0.1, 0.1))
    scans = [synthetic.cast_scan(occ, spec, poses[k], beams=361, max_range=8.0, seed=7 + k)
             for k in range(3)]
    inits = [poses[k] + np.array([0.03, -0.04, 0.02]) for k in range(3)]
    s1, p1, _ = rt.MatchBatch(inits, scans, dev)
    s2, p2, _ = rt.MatchBatch(inits, scans, twin)
    np.testing.assert_array_equal(s1, s2)
    np.testing.assert_array_equal(p1, p2)
    cm = sm.CeresScanMatcher2D()
    for k in range(3):
        c1, st1 = cm.Match(p1[k][:2], p1[k], scans[k], dev)
        c2, st2 = cm.Match(p1[k][:2], p1[k], scans[k], twin)
        np.testing.assert_array_equal(c1, c2)
        assert st1["iterations"] == st2["iterations"]
    twin.close()
