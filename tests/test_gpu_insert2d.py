"""ProbabilityGridRangeDataInserter2D, grid growth and submap cropping on the device
(csrc/insert2d.cu) against the CPU restatement in tests/insert2d_oracle.cc: every cell, the
limits and the known-cells box bit for bit after every insert; the matchers and the
precomputation stack on inserted and cropped handles against the same on restated cells."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import insert2d_oracle as O

pytestmark = pytest.mark.gpu

REF_RETURNS = np.array([[-3.5, 0.5, 0], [-2.5, 1.5, 0], [-1.5, 2.5, 0], [-0.5, 3.5, 0]],
                       np.float32)   # range_data_inserter_2d_test.cc:48-55


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _pair(sm, hit=0.55, miss=0.49, free_space=True):
    opts = sm.ProbabilityGridRangeDataInserterOptions2D(hit, miss, free_space)
    return sm.ProbabilityGridRangeDataInserter2D(opts), O.Inserter(hit, miss, free_space)


def _empty(sm, origin, resolution=0.05):
    """ActiveSubmaps2D::CreateGrid on both sides."""
    ora = O.Grid.create_grid(origin, resolution)
    res, max_x, max_y, nx, ny = ora.limits
    return sm.RealTimeGrid2D.empty(res, max_x, max_y, nx, ny), ora


def _from_cells(sm, spec):
    ora = O.Grid(spec.resolution, spec.max_x, spec.max_y, spec.cells.shape[1],
                 spec.cells.shape[0], spec.cells)
    return sm.RealTimeGrid2D(spec), ora


def assert_grid_equal(dev, ora):
    st = dev.read()
    res, max_x, max_y, nx, ny = ora.limits
    assert (st.resolution, st.max_x, st.max_y) == (res, max_x, max_y)
    assert st.cells.shape == (ny, nx) and dev.shape == (ny, nx)
    np.testing.assert_array_equal(st.cells, ora.cells)
    assert st.known_cells_box == ora.known_box
    return st


def _insert(pair, grids, origin, returns, misses=None):
    dev_ins, ora_ins = pair
    dev, ora = grids
    dev_ins.Insert(origin, returns, dev, misses)
    ora_ins.insert(origin, returns, ora, misses)
    assert dev_ins.last_stats["host_syncs"] == 1


def _world_scan(occ, spec, pose, seed, beams=1081, max_range=8.0):
    """A scan cast in the synthetic world, in the world frame: returns short of max_range,
    and the beams that reached it as misses (as LocalTrajectoryBuilder2D turns them)."""
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
    poses = [synthetic.random_free_pose(occ, spec, rng, margin_cells=40) for _ in range(50)]
    return spec, occ, poses


# ---- the reference's cases ----
def test_insert_point_cloud(sm):
    pair = _pair(sm, 0.7, 0.4)
    grids = (sm.RealTimeGrid2D(synthetic.GridSpec(np.zeros((5, 5), np.uint16), 1.0, 1.0, 5.0)),
             O.Grid(1.0, 1.0, 5.0, 5, 5))
    _insert(pair, grids, [-0.5, 0.5, 0], REF_RETURNS)
    st = assert_grid_equal(*grids)
    assert st.cells.shape == (5, 5) and (st.max_x, st.max_y) == (1.0, 5.0)
    U, M, H = 0, 1, 2
    expected = [[U, U, U, U, U], [U, H, M, M, M], [U, U, H, M, M], [U, U, U, H, M],
                [U, U, U, U, H]]
    for row in range(5):
        for column in range(5):
            v = int(st.cells[column, row])
            if expected[column][row] == U:
                assert v == 0
            else:
                want = 0.4 if expected[column][row] == M else 0.7
                assert abs(grids[1].get_probability(row, column) - want) < 1e-4 and v != 0


def test_probability_progression(sm):
    pair = _pair(sm, 0.7, 0.4)
    grids = _empty(sm, [-2.0, 2.0], 1.0)
    for _ in range(1001):
        _insert(pair, grids, [-0.5, 0.5, 0], REF_RETURNS)
    assert_grid_equal(*grids)
    ora = grids[1]
    assert abs(ora.get_probability(*ora.cell_index(-3.5, 0.5)) - 0.9) < 1e-3
    assert abs(ora.get_probability(*ora.cell_index(-2.5, 0.5)) - 0.1) < 1e-3


# ---- seeded local-SLAM sequences ----
@pytest.mark.parametrize("start", ["empty", "cells"])
def test_fifty_seeded_inserts(sm, world, start):
    spec, occ, poses = world
    pair = _pair(sm)
    if start == "empty":
        grids = _empty(sm, poses[0][:2])
    else:
        sub, _ = synthetic.crop_grid(spec, occ, 200, 200, 160, 120)
        grids = _from_cells(sm, sub)
    for k, pose in enumerate(poses):
        origin, returns, misses = _world_scan(occ, spec, pose, seed=k)
        _insert(pair, grids, origin, returns, misses)
        assert_grid_equal(*grids)


# ---- edges ----
def test_several_doublings_and_growth_on_each_side(sm):
    pair = _pair(sm)
    grids = _empty(sm, [0.0, 0.0])
    _insert(pair, grids, [0, 0, 0], np.float32([[0.3, 0.2, 0]]))
    for far in ([-20.0, 0.1], [0.2, 25.0], [31.0, -0.3], [0.4, -33.0]):
        _insert(pair, grids, [0, 0, 0], np.float32([far + [0.0]]))
        assert_grid_equal(*grids)
    assert grids[0].shape[0] >= 800   # several doublings in one insert


@pytest.mark.parametrize("free_space", [False, True])
def test_misses_only_and_no_free_space(sm, world, free_space):
    spec, occ, poses = world
    pair = _pair(sm, 0.6, 0.45, free_space)
    grids = _empty(sm, poses[1][:2])
    origin, returns, misses = _world_scan(occ, spec, poses[1], seed=1)
    _insert(pair, grids, origin, np.zeros((0, 3), np.float32), misses)   # misses only
    assert_grid_equal(*grids)
    _insert(pair, grids, origin, returns, misses)
    assert_grid_equal(*grids)
    _insert(pair, grids, origin + np.float32([0.5, 0, 0]), np.zeros((0, 3), np.float32))  # origin only
    assert_grid_equal(*grids)


def test_special_rays(sm):
    """Rays inside the origin's pixel, vertical and horizontal rays, exact corner crossings
    and returns on cell borders."""
    pair = _pair(sm, 0.7, 0.4)
    r = 0.05
    grids = _empty(sm, [0.0, 0.0], r)
    _, max_x, max_y, _, _ = grids[1].limits
    # cell borders: max - k * resolution in float
    border = lambda k: float(np.float32(max_x - k * r))  # noqa: E731
    o = np.float32([border(50), border(50), 0])       # the origin on a cell corner
    pts = [[o[0] + 0.01, o[1] + 0.01], [o[0] - 0.004, o[1]],                # own pixel
           [o[0], o[1] + 1.0], [o[0], o[1] - 1.3], [o[0] + 0.8, o[1]], [o[0] - 0.9, o[1]],
           [o[0] + 0.5, o[1] + 0.5], [o[0] - 0.5, o[1] + 0.5], [o[0] + 0.75, o[1] - 0.75],
           [o[0] + 0.5, o[1] + 1.0], [o[0] - 1.0, o[1] - 0.5],
           [border(30), border(62)], [border(71), border(40)], [border(44), border(44)]]
    ret = np.float32([[x, y, 0] for x, y in pts])
    _insert(pair, grids, o, ret, ret[::-1] * np.float32([1.01, 0.99, 0]))
    assert_grid_equal(*grids)
    # the same from a pixel centre
    _insert(pair, grids, o + np.float32([r / 2, r / 2, 0]), ret)
    assert_grid_equal(*grids)


def test_refused_calls_leave_the_handle_unchanged(sm, world):
    spec, occ, poses = world
    pair = _pair(sm)
    grids = _empty(sm, poses[2][:2])
    origin, returns, misses = _world_scan(occ, spec, poses[2], seed=2)
    _insert(pair, grids, origin, returns, misses)
    before = grids[0].read()
    lib = sm.lib()
    ins = pair[0]._h
    bad = returns.copy()
    bad[7, 1] = np.nan
    far = np.float32([[1.0e4, 0, 0]])   # past the 30000-cell guard
    o = np.ascontiguousarray(origin)
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    for ret in (bad, far):
        ret = np.ascontiguousarray(ret)
        assert lib.csm_range_inserter2d_insert(ins, p(o), p(ret), len(ret), None, 0,
                                               grids[0]._h, None) == 1
    assert lib.csm_range_inserter2d_insert(ins, None, p(returns), len(returns), None, 0,
                                           grids[0]._h, None) == 1
    assert lib.csm_range_inserter2d_insert(ins, p(o), None, 3, None, 0, grids[0]._h, None) == 1
    tsdf, _ = synthetic.make_tsdf2d(3, size_cells=64)
    tg = sm.RealTimeGrid2D(tsdf)
    assert lib.csm_range_inserter2d_insert(ins, p(o), p(returns), len(returns), None, 0,
                                           tg._h, None) == 1
    out = C.c_void_p()
    assert lib.csm_rt_grid2d_crop(tg._h, C.byref(out)) == 1
    assert lib.csm_stack2d_create_from_rt_grid2d(tg._h, 7, C.byref(out)) == 1
    tg.close()
    after = grids[0].read()
    np.testing.assert_array_equal(after.cells, before.cells)
    assert (after.resolution, after.max_x, after.max_y, after.known_cells_box) == \
        (before.resolution, before.max_x, before.max_y, before.known_cells_box)
    _insert(pair, grids, origin, returns, misses)   # still usable
    assert_grid_equal(*grids)


# ---- readers of an inserted handle ----
def _submap(sm, world, scans=20):
    spec, occ, poses = world
    pair = _pair(sm)
    grids = _empty(sm, poses[0][:2])
    for k in range(scans):
        origin, returns, misses = _world_scan(occ, spec, poses[k % 3] + np.array([0.02 * k, 0, 0]),
                                              seed=100 + k)
        _insert(pair, grids, origin, returns, misses)
    assert_grid_equal(*grids)
    return grids


def test_matchers_read_an_inserted_handle_as_restated_cells(sm, world):
    spec, occ, poses = world
    dev, ora = _submap(sm, world)
    res, max_x, max_y, nx, ny = ora.limits
    twin = sm.RealTimeGrid2D(synthetic.GridSpec(ora.cells, res, max_x, max_y))
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


def test_crop_and_stack_from_the_handle(sm, world):
    spec, occ, poses = world
    dev, ora = _submap(sm, world)
    crop_dev, crop_ora = dev.ComputeCroppedGrid(), ora.crop()
    st = assert_grid_equal(crop_dev, crop_ora)
    opts = sm.FastCorrelativeScanMatcherOptions2D(3.0, 0.5, 7)
    m_dev = sm.FastCorrelativeScanMatcher2D.from_device_grid(crop_dev, opts)
    m_host = sm.FastCorrelativeScanMatcher2D(synthetic.GridSpec(crop_ora.cells, st.resolution,
                                                                st.max_x, st.max_y), opts)
    for level in range(7):
        np.testing.assert_array_equal(m_dev.precomputation_grid(level),
                                      m_host.precomputation_grid(level))
    for k in range(3):
        scan = synthetic.cast_scan(occ, spec, poses[k], beams=361, max_range=8.0, seed=50 + k)
        # the scan in the submap frame = the world frame here; MatchFullSubmap searches all of it
        c, s = math.cos(poses[k][2]), math.sin(poses[k][2])
        w = np.stack([c * scan[:, 0] - s * scan[:, 1], s * scan[:, 0] + c * scan[:, 1],
                      np.zeros(len(scan))], 1).astype(np.float32)
        a = m_dev.MatchFullSubmap(w, 0.3)
        b = m_host.MatchFullSubmap(w, 0.3)
        assert a[0] == b[0] and np.float32(a[1]) == np.float32(b[1])
        np.testing.assert_array_equal(a[2], b[2])
    m_dev.close()
    m_host.close()


def test_crop_of_an_empty_handle_is_one_unknown_cell(sm):
    dev, ora = _empty(sm, [1.0, -2.0])
    crop = dev.ComputeCroppedGrid()
    st = assert_grid_equal(crop, ora.crop())
    assert st.cells.shape == (1, 1) and st.known_cells_box is None


def test_crop_of_a_handle_made_from_cells(sm, world):
    spec, occ, _ = world
    sub, _ = synthetic.crop_grid(spec, occ, 100, 150, 90, 70)
    cells = sub.cells.copy()
    cells[:5, :] = 0
    cells[:, -9:] = 0
    dev, ora = _from_cells(sm, synthetic.GridSpec(cells, sub.resolution, sub.max_x, sub.max_y))
    assert_grid_equal(dev, ora)
    assert_grid_equal(dev.ComputeCroppedGrid(), ora.crop())
