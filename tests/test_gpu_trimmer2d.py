"""OverlappingSubmapsTrimmer2D's coverage pass on device grids (csm_trim_overlapping_submaps2d):
trim flags and per-submap covered-entry counts equal the CPU restatement's
(tests/trimmer2d_oracle.cc), bit for bit, and the handles are left unchanged."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import bench_trimmer2d as B
from benchmarks import synthetic
from tests import trimmer2d_cases as K
from tests import trimmer2d_oracle as O

pytestmark = pytest.mark.gpu

IDENT = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


@pytest.fixture(scope="module")
def P():
    from cartographer_b200 import pose_graph
    return pose_graph


def _yaw(x, y, yaw):
    return [x, y, 0.0, math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)]


def _host(grid):
    st = grid.read()
    return st.cells, st.known_cells_box, (st.max_x, st.max_y, st.resolution)


def _state(grid):
    st = grid.read()
    return st.cells.copy(), st.known_cells_box, st.max_x, st.max_y, st.resolution, (
        None if st.weight_cells is None else st.weight_cells.copy())


def _same_state(a, b):
    assert all(np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y
               for x, y in zip(a, b))


def _compare(P, records, first, fresh, min_cells):
    """Device against restatement; the restatement reads the handles after the device call, so
    that handles made from cells are walked before their known-cells box is ever computed."""
    trim, counts, st = P.trim_overlapping_submaps2d(records, first, fresh, min_cells)
    subs = [_host(g) + (pose, t) for g, pose, t in records]
    want_trim, want_counts, want = O.trim(subs, first, fresh, min_cells)
    np.testing.assert_array_equal(counts, want_counts)
    np.testing.assert_array_equal(trim, want_trim)
    assert st["entries"] == want["entries"] and st["coverage_cells"] == want["coverage_cells"]
    assert st["host_syncs"] <= 3
    return trim, counts, st


def _from_cells(sm, cells, limits):
    return sm.RealTimeGrid2D(synthetic.GridSpec(cells, limits[2], limits[0], limits[1]))


@pytest.mark.parametrize("name", sorted(K.REFERENCE_CASES))
def test_reference_cases_on_device_handles(sm, P, name):
    b = K.Builder(lambda g: _from_cells(sm, g.cells, g.limits))
    K.REFERENCE_CASES[name](b, P.OverlappingSubmapsTrimmer2D)
    for d in b.pg.submap_data.values():
        d.submap.grid.close()


def _world_scan(occ, spec, pose, seed, beams=541, max_range=6.0):
    pts = synthetic.cast_scan(occ, spec, pose, beams=beams, max_range=max_range, seed=seed)
    c, s = math.cos(pose[2]), math.sin(pose[2])
    w = np.stack([c * pts[:, 0] - s * pts[:, 1] + pose[0], s * pts[:, 0] + c * pts[:, 1] + pose[1],
                  np.zeros(len(pts))], 1).astype(np.float32)
    far = np.hypot(pts[:, 0], pts[:, 1]) >= max_range - 0.05
    return np.float32([pose[0], pose[1], 0]), w[~far], w[far]


@pytest.fixture(scope="module")
def inserted(sm):
    """Submaps made by the device inserters: ProbabilityGrids cropped with csm_rt_grid2d_crop,
    their uncropped originals and TSDF2D grids, with local poses at their scan origins."""
    spec, occ = synthetic.make_grid2d(21, size_cells=600)
    rng = np.random.RandomState(11)
    poses = [synthetic.random_free_pose(occ, spec, rng, margin_cells=40) for _ in range(12)]
    ins = sm.ProbabilityGridRangeDataInserter2D()
    topts = sm.TSDFRangeDataInserterOptions2D()
    tins = sm.TSDFRangeDataInserter2D(topts)
    out = []
    for k in range(6):
        a, b = poses[2 * k], poses[2 * k + 1]
        if k % 3 == 2:
            g = sm.RealTimeGrid2D.empty_tsdf(0.05, a[0] + 2.5, a[1] + 2.5, topts.truncation_distance,
                                             topts.maximum_weight)
            for j, p in enumerate((a, b)):
                origin, returns, _ = _world_scan(occ, spec, p, 300 + 2 * k + j)
                tins.Insert(origin, returns, g)
            out.append((g, _yaw(a[0], a[1], 0.0)))
            continue
        g = sm.RealTimeGrid2D.empty(0.05, a[0] + 2.5, a[1] + 2.5)
        for j, p in enumerate((a, b)):
            origin, returns, misses = _world_scan(occ, spec, p, 100 + 2 * k + j)
            ins.Insert(origin, returns, g, misses)
        crop = g.ComputeCroppedGrid()
        out.append((crop, _yaw(a[0], a[1], 0.0)))
        out.append((g, _yaw(a[0], a[1], 0.0)))
    yield out
    for g, _ in out:
        g.close()
    ins.close()
    tins.close()


@pytest.mark.parametrize("fresh,min_area", [(1, 0.0), (1, 2.0), (2, 1.0), (3, 5.0), (0, 0.0)])
def test_inserted_and_cropped_maps(P, inserted, fresh, min_area):
    rng = np.random.RandomState(fresh * 10 + int(min_area))
    records = []
    for i, (g, local) in enumerate(inserted):
        glob = _yaw(local[0] + rng.uniform(-0.2, 0.2), local[1] + rng.uniform(-0.2, 0.2),
                    rng.uniform(-0.3, 0.3))
        records.append((g, P.global_frame_from_local_frame(glob, local), 1000 * (i // 2)))
    first = _host(inserted[0][0])[2]
    before = [_state(g) for g, _ in inserted]
    _compare(P, records, first, fresh, P.double_to_uint16(min_area / first[2] ** 2))
    for (g, _), b in zip(inserted, before):
        _same_state(_state(g), b)


def test_small_empty_pitched_and_tsdf_handles(sm, P):
    empty = sm.RealTimeGrid2D.empty(0.05, 1.0, 1.0, 10, 10)
    one = empty.ComputeCroppedGrid()
    single = np.zeros((5, 7), np.uint16)
    single[3, 2] = 12345
    g1 = _from_cells(sm, single, (0.3, 0.2, 0.05))
    crop1 = g1.ComputeCroppedGrid()   # 1 x 1 crop
    rng = np.random.RandomState(4)
    big = np.zeros((130, 261), np.uint16)   # 261 is not a multiple of 8: a pitched handle
    big[1:129, 3:259] = np.where(rng.rand(128, 256) < 0.7, rng.randint(1, 32768, (128, 256)), 0)
    pitched = _from_cells(sm, big, (3.0, 2.0, 0.05))
    tsd = np.where(rng.rand(60, 70) < 0.5, rng.randint(1, 32768, (60, 70)), 0).astype(np.uint16)
    wgt = np.where(tsd > 0, 100, 0).astype(np.uint16)
    tsdf = sm.RealTimeGrid2D(sm.TSDF2DSpec(tsd, wgt, 0.05, 2.0, 1.5, 0.3, 10.0))
    handles = [pitched, empty, one, g1, crop1, tsdf]
    records = [(h, _yaw(0.1 * i, -0.05 * i, 0.2 * i), 50 - i) for i, h in enumerate(handles)]
    first = (3.0, 2.0, 0.05)
    for fresh, min_cells in ((1, 0), (2, 3), (4, 100)):
        trim, counts, _ = _compare(P, records, first, fresh, min_cells)
        assert trim[1] and counts[1] == 0   # all unknown: no entry, trimmed even at min 0
    for h in handles:
        h.close()


def _stack(sm, times, corner=(0.5, 0.5)):
    """One-cell submaps on one global cell, in list order, with the given freshness."""
    grids = [_from_cells(sm, np.ones((1, 1), np.uint16), (corner[0], corner[1], 1.0))
             for _ in times]
    return grids, [(g, IDENT, t) for g, t in zip(grids, times)]


def test_ties_across_the_cut_take_the_device_and_the_host_path(sm, P):
    # 5 entries, fresh 2: T* = 2, one newer entry, one of three tied submaps in list order
    grids, records = _stack(sm, [3, 2, 2, 2, 1])
    trim, counts, st = _compare(P, records, (0.0, 0.0, 1.0), 2, 1)
    assert st["device_tie_cells"] == 1 and st["host_sorted_cells"] == 0 and st["host_syncs"] == 2
    assert list(counts) == [1, 1, 0, 0, 0]
    # 16 entries with a tie across the cut: still insertion sort, on the device
    grids2, records2 = _stack(sm, [5] + [4] * 10 + [1] * 5, corner=(3.5, 3.5))
    _, _, st = _compare(P, records2, (0.0, 0.0, 1.0), 3, 1)
    assert st["device_tie_cells"] == 1 and st["host_sorted_cells"] == 0
    # 17 and 40 entries with ties across the cut: std::sort on the host
    for times, fresh in (([5] + [4] * 10 + [1] * 6, 3), ([1] * 5 + [3] * 30 + [9] * 5, 7)):
        grids3, records3 = _stack(sm, times, corner=(7.5, 7.5))
        _, _, st = _compare(P, records3, (0.0, 0.0, 1.0), fresh, 1)
        assert st["host_sorted_cells"] == 1 and st["host_syncs"] == 3
        for g in grids3:
            g.close()
    # a tie inside one submap across the cut is settled on the device whatever the size
    cells = np.ones((2, 10), np.uint16)   # 20 cells of resolution 0.1 in the global cell (0, 1)
    g = _from_cells(sm, cells, (0.2, 1.0, 0.1))
    newer = _from_cells(sm, np.ones((1, 1), np.uint16), (1.0, 1.5, 1.0))   # the same cell
    _, counts, st = _compare(P, [(g, IDENT, 9), (newer, IDENT, 10)], (0.5, 1.5, 1.0), 5, 1)
    assert st["coverage_cells"] == 1 and list(counts) == [4, 1]
    assert st["host_sorted_cells"] == 0 and st["device_tie_cells"] == 0
    for h in grids + grids2 + [g, newer]:
        h.close()


@pytest.mark.parametrize("total,before", [(17, 0), (18, 0), (18, 1), (24, 3), (31, 0), (32, 0),
                                          (32, 3), (33, 1), (64, 3)])
def test_small_calls_with_a_host_sorted_cell(sm, P, total, before):
    """Calls of few entries whose one host-sorted cell (17 tied one-cell submaps across the cut)
    lies first, or after `before` single-entry cells in key order, with single-entry cells after
    it up to `total` entries: the cells left to the host have their own workspace, so the sorted
    keys and positions the cut reads stay intact (every cell is found once, every count right),
    and a second call gives the same."""
    after = total - 17 - before
    grids, records = _stack(sm, [5] + [4] * 10 + [1] * 6)   # key x 0
    # one-cell submaps at corner x c put their cell at key x lround(-(c - 0.5)): smaller keys
    # (before the stack in sort order) for c > 0.5, larger ones for c < 0.5
    for k in range(before):
        g, = _stack(sm, [7], corner=(3.5 + 2 * k, 0.5))[0]
        grids.append(g)
        records.insert(0, (g, IDENT, 7))
    for k in range(after):
        g, = _stack(sm, [2], corner=(-2.5 - 2 * k, 0.5))[0]
        grids.append(g)
        records.append((g, IDENT, 2))
    first = _compare(P, records, (0.0, 0.0, 1.0), 3, 1)
    trim, counts, st = first
    assert st["entries"] == total and st["coverage_cells"] == 1 + before + after
    assert st["host_sorted_cells"] == 1 and st["host_syncs"] == 3
    assert int(counts.sum()) == 3 + before + after
    again = P.trim_overlapping_submaps2d(records, (0.0, 0.0, 1.0), 3, 1)
    np.testing.assert_array_equal(again[0], trim)
    np.testing.assert_array_equal(again[1], counts)
    for g in grids:
        g.close()


def test_rotated_submaps_put_duplicates_into_one_cell(sm, P):
    rng = np.random.RandomState(8)
    cells = np.where(rng.rand(80, 90) < 0.8, rng.randint(1, 32768, (80, 90)), 0).astype(np.uint16)
    grids = [_from_cells(sm, cells, (2.0, 2.0, 0.05)) for _ in range(3)]
    records = [(g, _yaw(0.013 * i, -0.021 * i, math.radians(45 + 7 * i)), i)
               for i, g in enumerate(grids)]
    # first resolution 0.05 with 45 degree rotation, and a coarser 0.07 first grid
    for first in ((2.0, 2.0, 0.05), (1.7, 2.3, 0.07)):
        _, _, st = _compare(P, records, first, 2, 10)
        assert st["entries"] > st["coverage_cells"]
    for g in grids:
        g.close()


@pytest.mark.parametrize("minimum,trimmed", [(0, False), (1, True)])
def test_65536_covered_cells(sm, P, minimum, trimmed):
    g = _from_cells(sm, np.ones((256, 256), np.uint16), (0.0, 0.0, 1.0))
    trim, counts, _ = _compare(P, [(g, IDENT, 1)], (0.0, 0.0, 1.0), 1, minimum)
    assert counts[0] == 65536 and trim[0] == trimmed
    g.close()


def test_refusals_leave_handles_unchanged(sm, P):
    from cartographer_b200._lib import CsmError
    cells = np.ones((4, 4), np.uint16)
    g = _from_cells(sm, cells, (1.0, 1.0, 0.1))
    before = _state(g)
    with pytest.raises(CsmError) as e:   # a key past int32
        P.trim_overlapping_submaps2d([(g, [3e9, 0, 0, 1, 0, 0, 0], 1)], (0.0, 0.0, 0.1), 1, 0)
    assert e.value.status == 3
    _same_state(_state(g), before)
    recs = (P.CsmCoverageSubmap2D * 2)()
    recs[0].grid = g._h
    recs[0].rotation[0] = recs[1].rotation[0] = 1.0
    trim = np.full(2, 7, np.uint8)
    counts = np.full(2, 7, np.uint32)
    st = P.lib().csm_trim_overlapping_submaps2d(
        recs, 2, C.c_double(0), C.c_double(0), C.c_double(0.1), C.c_uint16(1), C.c_uint16(0),
        trim.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), None)
    assert st == 1 and np.all(trim == 7) and np.all(counts == 7)   # a null handle
    recs[1].grid = g._h
    recs[1].translation[0] = math.nan
    st = P.lib().csm_trim_overlapping_submaps2d(
        recs, 2, C.c_double(0), C.c_double(0), C.c_double(0.1), C.c_uint16(1), C.c_uint16(0),
        trim.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p), None)
    assert st == 1 and np.all(trim == 7)
    if sm.device_count() >= 2:
        g1 = sm.RealTimeGrid2D(synthetic.GridSpec(cells, 0.1, 1.0, 1.0), device=1)
        with pytest.raises(CsmError) as e:
            P.trim_overlapping_submaps2d([(g, IDENT, 1), (g1, IDENT, 2)], (0.0, 0.0, 0.1), 1, 0)
        assert e.value.status == 1
        g1.close()
    _same_state(_state(g), before)
    g.close()


def test_benchmark_size_map(sm, P):
    m = B.lifelong_map(1000, seed=1)
    grids = [_from_cells(sm, c, lim) for c, lim, _, _, _ in m]
    records = [(g, P.global_frame_from_local_frame(glob, loc), t)
               for g, (_, _, glob, loc, t) in zip(grids, m)]
    first = m[0][1]
    trim, counts, st = _compare(P, records, first, 3, P.double_to_uint16(10.0 / first[2] ** 2))
    assert st["entries"] > 50_000_000 and 0 < trim.sum() < len(trim)
    for g in grids:
        g.close()
