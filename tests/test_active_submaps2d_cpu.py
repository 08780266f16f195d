"""ActiveSubmaps2D's host-side rules without a GPU: create_grid_limits against the oracle's
CreateGrid and hand values, the lifecycle restatement (tests/active_submaps2d_oracle.py)
against hand-derived schedules, the slot reservation of csm_range_inserter2d_insert_submaps
against RayToPixelMask's exact lengths, and the new entry point's symbol, declaration and
refusals."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tests import active_submaps2d_oracle as A
from tests import insert2d_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


# ---- CreateGrid's limits ----
@pytest.mark.parametrize("resolution", [0.05, 0.1])
@pytest.mark.parametrize("origin", [(0.0, 0.0), (1.3, -2.7), (-1234.567, 89.01)])
def test_create_grid_limits_equal_the_oracle(resolution, origin):
    from cartographer_b200 import scan_matching as sm
    assert sm.create_grid_limits(origin, resolution) == O.Grid.create_grid(origin, resolution).limits


def test_create_grid_limits_hand_values():
    from cartographer_b200 import scan_matching as sm
    # the float option 0.05 is 0.05000000074505806 in double; 50 cells of it
    r = 0.05000000074505806
    assert sm.create_grid_limits((0.0, 0.0), 0.05) == (r, 50 * r, 50 * r, 100, 100)
    # the float origin 1.3 is 1.2999999523162842
    res, max_x, max_y, nx, ny = sm.create_grid_limits((1.3, -2.7), 0.1)
    assert res == 0.10000000149011612 and (nx, ny) == (100, 100)
    assert max_x == 1.2999999523162842 + 50 * res
    assert max_y == -2.700000047683716 + 50 * res


# ---- the lifecycle ----
def _schedule(num_range_data, scans):
    active = A.ActiveSubmaps(num_range_data, grids=False)
    return [active.insert_range_data((0.1 * k, 0.0, 0.0)) for k in range(scans)], active


def test_schedule_num_range_data_1():
    events, _ = _schedule(1, 4)
    assert [(e["created"], e["evicted"], e["finished"], e["inserted"]) for e in events] == [
        (0, None, None, [0]),
        (1, None, 0, [0, 1]),
        (2, 0, 1, [1, 2]),
        (3, 1, 2, [2, 3])]


def test_schedule_num_range_data_2():
    events, active = _schedule(2, 7)
    assert [(e["created"], e["evicted"], e["finished"], e["inserted"]) for e in events] == [
        (0, None, None, [0]),
        (None, None, None, [0]),
        (1, None, None, [0, 1]),
        (None, None, 0, [0, 1]),      # submap 0 holds 4 = 2 * 2 scans
        (2, 0, None, [1, 2]),
        (None, None, 1, [1, 2]),
        (3, 1, None, [2, 3])]
    assert [(s.index, s.num_range_data, s.insertion_finished) for s in active.submaps] == \
        [(2, 3, False), (3, 1, False)]


def test_schedule_num_range_data_3():
    events, active = _schedule(3, 10)
    created = [k for k, e in enumerate(events) if e["created"] is not None]
    finished = {e["finished"]: k for k, e in enumerate(events) if e["finished"] is not None}
    evicted = {e["evicted"]: k for k, e in enumerate(events) if e["evicted"] is not None}
    assert created == [0, 3, 6, 9]
    assert finished == {0: 5, 1: 8}
    assert evicted == {0: 6, 1: 9}
    # each submap's local pose is the float origin of the scan that created it
    assert [s.local_pose for s in active.submaps] == [
        (float(F(0.6)), 0.0, 0.0, 1.0, 0.0, 0.0, 0.0), (float(F(0.9)), 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)]
    assert [s.num_range_data for s in active.submaps] == [4, 1]


def test_python_and_oracle_refuse_the_same_options():
    from cartographer_b200 import scan_matching as sm
    with pytest.raises(AssertionError):
        A.ActiveSubmaps(0, grids=False)
    for bad in (sm.SubmapsOptions2D(num_range_data=0), sm.SubmapsOptions2D(grid_type="TSDF"),
                sm.SubmapsOptions2D(range_data_inserter_type="TSDF_INSERTER_2D")):
        with pytest.raises(ValueError):
            sm.ActiveSubmaps2D(bad)
    o = sm.SubmapsOptions2D()
    assert (o.num_range_data, o.resolution, o.grid_type) == (90, 0.05, "PROBABILITY_GRID")
    p = o.probability_grid_range_data_inserter_options
    assert (p.hit_probability, p.miss_probability, p.insert_free_space) == (0.55, 0.49, True)


# ---- the slot reservation is never short ----
def _mask_lengths(limits, origin, points):
    b = A.superscaled_index(limits, origin[0], origin[1])
    out = []
    for p in points:
        e = A.superscaled_index(limits, p[0], p[1])
        out.append(len(O.ray_to_pixel_mask(b, e, A.SUBPIXEL_SCALE)))
    return out


def _check_bound(limits, origin, points):
    res = limits[0]
    lengths = _mask_lengths(limits, origin, points)
    o = np.asarray(origin, np.float32).astype(np.float64)
    for p, k in zip(np.asarray(points, np.float32).astype(np.float64), lengths):
        # each ray below its L1 length in cells + 3, up to the double rounding on cell borders
        assert k <= (abs(p[0] - o[0]) + abs(p[1] - o[1])) / res + 3 + 1e-6
    assert sum(lengths) <= A.slot_reservation(origin, points, res)
    return lengths


@pytest.mark.parametrize("seed", range(4))
def test_slot_bound_random_rays(seed):
    rng = np.random.RandomState(seed)
    res = float(F([0.05, 0.1, 0.025, 0.5][seed]))
    limits = (res, 40.0, 40.0)   # every point inside the grid
    origin = np.float32([rng.uniform(-3, 3), rng.uniform(-3, 3), 0])
    pts = np.zeros((400, 3), F)
    pts[:, :2] = origin[:2] + rng.uniform(-8, 8, (400, 2)).astype(F)
    _check_bound(limits, origin, pts)


@pytest.mark.parametrize("res", [0.05, 0.1, 1.0])
def test_slot_bound_adversarial_rays(res):
    res = float(F(res))
    max_x, max_y = 50 * res, 50 * res
    limits = (res, max_x, max_y)
    # cell borders in float; k = 0 is the max edge, where the last float below max is inside
    edge = float(np.nextafter(F(max_x), F(-np.inf)))
    border = lambda k: float(F(max_x - k * res)) if k else edge  # noqa: E731
    half = lambda k: float(F(max_x - (k + 0.5) * res))  # noqa: E731  cell centres
    o = (border(50), border(50), 0.0)   # the origin on a cell corner
    pts = []
    for kx, ky in [(30, 62), (71, 40), (44, 44), (50, 80), (80, 50), (20, 20), (99, 99), (0, 0),
                   (0, 99), (99, 0), (1, 1), (50, 50), (49, 51)]:
        pts.append((border(kx), border(ky), 0.0))    # exact corners and the max edge
        pts.append((half(kx), half(ky), 0.0))        # cell centres
    for d in (0.0, 1e-7, -1e-7, 0.5 * res, -0.5 * res, 0.49999 * res):
        pts.append((o[0] + d, o[1], 0.0))            # zero length, axis-parallel, ± half cells
        pts.append((o[0], o[1] + d + 3 * res, 0.0))
        pts.append((o[0] + 7 * res + d, o[1] + 7 * res - d, 0.0))   # diagonal through corners
    lengths = _check_bound(limits, o, pts)
    assert max(lengths) > 50 and min(lengths) == 1
    # from a cell centre, and from the max edge
    _check_bound(limits, (half(50), half(50), 0.0), pts)
    _check_bound(limits, (border(0), border(0), 0.0), pts[:20])


# ---- the entry point ----
def test_symbol_and_declaration():
    from cartographer_b200._lib import SO_PATH
    syms = subprocess.run(["nm", "-D", "--defined-only", SO_PATH], capture_output=True,
                          text=True, check=True).stdout
    assert re.search(r"\bcsm_range_inserter2d_insert_submaps\b", syms)
    header = open(os.path.join(ROOT, "include", "csm_abi.h")).read()
    decl = re.search(r"csm_status csm_range_inserter2d_insert_submaps\((.*?)\);", header, re.S)
    args = [re.sub(r"/\*.*?\*/", "", a).split()[-1].lstrip("*") for a in decl.group(1).split(",")]
    assert args == ["inserter", "origin[3]", "returns", "num_returns", "misses", "num_misses",
                    "grids", "num_grids", "stats"]
    assert "csm_rt_grid2d* const* grids" in decl.group(1)


def test_refusals_without_a_device():
    from cartographer_b200._lib import lib
    L = lib()
    org = np.zeros(3, F)
    pts = np.zeros((1, 3), F)
    op, pp = org.ctypes.data_as(C.c_void_p), pts.ctypes.data_as(C.c_void_p)
    grids = (C.c_void_p * 2)(8, 16)
    f = L.csm_range_inserter2d_insert_submaps
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                  C.c_void_p, C.c_int32, C.c_void_p]
    assert f(None, op, pp, 1, None, 0, grids, 2, None) == 1        # null inserter
    assert f(8, None, pp, 1, None, 0, grids, 2, None) == 1         # null origin
    assert f(8, op, pp, 1, None, 0, None, 2, None) == 1            # null list
    assert f(8, op, pp, 1, None, 0, grids, 0, None) == 1           # no grids
    assert f(8, op, pp, 1, None, 0, grids, -1, None) == 1
    assert f(8, op, pp, 1, None, 0, grids, 65536, None) == 1
    assert f(8, op, None, 1, None, 0, grids, 2, None) == 1         # returns missing
    assert f(8, op, pp, -1, None, 0, grids, 2, None) == 1
    assert f(8, op, pp, 1, None, 2, grids, 2, None) == 1           # misses missing
    assert f(8, op, pp, 1, None, 0, (C.c_void_p * 2)(8, None), 2, None) == 1   # null entry
    assert f(8, op, pp, 1, None, 0, (C.c_void_p * 3)(8, 16, 8), 3, None) == 1  # a duplicate
