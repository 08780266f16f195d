"""The CPU restatement of ProbabilityGridRangeDataInserter2D (tests/insert2d_oracle.cc) against
the reference's known answers (ray_to_pixel_mask_test.cc, range_data_inserter_2d_test.cc,
probability_grid_test.cc), an independent C++ build of its tables and the numpy RayToPixelMask
of tests/tsdf_inserter.py; the 2D inserter's C ABI records and status codes without a device."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import insert2d_oracle as O
from tests import tsdf_inserter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lround(v):
    return int(math.copysign(math.floor(abs(v) + 0.5), v))


def _cell_index(resolution, max_xy, px, py):
    """MapLimits::GetCellIndex: the float point in double arithmetic."""
    px, py = float(np.float32(px)), float(np.float32(py))
    return (_lround((max_xy[1] - py) / resolution - 0.5), _lround((max_xy[0] - px) / resolution - 0.5))


# ---- ray_to_pixel_mask_test.cc ----
@pytest.mark.parametrize("begin,end,want", [
    ((1, 1), (1, 1), [(1, 1)]),                                              # SingleCell
    ((1, 1), (3, 1), [(1, 1), (2, 1), (3, 1)]),                              # AxisAlignedX
    ((3, 1), (1, 1), [(1, 1), (2, 1), (3, 1)]),
    ((1, 1), (1, 3), [(1, 1), (1, 2), (1, 3)]),                              # AxisAlignedY
    ((1, 3), (1, 1), [(1, 1), (1, 2), (1, 3)]),
    ((1, 1), (3, 3), [(1, 1), (2, 2), (3, 3)]),                              # Diagonal
    ((3, 3), (1, 1), [(1, 1), (2, 2), (3, 3)]),
    ((1, 3), (3, 1), [(1, 3), (2, 2), (3, 1)]),
    ((3, 1), (1, 3), [(1, 3), (2, 2), (3, 1)]),
    ((1, 1), (2, 5), [(1, 1), (1, 2), (1, 3), (2, 3), (2, 4), (2, 5)]),      # SteepLine
    ((1, 1), (2, 4), [(1, 1), (1, 2), (2, 3), (2, 4)]),
    ((1, 1), (5, 2), [(1, 1), (2, 1), (3, 1), (3, 2), (4, 2), (5, 2)]),      # FlatLine
    ((1, 1), (4, 2), [(1, 1), (2, 1), (3, 2), (4, 2)]),
])
def test_ray_to_pixel_mask_unit_scale(begin, end, want):
    assert O.ray_to_pixel_mask(begin, end, 1) == want


def test_ray_to_pixel_mask_multi_scale_axis_aligned_x():
    s = 1
    while s < 10000:
        r = 0.1 / s
        b = _cell_index(r, (1.0, 1.0), 0.05, 0.05)
        e = _cell_index(r, (1.0, 1.0), 0.35, 0.05)
        assert O.ray_to_pixel_mask(b, e, s) == [(9, 6), (9, 7), (9, 8), (9, 9)], s
        s *= 2


def test_ray_to_pixel_mask_multi_scale_skewed_line():
    for s, want in ((1, [(8, 7), (8, 8), (9, 8), (9, 9)]),
                    (20, [(8, 7), (8, 8), (8, 9), (9, 9)])):
        r = 0.1 / s
        b = _cell_index(r, (1.0, 1.0), 0.01, 0.09)
        e = _cell_index(r, (1.0, 1.0), 0.21, 0.19)
        assert O.ray_to_pixel_mask(b, e, s) == want


def _seeded_rays(seed, count):
    rng = np.random.RandomState(seed)
    rays = []
    for _ in range(count):
        s = int(rng.choice([1, 2, 3, 10, 1000]))
        span = int(rng.choice([3, 20, 200])) * s
        b = tuple(int(v) for v in rng.randint(0, span, 2))
        e = tuple(int(v) for v in rng.randint(0, span, 2))
        rays.append((b, e, s))
    # exact corner crossings: pixel centres along diagonals and along 1:2 / 2:1 slopes, and
    # points on pixel borders
    for _ in range(count // 4):
        s = int(rng.choice([2, 10, 1000]))
        px, py = (int(v) for v in rng.randint(0, 40, 2))
        k = int(rng.randint(1, 12))
        sx, sy = (int(v) for v in rng.choice([-1, 1], 2))
        mx, my = [(1, 1), (1, 2), (2, 1), (3, 1)][rng.randint(4)]
        ex, ey = px + sx * k * mx, py + sy * k * my
        if ex < 0 or ey < 0:
            continue
        off = s // 2 if rng.randint(2) else 0
        rays.append(((px * s + off, py * s + off), (ex * s + off, ey * s + off), s))
    return rays


def test_masks_equal_the_numpy_restatement_and_stay_within_their_bound():
    corners = 0
    for b, e, s in _seeded_rays(3, 4000):
        got = O.ray_to_pixel_mask(b, e, s)
        assert got == [tuple(c) for c in tsdf_inserter.ray_to_pixel_mask(b, e, s)], (b, e, s)
        bound = abs(e[0] // s - b[0] // s) + abs(e[1] // s - b[1] // s) + 1
        assert len(got) <= bound, (b, e, s)
        assert got[0] in ((b[0] // s, b[1] // s), (e[0] // s, e[1] // s))
        assert {(b[0] // s, b[1] // s), (e[0] // s, e[1] // s)} <= set(got)
        corners += len(got) < bound
    assert corners > 300   # diagonal steps (exact corners) are well represented


# ---- range_data_inserter_2d_test.cc ----
REF_RETURNS = np.array([[-3.5, 0.5, 0], [-2.5, 1.5, 0], [-1.5, 2.5, 0], [-0.5, 3.5, 0]],
                       np.float32)


def _insert_point_cloud(ins, g):
    ins.insert([-0.5, 0.5, 0.0], REF_RETURNS, g)


def test_insert_point_cloud():
    ins, g = O.Inserter(0.7, 0.4, True), O.Grid(1.0, 1.0, 5.0, 5, 5)
    _insert_point_cloud(ins, g)
    assert g.limits == (1.0, 1.0, 5.0, 5, 5)
    U, M, H = 0, 1, 2
    expected = [[U, U, U, U, U], [U, H, M, M, M], [U, U, H, M, M], [U, U, U, H, M],
                [U, U, U, U, H]]
    cells = g.cells
    for row in range(5):
        for column in range(5):
            state = expected[column][row]
            if state == U:
                assert cells[column, row] == 0
            else:
                want = 0.4 if state == M else 0.7
                assert abs(g.get_probability(row, column) - want) < 1e-4


def test_probability_progression():
    ins, g = O.Inserter(0.7, 0.4, True), O.Grid(1.0, 1.0, 5.0, 5, 5)
    _insert_point_cloud(ins, g)
    hit, miss = g.cell_index(-3.5, 0.5), g.cell_index(-2.5, 0.5)
    assert abs(g.get_probability(*hit) - 0.7) < 1e-4
    assert abs(g.get_probability(*miss) - 0.4) < 1e-4
    for _ in range(1000):
        _insert_point_cloud(ins, g)
    assert abs(g.get_probability(*hit) - 0.9) < 1e-3
    assert abs(g.get_probability(*miss) - 0.1) < 1e-3


# ---- probability_grid_test.cc ----
def test_apply_odds():
    g = O.Grid(1.0, 1.0, 1.0, 2, 2)
    assert (g.cells == 0).all()
    g.set_probability(1, 0, 0.5)
    g.apply_odds(1, 0, 0.9 / 0.1)
    g.finish_update()
    assert g.get_probability(1, 0) > 0.5
    g.set_probability(0, 1, 0.5)
    g.apply_odds(0, 1, np.float32(0.1) / (np.float32(1) - np.float32(0.1)))
    g.finish_update()
    assert g.get_probability(0, 1) < 0.5
    odds = lambda p: float(np.float32(p) / (np.float32(1) - np.float32(p)))  # noqa: E731
    assert g.apply_odds(1, 1, odds(0.42))
    assert abs(g.get_probability(1, 1) - 0.42) < 1e-4
    assert not g.apply_odds(1, 1, odds(0.9))     # ignored until FinishUpdate
    assert abs(g.get_probability(1, 1) - 0.42) < 1e-4
    g.finish_update()
    g.apply_odds(1, 1, odds(0.9))
    assert g.get_probability(1, 1) > 0.42


def test_correct_cropping():
    rng = np.random.RandomState(42)
    g = O.Grid(0.05, 10.0, 10.0, 400, 400)
    for y in range(100, 300):
        for x in range(100, 300):
            g.set_probability(x, y, rng.uniform(0.1, 0.9))
    assert g.known_box == (100, 100, 299, 299)
    c = g.crop()
    res, max_x, max_y, nx, ny = c.limits
    assert (nx, ny) == (200, 200)
    assert max_x == 10.0 - 0.05 * 100 and max_y == 10.0 - 0.05 * 100
    table = O.crop_table()
    np.testing.assert_array_equal(c.cells, table[g.cells[100:300, 100:300]])
    assert c.known_box == (0, 0, 199, 199)


def test_empty_grid_crops_to_one_unknown_cell():
    c = O.Grid(0.05, 1.0, 1.0, 10, 10).crop()
    assert c.limits == (0.05, 1.0, 1.0, 1, 1)
    assert c.known_box is None and c.cells.tolist() == [[0]]


def test_growth_doubles_around_the_old_block():
    ins, g = O.Inserter(0.55, 0.49, True), O.Grid.create_grid([0.0, 0.0], 0.05)
    ins.insert([0, 0, 0], np.float32([[0.3, 0.2, 0]]), g)
    before, box = g.cells, g.known_box
    ins.insert([0, 0, 0], np.float32([[-7.0, 0.1, 0]]), g)   # two doublings: 100 -> 400 cells
    res, max_x, max_y, nx, ny = g.limits
    assert (nx, ny) == (400, 400)
    assert max_x == pytest.approx(2.5 + 0.05 * 50 + 0.05 * 100)
    ox, oy = 50 + 100, 50 + 100
    assert (g.cells[oy:oy + 100, ox:ox + 100][before != 0] != 0).all()
    nb = g.known_box
    assert nb[0] <= box[0] + ox and nb[1] <= box[1] + oy and nb[3] >= box[3] + oy


def test_tables_match_a_cpp_build():
    """ComputeLookupTableToApplyCorrespondenceCostOdds and the crop round trip compiled from
    oracle/oracle_common.h's float helpers."""
    src = r'''
#include <cstdio>
#include "oracle/oracle_common.h"
using namespace oracle;
static float Cost(int v) {
  return SlowValueToBoundedFloat(v, 0, kMaxCorrespondenceCost, kMinCorrespondenceCost,
                                 kMaxCorrespondenceCost);
}
int main() {
  const double probs[4] = {0.7, 0.4, 0.55, 0.49};
  for (double prob : probs) {
    const float odds = Odds(static_cast<float>(prob));
    for (int cell = 0; cell != 32768; ++cell) {
      const float p = cell == 0 ? ProbabilityFromOdds(odds)
          : ProbabilityFromOdds(odds * Odds(CorrespondenceCostToProbability(Cost(cell))));
      std::printf("%d\n", CorrespondenceCostToValue(ProbabilityToCorrespondenceCost(p)) + kUpdateMarker);
    }
  }
  std::printf("0\n");
  for (int v = 1; v != 32768; ++v)
    std::printf("%d\n", CorrespondenceCostToValue(ProbabilityToCorrespondenceCost(
                            CorrespondenceCostToProbability(Cost(v)))));
}
'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.cc"), "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", ROOT,
                               os.path.join(d, "t.cc"), "-o", os.path.join(d, "t")])
        want = np.array(subprocess.check_output([os.path.join(d, "t")]).split(), np.int64)
    got = []
    for hit, miss in ((0.7, 0.4), (0.55, 0.49)):
        h, m = O.Inserter(hit, miss).tables()
        got += [h, m]
    got.append(O.crop_table())
    np.testing.assert_array_equal(np.concatenate(got).astype(np.int64), want)


# ---- the C ABI without a device ----
@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def _layout(ctype, cname):
    head = '#include <stdio.h>\n#include <stddef.h>\n#include "include/csm_abi.h"\nint main(){'
    body = 'printf("%%zu\\n", sizeof(%s));' % cname + "".join(
        'printf("%%zu\\n", offsetof(%s, %s));' % (cname, f) for f, _ in ctype._fields_)
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(head + body + "}")
        subprocess.check_call(["gcc", "-I", ROOT, os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        got = [int(v) for v in subprocess.check_output([os.path.join(d, "t")]).split()]
    assert got == [C.sizeof(ctype)] + [getattr(ctype, f).offset for f, _ in ctype._fields_]


def test_record_layouts(csm):
    from cartographer_b200 import scan_matching as sm
    _layout(sm.CsmRangeInserterOptions2D, "csm_range_inserter_options2d")
    _layout(sm.CsmRtGrid2DInfo, "csm_rt_grid2d_info")


def test_symbols_are_exported(csm):
    out = subprocess.check_output(["nm", "-D", "--defined-only", csm.SO_PATH], text=True)
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for sym in ("csm_range_inserter2d_create", "csm_range_inserter2d_destroy",
                "csm_range_inserter2d_insert", "csm_rt_grid2d_create_empty", "csm_rt_grid2d_crop",
                "csm_rt_grid2d_read", "csm_stack2d_create_from_rt_grid2d"):
        assert sym in names, sym


def test_invalid_calls_and_no_device(csm):
    from cartographer_b200 import scan_matching as sm
    lib = csm.lib()
    out = C.c_void_p()
    for bad in (dict(hit_probability=0.5), dict(hit_probability=1.0), dict(miss_probability=0.5),
                dict(miss_probability=-0.1)):
        o = sm.ProbabilityGridRangeDataInserterOptions2D(**bad)._c()
        assert lib.csm_range_inserter2d_create(C.byref(o), 0, C.byref(out)) == 1
    assert lib.csm_range_inserter2d_create(None, 0, C.byref(out)) == 1
    assert lib.csm_range_inserter2d_insert(None, None, None, 0, None, 0, None, None) == 1
    assert lib.csm_range_inserter2d_destroy(None) == 0
    info = sm.CsmRtGrid2DInfo()
    assert lib.csm_rt_grid2d_read(None, C.byref(info), None, C.c_int64(0)) == 1
    assert lib.csm_rt_grid2d_crop(None, C.byref(out)) == 1
    assert lib.csm_stack2d_create_from_rt_grid2d(None, 7, C.byref(out)) == 1
    d = C.c_double
    assert lib.csm_rt_grid2d_create_empty(d(0.0), d(1.0), d(1.0), 100, 100, 0, C.byref(out)) == 1
    assert lib.csm_rt_grid2d_create_empty(d(0.05), d(1.0), d(1.0), 30000, 100, 0, C.byref(out)) == 1
    count = C.c_int32(0)
    if lib.csm_device_count(C.byref(count)) == 0 and count.value > 0:
        pytest.skip("GPU present")
    o = sm.ProbabilityGridRangeDataInserterOptions2D()._c()
    assert lib.csm_range_inserter2d_create(C.byref(o), 0, C.byref(out)) == 2, "expected CSM_E_CUDA"
    assert lib.csm_rt_grid2d_create_empty(d(0.05), d(1.0), d(1.0), 100, 100, 0, C.byref(out)) == 2
