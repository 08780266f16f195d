"""The CPU restatement of XRayPointsProcessor (tests/xray_oracle.cc) on hand-derived cases (the
reference has no test of this processor), the PNG encoding, and the csm_xray entry points'
symbols, declarations and refusals, which need no device."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from cartographer_b200 import points_processing as pp
from tests import xray_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WHITE = 0xFFFFFFFF
f32, f64 = np.float32, np.float64


def _word(r, g, b):
    return 0xFF000000 | r << 16 | g << 8 | b


def _byte(c):
    """FloatComponentToUint8 in numpy: clamp, * 255 in float, round half away from zero."""
    c = f32(c)
    c = f32(1) if c > 1 else (f32(0) if c < 0 else c)
    x = f32(c * f32(255))
    return int(math.floor(float(x) + 0.5))


def _mix(b, t):
    """Mix(1.f, b, t) with the reference's types: a double product plus a float product."""
    return f32(f64(1.0) * (1.0 - f64(t)) + f64(f32(f32(t) * f32(b))))


def _saturation(n, n_max, factor):
    top = max(f32(np.finfo(np.float32).tiny), f32(math.log(n_max)))
    s = f32(math.log(n) / f64(top) * factor)
    return s if s < f32(1) else f32(1)


# ---- Insert and the image on small scenes ----

def test_single_point_is_white():
    # n == 1 everywhere: max stays FLT_MIN, log(1) / max = 0, Mix(1, mean, 0) = 1
    p = O.Processor(0.1)
    assert p.insert([[1.0, 2.0, 3.0]], [[0.2, 0.4, 0.6]])
    lo, hi, empty = p.bounding_box()
    assert not empty and lo.tolist() == hi.tolist() == [10, 20, 30]
    assert p.draw().tolist() == [[WHITE]]
    yz, sums, counts = p.columns()
    assert yz.tolist() == [[20, 30]] and counts.tolist() == [1]
    np.testing.assert_array_equal(sums, f32([[0.2, 0.4, 0.6]]))


def test_columns_of_three_two_and_one_voxels():
    p = O.Processor(1.0)
    red = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0], [2.2, 0.0, 0.0]]
    green = [[0.0, 1.0, 0.0], [1.0, 1.0, 0.0]]
    blue = [[5.0, 2.0, 0.0]]
    assert p.insert(red, [[1, 0, 0]] * 4)
    assert p.insert(green, [[0, 1, 0]] * 2)
    assert p.insert(blue, [[0, 0, 1]])
    assert p.voxels().tolist() == [[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0], [1, 1, 0],
                                   [5, 2, 0]]
    assert p.columns()[2].tolist() == [4, 2, 1]              # points, not voxels
    img = p.draw()
    assert img.shape == (1, 3)                               # y in [0, 2], z in [0, 0]
    # pixel x = max.y - y: blue (n = 1), green (n = 2), red (n = 3 = max)
    light = round(255 * (1 - math.log(2) / math.log(3)))     # 94
    assert light == 94 and _byte(_mix(0.0, _saturation(2, 3, 1.0))) == light
    assert img.tolist() == [[WHITE, _word(light, 255, light), _word(255, 0, 0)]]


def test_colourless_batches_count_as_black():
    p = O.Processor(1.0)
    assert p.insert([[0.0, 0.0, 0.0]], [[1.0, 1.0, 1.0]])
    assert p.insert([[1.0, 0.0, 0.0]])                       # no colours
    yz, sums, counts = p.columns()
    assert sums.tolist() == [[1.0, 1.0, 1.0]] and counts.tolist() == [2]
    # n = 2 = max: saturation 1, the mean 0.5 -> 127.5 -> 128
    assert p.draw().tolist() == [[_word(128, 128, 128)]]


def test_rounding_ties_on_both_signs_after_a_rotation():
    # 180 degrees about z (q = (0, 0, 0, 1)) maps (x, y, z) to (-x, -y, z) exactly; then + t
    t = (0.25, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)
    p = O.Processor(1.0, transform=t)
    assert p.insert([[0.25, 1.5, -2.5], [-0.25, -0.5, 0.5], [0.75, 2.5, 1.5]])
    # (0, -1.5, -2.5), (0.5, 0.5, 0.5), (-0.5, -2.5, 1.5): lround rounds half away from zero
    assert p.voxels().tolist() == [[0, -2, -3], [1, 1, 1], [-1, -3, 2]]
    lo, hi, _ = p.bounding_box()
    assert lo.tolist() == [-1, -3, -3] and hi.tolist() == [1, 1, 2]


@pytest.mark.parametrize("factor,expected", [(0.5, 128), (1.0, 0), (3.0, 0)])
def test_saturation_factor(factor, expected):
    # a column of two voxels (the max) in black next to a lone voxel: saturation = factor,
    # capped at 1
    p = O.Processor(1.0, saturation_factor=factor)
    assert p.insert([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    img = p.draw()
    assert img[0, 1] == _word(expected, expected, expected)
    assert img[0, 0] == WHITE
    assert _byte(_mix(0.0, _saturation(2, 2, factor))) == expected


def test_saturation_clamps_above_one():
    # n = 2 next to n = 3 at factor 3: log 2 / log 3 * 3 = 1.89 -> 1; at 1: 0.63 -> lighter
    for factor, want in ((3.0, 0), (1.0, 94)):
        p = O.Processor(1.0, saturation_factor=factor)
        assert p.insert([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0],
                         [0.0, 1.0, 0.0], [1.0, 1.0, 0.0]])
        assert p.draw()[0, 0] == _word(want, want, want)


# Mix(1.f, b, t) where the reference's double evaluation and an all-float one round to
# different bytes: 210 against 209 (found by a seeded search over uniform floats).
MIX_B = np.array([1045960876], np.uint32).view(np.float32)[0]   # 0.21103162
MIX_T = np.array([1046975982], np.uint32).view(np.float32)[0]   # 0.22615787


def test_mix_is_evaluated_in_double():
    all_float = f32(f32(f32(1) * f32(f32(1) - MIX_T)) + f32(MIX_T * MIX_B))
    assert _byte(all_float) == 209
    assert _byte(_mix(MIX_B, MIX_T)) == 210
    assert O.channel(MIX_B, MIX_T) == 210


def test_column_sum_depends_on_point_order():
    tiny = 2.0 ** -24
    a, b = O.Processor(1.0), O.Processor(1.0)
    # (1 + 2^-24) + 2^-24 rounds to 1 twice; 2^-24 + 2^-24 + 1 = 1 + 2^-23 exactly
    assert a.insert([[0, 0, 0], [1, 0, 0], [2, 0, 0]], [[1, 0, 0], [tiny, 0, 0], [tiny, 0, 0]])
    assert b.insert([[0, 0, 0], [1, 0, 0], [2, 0, 0]], [[tiny, 0, 0], [tiny, 0, 0], [1, 0, 0]])
    assert a.columns()[1][0, 0] == f32(1.0)
    assert b.columns()[1][0, 0] == f32(1.0 + 2.0 ** -23)


def test_aggregations_share_one_box():
    p = O.Processor(1.0, num_aggregations=3)
    batch = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]]
    assert p.insert(batch, aggregation=0)
    assert p.insert(batch, aggregation=1)                   # a batch in two floors
    assert p.insert([[0.0, 4.0, 2.0]], aggregation=1)
    lo, hi, _ = p.bounding_box()
    assert lo.tolist() == [0, 0, 0] and hi.tolist() == [1, 4, 2]
    img0, img1, img2 = p.draw(0), p.draw(1), p.draw(2)
    assert img0.shape == img1.shape == img2.shape == (3, 5)
    # aggregation 0 has only (y, z) = (0, 0), at pixel (4 - 0, 2 - 0); n = 2 = its own max
    assert img0[2, 4] == _word(0, 0, 0) and (img0 == WHITE).sum() == 14
    assert img1[2, 4] == _word(0, 0, 0) and img1[0, 0] == WHITE          # (4, 2): n = 1
    assert (img2 == WHITE).all()                            # a floor without points


def test_empty_box_draws_nothing():
    p = O.Processor(0.05)
    assert p.bounding_box()[2] and p.draw() is None
    assert p.insert(np.zeros((0, 3), np.float32))
    assert p.bounding_box()[2] and p.draw() is None


def test_cube_edges():
    for v, ok in ((-8192.0, True), (8191.0, True), (8191.49, True), (8191.5, False),
                  (8192.0, False), (-8192.5, False), (-8193.0, False)):
        for axis in range(3):
            point = [0.0, 0.0, 0.0]
            point[axis] = v
            p = O.Processor(1.0)
            assert p.insert([[0.0, 0.0, 0.0], point]) == ok, (v, axis)
            assert len(p.voxels()) == (2 if ok else 0)      # a refused batch adds nothing
            assert p.bounding_box()[2] != ok


def test_cairo_word_layout():
    p = O.Processor(1.0)
    assert p.insert([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]], [[1.0, 0.5, 0.0]] * 2)
    (word,), = p.draw().tolist()
    assert word == 0xFFFF8000
    assert pp.cairo_to_rgb(np.uint32([[word]])).tolist() == [[[255, 128, 0]]]


def test_png_round_trip():
    rng = np.random.RandomState(7)
    p = O.Processor(0.5, transform=(0.1, -0.2, 0.3, 0.9238795, 0.0, 0.0, 0.38268343))
    pts = rng.uniform(-4, 4, (500, 3)).astype(np.float32)
    assert p.insert(pts, rng.uniform(0, 1, (500, 3)).astype(np.float32))
    img = p.draw()
    data = pp.encode_png(img)
    assert data[:8] == b"\x89PNG\r\n\x1a\n" and data.count(b"IDAT") == 1
    got = pp.decode_png(data)
    assert got.shape == img.shape + (3,)
    np.testing.assert_array_equal(got[..., 0], (img >> 16) & 0xFF)
    np.testing.assert_array_equal(got[..., 1], (img >> 8) & 0xFF)
    np.testing.assert_array_equal(got[..., 2], img & 0xFF)
    assert (img == WHITE).any() and (img != WHITE).any()


# ---- the library: symbols, declarations, refusals (no device needed) ----

ENTRY_POINTS = ["csm_xray_create", "csm_xray_destroy", "csm_xray_insert",
                "csm_xray_bounding_box", "csm_xray_draw", "csm_xray_voxels", "csm_xray_columns"]


@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def test_symbols_exported(csm):
    L = csm.lib()
    for name in ENTRY_POINTS:
        assert hasattr(L, name), name


def test_declarations_have_the_documented_types(tmp_path):
    src = tmp_path / "decl.c"
    src.write_text("""
#include "csm_abi.h"
csm_status (*create)(double, double, const float*, int32_t, int32_t, csm_xray**) = csm_xray_create;
csm_status (*destroy)(csm_xray*) = csm_xray_destroy;
csm_status (*insert)(csm_xray*, int32_t, const float* const*, const float* const*, const int32_t*,
                     int32_t, csm_stats*) = csm_xray_insert;
csm_status (*box)(const csm_xray*, int32_t*, int32_t*, int32_t*) = csm_xray_bounding_box;
csm_status (*draw)(csm_xray*, int32_t, uint32_t*, int64_t, int32_t*, int32_t*, csm_stats*) =
    csm_xray_draw;
csm_status (*voxels)(const csm_xray*, int32_t, int32_t*, int64_t, int64_t*) = csm_xray_voxels;
csm_status (*columns)(const csm_xray*, int32_t, int32_t*, float*, uint32_t*, int64_t, int64_t*) =
    csm_xray_columns;
_Static_assert(sizeof(csm_stats) == 64, "csm_stats");
""")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-fsyntax-only",
                           "-I", os.path.join(ROOT, "include"), str(src)])


def test_refusals_without_a_device(csm):
    from cartographer_b200 import _lib
    L = csm.lib()
    h = C.c_void_p()
    t = np.float32([0, 0, 0, 1, 0, 0, 0])
    tp = _lib.ptr(t, C.c_float)
    for vs, sf in ((0.0, 1.0), (-0.1, 1.0), (np.inf, 1.0), (np.nan, 1.0), (1e-50, 1.0),
                   (0.1, np.nan), (0.1, np.inf)):
        assert L.csm_xray_create(C.c_double(vs), C.c_double(sf), tp, 1, 0, C.byref(h)) == 1
        assert h.value is None
    bad = np.float32([0, 0, np.nan, 1, 0, 0, 0])
    assert L.csm_xray_create(C.c_double(0.1), C.c_double(1.0), _lib.ptr(bad, C.c_float), 1, 0,
                             C.byref(h)) == 1
    assert L.csm_xray_create(C.c_double(0.1), C.c_double(1.0), tp, 0, 0, C.byref(h)) == 1
    assert L.csm_xray_create(C.c_double(0.1), C.c_double(1.0), None, 1, 0, C.byref(h)) == 1
    assert L.csm_xray_create(C.c_double(0.1), C.c_double(1.0), tp, 1, 0, None) == 1
    pts = np.zeros((2, 3), np.float32)
    ptrs = (C.POINTER(C.c_float) * 1)(_lib.ptr(pts, C.c_float))
    cnt = np.array([2], np.int32)
    lo, hi, e = np.zeros(3, np.int32), np.zeros(3, np.int32), C.c_int32()
    w, ht, n = C.c_int32(), C.c_int32(), C.c_int64()
    assert L.csm_xray_insert(None, 0, ptrs, None, _lib.ptr(cnt, C.c_int32), 1, None) == 1
    assert L.csm_xray_bounding_box(None, _lib.ptr(lo, C.c_int32), _lib.ptr(hi, C.c_int32),
                                   C.byref(e)) == 1
    assert L.csm_xray_draw(None, 0, None, C.c_int64(0), C.byref(w), C.byref(ht), None) == 1
    assert L.csm_xray_voxels(None, 0, None, C.c_int64(0), C.byref(n)) == 1
    assert L.csm_xray_columns(None, 0, None, None, None, C.c_int64(0), C.byref(n)) == 1
    assert L.csm_xray_destroy(None) == 0
