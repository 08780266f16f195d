"""DrawProbabilityGrid's restatement (tests/probability_grid_draw_oracle.cc) on hand-derived
images, the grey level of every cell value through the library's host table against the
restatement's per-cell float expression and a numpy one, the map-writing stages' constants, and
the csm_rt_grid2d_draw symbols, declarations and refusals, which need no device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import probability_grid_draw_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _word(v):
    return 0xFF000000 | v << 16 | v << 8 | v


def _numpy_scaled(values):
    """255 * ((1 - GetProbability(v)) - kMinProbability) / (kMax - kMin), every step in float32."""
    k_min = f32(0.1)
    k_max = f32(1) - k_min
    lo, hi = f32(1) - k_max, f32(1) - k_min              # kMin/kMaxCorrespondenceCost
    step = f32((hi - lo) / f32(32766))
    cost = (np.asarray(values, np.float32) * step).astype(f32) + f32(lo - step)
    probability = f32(1) - (f32(1) - cost)
    return (f32(255) * ((probability - k_min) / (k_max - k_min))).astype(f32)


def _round_half_away(x):
    """RoundToInt (std::lround) of non-negative floats, exactly: x + 0.5 is exact in double."""
    return np.floor(np.asarray(x, np.float64) + 0.5).astype(np.int64)


# ---- the restatement on hand-derived cases ----
def test_unknown_and_extreme_values():
    assert O.grey(0) == 128                       # kUnknownValue
    assert O.grey(1) == 0                         # cost 0.1: probability 0.9, drawn black
    assert O.grey(32767) == 255                   # cost 0.9: probability 0.1, drawn white


def test_values_next_to_half_ties_round_as_in_float():
    # no value lands on an exact .5; these three come closest, on both sides
    for value, scaled, grey in ((5462, 42.500008, 43), (27306, 212.49998, 212),
                                (16384, 127.500015, 128)):
        assert abs(float(O.scaled(value)) - scaled) < 1e-5
        assert O.grey(value) == grey


def test_empty_box_draws_one_unknown_pixel_at_the_origin():
    pixels, offset = O.draw(np.zeros((3, 4), np.uint16), None)
    assert pixels.tolist() == [[_word(128)]] and offset == (0, 0)


def test_offset_and_orientation():
    cells = np.zeros((6, 7), np.uint16)             # cells[y, x]
    cells[1, 2] = 1                                  # black, the box's (min x, min y) corner
    cells[4, 5] = 32767                              # white, its (max x, max y) corner
    cells[1, 5] = 16384                              # 128, top right
    pixels, offset = O.draw(cells, (2, 1, 5, 4))
    assert offset == (2, 1) and pixels.shape == (4, 4)   # (height, width)
    want = np.full((4, 4), _word(128), np.uint32)
    want[0, 0] = _word(0)
    want[3, 3] = _word(255)
    want[0, 3] = _word(128)
    np.testing.assert_array_equal(pixels, want)
    # pixel (x, y) is cell (offset.x + x, offset.y + y), row-major with a stride of width
    cells[3, 4] = 20000
    pixels, _ = O.draw(cells, (2, 1, 5, 4))
    assert pixels[3 - 1, 4 - 2] == _word(O.grey(20000)) != _word(128)


# ---- every cell value ----
def test_every_value_in_float_against_numpy():
    values = np.arange(1, 32768)
    scaled = _numpy_scaled(values)
    frac = scaled.astype(np.float64) - np.floor(scaled)
    assert not (frac == 0.5).any()
    want = _round_half_away(scaled)
    got = np.array([O.grey(v) for v in values])
    np.testing.assert_array_equal(got, want)


@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def test_library_table_matches_the_restatement(csm):
    table = np.zeros(32768, np.uint8)
    assert csm.lib().csm_rt_grid2d_draw_table(csm.ptr(table, C.c_uint8)) == 0
    want = np.array([O.grey(v) for v in range(32768)])
    np.testing.assert_array_equal(table, want)


# ---- the library: symbols, declarations, refusals (no device needed) ----
def test_symbols_exported(csm):
    L = csm.lib()
    for name in ("csm_rt_grid2d_draw", "csm_rt_grid2d_draw_table"):
        assert hasattr(L, name), name


def test_declarations_have_the_documented_types(tmp_path):
    src = tmp_path / "decl.c"
    src.write_text("""
#include "csm_abi.h"
csm_status (*draw)(const csm_rt_grid2d*, uint32_t*, int64_t, int32_t*, int32_t*, int32_t*,
                   csm_stats*) = csm_rt_grid2d_draw;
csm_status (*table)(uint8_t*) = csm_rt_grid2d_draw_table;
""")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-fsyntax-only",
                           "-I", os.path.join(ROOT, "include"), str(src)])


def test_refusals_without_a_device(csm):
    L = csm.lib()
    w, h = C.c_int32(-1), C.c_int32(-1)
    offset = np.full(2, -1, np.int32)
    op = csm.ptr(offset, C.c_int32)
    assert L.csm_rt_grid2d_draw(None, None, C.c_int64(0), C.byref(w), C.byref(h), op, None) == 1
    assert (w.value, h.value, offset.tolist()) == (-1, -1, [-1, -1])
    assert L.csm_rt_grid2d_draw_table(None) == 1


def test_stage_constants():
    from cartographer_b200 import points_processing as pp
    assert pp.ProbabilityGridPointsProcessor.kConfigurationFileActionName == \
        "write_probability_grid"
    assert pp.HybridGridPointsProcessor.kConfigurationFileActionName == "write_hybrid_grid"
    with pytest.raises(ValueError, match="OutputType jpg does not exist!"):
        pp.ProbabilityGridPointsProcessor(0.05, None, "map", output_type="jpg")
