"""The CPU restatement of OutlierRemovingPointsProcessor (tests/outlier_removal_oracle.cc) on
hand-derived cases (the reference has no test of this processor), and the csm_outlier_remover
entry points' symbols, declarations and refusals, which need no device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import outlier_removal_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stream(batches, voxel_size, limit=3.0):
    return O.run(batches, voxel_size, limit)


# ---- the three phases on small scenes ----

def test_lone_point_is_kept():
    hits, rays, (kept,) = _stream([((0, 0, 0), [[1.0, 2.0, 3.0]])], 0.05)
    assert hits[0].tolist() == [[20, 40, 60]] and hits[1].tolist() == [1]
    assert rays[2].tolist() == [0]                 # 0 < 3 * 1
    assert kept.tolist() == [0]


def test_point_in_front_of_a_seen_through_wall_is_removed():
    # ten returns from a wall at x = 5 and one from x = 3 on the same line: the samples of every
    # ray to the wall pass through voxel 30 (x = 3.0), which holds one hit
    wall = [[5.0, 0.0, 0.0]] * 10
    pts = wall + [[3.0, 0.0, 0.0]]
    idx, hits, rays = _stream([((0, 0, 0), pts)], 0.1)[1]
    by = {tuple(i): (h, r) for i, h, r in zip(idx.tolist(), hits, rays)}
    # the last sample of a ray to x = 5, x_50 = 4.9999976 < 5, lands in the wall's own voxel 50
    assert O.ray_samples(0.1, 5.0)[-1] == np.float32(4.9999976)
    assert by[(50, 0, 0)] == (10, 10)              # 10 < 3 * 10: the wall stays
    assert by[(30, 0, 0)][0] == 1 and by[(30, 0, 0)][1] >= 10
    (kept,) = _stream([((0, 0, 0), pts)], 0.1)[2]
    assert kept.tolist() == list(range(10))


def test_phases_accumulate_over_batches():
    a = ((0, 0, 0), [[5.0, 0.0, 0.0]] * 4)
    b = ((0, 0, 1), [[3.0, 0.0, 0.6], [3.0, 0.0, 0.0]])
    one = _stream([a, b], 0.1)
    p = O.Processor(0.1)
    for _, pts in (a, b):
        assert p.add_hits(pts)
    for o, pts in (a, b):
        assert p.count_rays(o, pts)
    for x, y in zip(one[1], p.voxels()):
        np.testing.assert_array_equal(x, y)


# ---- x += voxel_size in float with a double step ----

def _emulated(voxel_size, length):
    xs, x = [], np.float32(0)
    while x < np.float32(length):
        xs.append(x)
        x = np.float32(np.float64(x) + voxel_size)
    return np.array(xs, np.float32)


@pytest.mark.parametrize("voxel_size", [0.05, 0.1, 0.15])
def test_sample_sequence_is_float_steps_of_a_double(voxel_size):
    full = _emulated(voxel_size, 60.0)
    np.testing.assert_array_equal(O.ray_samples(voxel_size, 60.0), full)
    # not k * voxel_size in float: the rounding errors accumulate
    assert not np.array_equal(full, (np.arange(len(full)) * voxel_size).astype(np.float32))
    for k in (1, 2, 3, 7, 100, len(full) - 1):
        # a ray exactly as long as x_k stops before it: x < length is strict
        got = O.ray_samples(voxel_size, float(full[k]))
        np.testing.assert_array_equal(got, full[:k])
        np.testing.assert_array_equal(got, _emulated(voxel_size, float(full[k])))
        nxt = np.nextafter(full[k], np.float32(np.inf))
        np.testing.assert_array_equal(O.ray_samples(voxel_size, float(nxt)), full[:k + 1])


def test_zero_length_rays_take_no_sample():
    assert len(O.ray_samples(0.05, 0.0)) == 0
    p = O.Processor(0.1)
    assert p.add_hits([[1.0, 1.0, 1.0]] * 3)
    assert p.count_rays([1.0, 1.0, 1.0], [[1.0, 1.0, 1.0]] * 3)
    assert p.voxels()[2].tolist() == [0] and p.filter([[1.0, 1.0, 1.0]]).tolist() == [0]


def test_absorbed_step_is_refused_and_changes_nothing():
    assert O.ray_samples(1e-30, 1.0) is None        # x = 1e-30 + 1e-30 ... never reaches 1
    assert O.ray_samples(1e-30, 1e-29) is not None
    p = O.Processor(1e-6)
    assert p.add_hits([[1e-3, 0.0, 0.0]])
    before = p.voxels()
    # at 1e-6 steps x stops growing at 32 (after 25107770 steps): a ray of 32 ends, a longer
    # one never does
    assert O.ray_samples(1e-6, 32.0, cap=0) is not None
    assert O.ray_samples(1e-6, float(np.nextafter(np.float32(32), np.float32(64))), cap=0) is None
    assert not p.count_rays([0.0, 0.0, 0.0], [[1e-3, 0.0, 0.0], [40.0, 0.0, 0.0]])
    for x, y in zip(before, p.voxels()):
        np.testing.assert_array_equal(x, y)


# ---- GetCellIndex: lround, narrowed to int ----

def test_rounding_ties_on_both_signs():
    assert O.cell_index([0.5, -0.5, 1.5], 1.0) == (1, -1, 2)
    assert O.cell_index([-1.5, 2.5, -2.5], 1.0) == (-2, 3, -3)
    assert O.cell_index([0.025, -0.025, 0.49999997], 0.05) == (1, -1, 10)
    assert O.cell_index([0.49999997, -0.49999997, 0.0], 1.0) == (0, 0, 0)
    p = O.Processor(1.0)
    assert p.add_hits([[0.5, -0.5, 0.0], [-0.5, 0.5, 0.0]])
    assert p.voxels()[0].tolist() == [[1, -1, 0], [-1, 1, 0]]


def test_narrowing_at_large_coordinates():
    # lround's long, narrowed to its low 32 bits; at or beyond 2^63 (x86-64) it is LONG_MIN -> 0
    assert O.cell_index([2.0**32 + 512, 0.0, 0.0], 1.0) == (512, 0, 0)
    wrapped = int(np.array([-(2**31) - 512], np.int64).astype(np.int32)[0])
    assert O.cell_index([-(2.0**31) - 512, 0.0, 0.0], 1.0) == (wrapped, 0, 0)
    assert O.cell_index([1e30, -1e30, 3.0], 1.0) == (0, 0, 3)
    p = O.Processor(1.0)
    assert p.add_hits([[2.0**32 + 512, 0.0, 0.0], [1e30, 0.0, 0.0]])   # voxels 512 and 0
    assert p.voxels()[0].tolist() == [[0, 0, 0], [512, 0, 0]]
    assert not p.add_hits([[2.0**31, 0.0, 0.0]])                         # -2^31: outside


def test_hits_must_lie_in_the_growable_cube():
    for v, ok in ((-8192.0, True), (8191.0, True), (8191.49, True), (8191.5, False),
                  (8192.0, False), (-8192.5, False), (-8193.0, False)):
        p = O.Processor(1.0)
        assert p.add_hits([[0.0, 0.0, 0.0], [0.0, v, 0.0]]) == ok, v
        assert len(p.voxels()[0]) == (2 if ok else 0)   # a refused batch adds nothing


# ---- phase 3: !(rays < limit * hits) in double ----

def _voxel_with(hits, rays, limit):
    """A processor whose voxel (0, 0, 0) at 1 m holds `hits` hits and `rays` rays: each ray runs
    from z = -3 to z = 9 and samples z = -3, -2, ..., 8, voxel 0 once."""
    p = O.Processor(1.0, limit)
    assert p.add_hits([[0.0, 0.0, 0.0]] * hits)
    assert p.count_rays([0.0, 0.0, -3.0], [[0.0, 0.0, 9.0]] * rays)
    idx, h, r = p.voxels()
    assert idx.tolist() == [[0, 0, 0]] and (h[0], r[0]) == (hits, rays)
    return p


@pytest.mark.parametrize("hits,rays,limit,kept", [
    (1, 0, 3.0, True), (1, 3, 3.0, False), (1, 2, 3.0, True),
    (2, 1, 0.5, False), (2, 0, 0.5, True), (4, 1, 0.5, True),
    (1, 0, 0.0, False), (5, 0, 0.0, False),
])
def test_limit_comparison(hits, rays, limit, kept):
    p = _voxel_with(hits, rays, limit)
    assert (p.filter([[0.0, 0.0, 0.0]]).tolist() == [0]) == kept


def test_equality_compares_in_double():
    # 1 < 0.5000000000000001 * 2 holds in double; 1 < 0.5 * 2 does not
    assert _voxel_with(2, 1, 0.5000000000000001).filter([[0.0, 0.0, 0.0]]).tolist() == [0]


def test_points_never_hit_are_removed():
    p = O.Processor(0.1, 3.0)
    assert p.add_hits([[1.0, 0.0, 0.0]])
    assert p.count_rays([0, 0, 0], [[1.0, 0.0, 0.0]])
    # voxel {0, 0}: !(0 < 3 * 0), inside the cube or not
    assert p.filter([[1.0, 0.0, 0.0], [2.0, 0.0, 0.0], [1e6, 0.0, 0.0]]).tolist() == [0]


# ---- the library: symbols, declarations, refusals (no device needed) ----

ENTRY_POINTS = ["csm_outlier_remover_create", "csm_outlier_remover_destroy",
                "csm_outlier_remover_add_hits", "csm_outlier_remover_count_rays",
                "csm_outlier_remover_filter", "csm_outlier_remover_voxels",
                "csm_outlier_remover_info"]


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
csm_status (*create)(double, double, int32_t, csm_outlier_remover**) = csm_outlier_remover_create;
csm_status (*destroy)(csm_outlier_remover*) = csm_outlier_remover_destroy;
csm_status (*add_hits)(csm_outlier_remover*, const float* const*, const int32_t*, int32_t,
                       csm_stats*) = csm_outlier_remover_add_hits;
csm_status (*count_rays)(csm_outlier_remover*, const float*, const float* const*, const int32_t*,
                         int32_t, csm_stats*) = csm_outlier_remover_count_rays;
csm_status (*filter)(csm_outlier_remover*, const float* const*, const int32_t*, int32_t,
                     int32_t*, int32_t*, csm_stats*) = csm_outlier_remover_filter;
csm_status (*voxels)(const csm_outlier_remover*, int32_t*, int32_t*, int32_t*, int64_t,
                     int64_t*) = csm_outlier_remover_voxels;
csm_status (*info)(const csm_outlier_remover*, int32_t*, int64_t*, int64_t*) =
    csm_outlier_remover_info;
_Static_assert(sizeof(csm_stats) == 64, "csm_stats");
""")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-fsyntax-only",
                           "-I", os.path.join(ROOT, "include"), str(src)])


def test_refusals_without_a_device(csm):
    from cartographer_b200 import _lib
    L = csm.lib()
    h = C.c_void_p()
    for vs, lim in ((0.0, 3.0), (-0.1, 3.0), (np.inf, 3.0), (np.nan, 3.0), (0.1, np.nan),
                    (0.1, np.inf), (0.1, -np.inf)):
        assert L.csm_outlier_remover_create(C.c_double(vs), C.c_double(lim), 0, C.byref(h)) == 1
        assert h.value is None
    assert L.csm_outlier_remover_create(C.c_double(0.1), C.c_double(3.0), 0, None) == 1
    pts = np.zeros((2, 3), np.float32)
    ptrs = (C.POINTER(C.c_float) * 1)(_lib.ptr(pts, C.c_float))
    cnt = np.array([2], np.int32)
    org = np.zeros(3, np.float32)
    kept = np.zeros(2, np.int32)
    nk = np.zeros(1, np.int32)
    n = C.c_int64()
    assert L.csm_outlier_remover_add_hits(None, ptrs, _lib.ptr(cnt, C.c_int32), 1, None) == 1
    assert L.csm_outlier_remover_count_rays(None, _lib.ptr(org, C.c_float), ptrs,
                                            _lib.ptr(cnt, C.c_int32), 1, None) == 1
    assert L.csm_outlier_remover_filter(None, ptrs, _lib.ptr(cnt, C.c_int32), 1,
                                        _lib.ptr(kept, C.c_int32), _lib.ptr(nk, C.c_int32),
                                        None) == 1
    assert L.csm_outlier_remover_voxels(None, None, None, None, 0, C.byref(n)) == 1
    assert L.csm_outlier_remover_info(None, None, None, None) == 1
    assert L.csm_outlier_remover_destroy(None) == 0
