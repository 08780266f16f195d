"""The CPU restatement of VoxelFilter / AdaptiveVoxelFilter (tests/voxel_filter_oracle.cc)
against the reference's voxel_filter_test.cc cases, hand-derived keys, hand-traced adaptive
searches and libstdc++'s scaling path; and the voxel-filter entry points' refusals, which
return status codes without a device."""
import ctypes as C

import numpy as np
import pytest

from tests import voxel_filter_oracle as O

M = 2**31 - 1          # minstd_rand0 modulus
URNG_RANGE = 2**31 - 3  # its max() - min()


# ---- sensor/internal/voxel_filter_test.cc ----

def test_returns_one_point_in_each_voxel():
    pts = [[0, 0, 0], [0.1, -0.1, 0.1], [0.3, -0.1, 0], [0, 0, 0.1]]
    kept, _ = O.voxel_filter(pts, 0.3)
    assert len(kept) == 2 and 2 in kept


def test_correct_intensities():
    pts = [[-100, 0.3, np.float32(0.1) * i] for i in range(100)]
    kept, _ = O.voxel_filter(pts, 0.3)
    assert len(kept) > 0 and np.all(np.diff(kept) > 0) and kept.max() < 100


def test_handles_large_coordinates():
    pts = [[100000, 0, 0], [100000.001, -0.0001, 0.0001], [100000.003, -0.0001, 0],
           [-200000, 0, 0]]
    kept, _ = O.voxel_filter(pts, 0.01)
    assert len(kept) == 2 and 3 in kept


def test_ignores_time():
    kept, st = O.voxel_filter([[-100, 0.3, 0.4]] * 100, 0.3)
    assert len(kept) == 1 and st["calls"] == 99


# ---- keys ----

def _key(x, y, z):
    u = lambda v: v & (2**64 - 1)
    return u((u(x) << 42) + (u(y) << 21) + u(z))


def test_keys_round_half_away_from_zero_on_both_signs():
    assert O.key(0.5, -0.5, 1.5, 1.0) == _key(1, -1, 2)
    assert O.key(-1.5, 2.5, -2.5, 1.0) == _key(-2, 3, -3)
    assert O.key(0.49999997, -0.49999997, 0.0, 1.0) == _key(0, 0, 0)
    assert O.key(0.25, -0.75, 0.05, 0.1) == _key(3, -8, 1)   # 0.25f / 0.1f = 2.5 exactly
    assert O.key(0.0, 0.0, -1.0, 1.0) == 2**64 - 1            # the all-ones key exists


def test_key_wraps_and_distinct_voxels_collide():
    a = O.key(3.0, -1.0, float(2**21), 1.0)
    b = O.key(3.0, 0.0, 0.0, 1.0)
    assert a == b == _key(3, 0, 0)
    kept, _ = O.voxel_filter([[3.0, -1.0, 2.0**21], [3.0, 0.0, 0.0]], 1.0)
    assert len(kept) == 1


# ---- the adaptive search, traced by hand on points at x = 0, 1, ..., 7 ----

LINE = [[float(i), 0.0, 0.0] for i in range(8)]


def test_adaptive_early_return_is_the_range_filtered_cloud():
    kept, st = O.adaptive_voxel_filter(LINE + [[100.0, 0, 0]], 1.0, 8, 50.0)
    assert list(kept) == list(range(8)) and st["trials"] == 0


def test_adaptive_max_length_is_enough():
    kept, st = O.adaptive_voxel_filter(LINE, 1.0, 8 - 1, 1e9)
    # 8 points > 7; VoxelFilter(1) keeps all 8 >= 7
    assert list(kept) == list(range(8)) and st["length"] == 1.0 and st["trials"] == 1


def test_adaptive_halving_then_bisection():
    # 16: 1 voxel; 8: 2; 4: 3; 2: 5 >= 5 -> bisect 3 (3), 2.5 (4), 2.25 (4), 2.125 (4)
    kept, st = O.adaptive_voxel_filter(LINE, 16.0, 5, 1e9)
    assert st["length"] == 2.0 and st["trials"] == 8 and len(kept) == 5


def test_adaptive_nothing_qualifies_returns_the_last_low_filter():
    kept, st = O.adaptive_voxel_filter([[1.0, 2.0, 3.0]] * 4, 8.0, 2, 1e9)
    # 4 > 2 points, one voxel at every length: VoxelFilter(8 / 128), not the input cloud
    assert st["length"] == 8.0 / 128 and st["trials"] == 8 and len(kept) == 1
    direct, _ = O.voxel_filter([[1.0, 2.0, 3.0]] * 4, 8.0 / 128)
    assert list(kept) == list(direct)


def test_adaptive_min_num_points_compares_as_float():
    # with 4: 2.5 (4) and 2.75 (4) qualify; with 4.5 nothing after 2 does
    _, st4 = O.adaptive_voxel_filter(LINE, 4.0, 4.0, 1e9)
    _, st45 = O.adaptive_voxel_filter(LINE, 4.0, 4.5, 1e9)
    assert st4["length"] == 2.75 and st45["length"] == 2.0
    kept, st = O.adaptive_voxel_filter(LINE, 4.0, 8.5, 1e9)      # 8 <= 8.5: early return
    assert len(kept) == 8 and st["trials"] == 0


def test_adaptive_max_range_is_inclusive():
    pts = [[3.0, 4.0, 0.0], [3.0, 4.0, 0.01]]   # norm 5 exactly, and just beyond
    kept, _ = O.adaptive_voxel_filter(pts, 1.0, 10, 5.0)
    assert list(kept) == [0]


# ---- libstdc++'s scaling path for minstd_rand0 ----

def skip_ahead(j):
    """16807^j mod (2^31 - 1) for an array of j, by square and multiply."""
    j = np.asarray(j, np.uint64).copy()
    r = np.ones_like(j)
    b = np.full_like(j, 16807)
    while np.any(j):
        odd = (j & np.uint64(1)).astype(bool)
        r[odd] = (r[odd] * b[odd]) % np.uint64(M)
        b = (b * b) % np.uint64(M)
        j >>= np.uint64(1)
    return r


def scaled(raw, k):
    """The distribution's result from one accepted raw output, or None if it is rejected."""
    scaling = URNG_RANGE // k
    ret = int(raw) - 1
    return None if ret >= k * scaling else ret // scaling + 1


def test_skip_ahead_equals_stepping():
    n = 10**6
    stepped = O.generator(n).astype(np.uint64)
    np.testing.assert_array_equal(skip_ahead(np.arange(1, n + 1)), stepped)


def test_scaling_path_equals_uniform_int_distribution():
    raw = O.generator(200000)
    rng = np.random.RandomState(3)
    for k in list(range(2, 40)) + [1000, 30000, 300000, 2**20 + 7, 2**30 + 3]:
        for at in rng.randint(0, len(raw) - 100, 200):
            want, used = O.uniform(k, raw[at:at + 100])
            t = 0
            while scaled(raw[at + t], k) is None:
                t += 1
            assert (scaled(raw[at + t], k), t + 1) == (want, used), (k, at)


def test_rejected_outputs_draw_again():
    k = 2**30 + 3                         # past = k: about half the outputs are rejected
    past = k * (URNG_RANGE // k)
    raw = np.array([past + 1, past + 5, 12345], np.uint32)   # ret = past, past + 4: rejected
    assert O.uniform(k, raw) == (scaled(12345, k), 3)


def test_restatement_counts_rejections():
    kept, st = O.voxel_filter(np.zeros((30000, 3), np.float32), 1.0)
    assert len(kept) == 1 and st["calls"] == 29999 and st["rejections"] >= 1


# ---- refusals (no device needed: arguments are checked first) ----

@pytest.fixture(scope="module")
def csm():
    import os
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def _call(csm, fn, clouds, param, counts=None, kept=True, num_kept=True):
    clouds = [np.ascontiguousarray(c, np.float32) for c in clouds]
    ptrs = (C.POINTER(C.c_float) * max(len(clouds), 1))(*[csm.ptr(c, C.c_float) for c in clouds])
    counts = np.array([len(c) for c in clouds] if counts is None else counts, np.int32)
    out = np.full(max(int(np.abs(counts).sum()), 1), -7, np.int32)
    nk = np.full(max(len(clouds), 1), -7, np.int32)
    st = fn(ptrs, csm.ptr(counts, C.c_int32), param, len(clouds), 0,
            csm.ptr(out, C.c_int32) if kept else None, csm.ptr(nk, C.c_int32) if num_kept else None,
            None)
    assert np.all(out == -7) and np.all(nk == -7)   # nothing written
    return st


def test_refusals(csm):
    from cartographer_b200 import sensor
    lib = csm.lib()
    good = np.zeros((4, 3), np.float32)
    res = lambda v: csm.ptr(np.array([v], np.float32), C.c_float)
    vf = lib.csm_voxel_filter_batch
    for bad in (0.0, -1.0, np.inf, np.nan):
        assert _call(csm, vf, [good], res(bad)) == 1
    for coord in (np.nan, np.inf, -np.inf):
        pts = good.copy()
        pts[2, 1] = coord
        assert _call(csm, vf, [pts], res(0.1)) == 1
    assert _call(csm, vf, [good], res(0.1), counts=[-1]) == 1
    assert _call(csm, vf, [good], res(0.1), kept=False) == 1
    assert _call(csm, vf, [good], res(0.1), num_kept=False) == 1
    assert _call(csm, vf, [good], None) == 1
    avf = lib.csm_adaptive_voxel_filter_batch

    def opt(max_length, min_num_points=10.0, max_range=50.0):
        o = (sensor.CsmAdaptiveVoxelFilterOptions * 1)()
        o[0] = sensor.CsmAdaptiveVoxelFilterOptions(max_length, min_num_points, max_range, 0)
        return o
    for bad in (0.0, -2.0, np.inf, np.nan):
        assert _call(csm, avf, [good], opt(bad)) == 1
    assert _call(csm, avf, [good], opt(1.0, np.nan)) == 1
    assert _call(csm, avf, [good], opt(1.0, 10.0, np.nan)) == 1
    assert _call(csm, avf, [good], None) == 1
    pts = good.copy()
    pts[0, 0] = np.nan
    assert _call(csm, avf, [pts], opt(1.0)) == 1
