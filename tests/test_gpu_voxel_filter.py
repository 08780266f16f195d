"""The device VoxelFilter / AdaptiveVoxelFilter (csm_voxel_filter_batch,
csm_adaptive_voxel_filter_batch) against the CPU restatement (tests/voxel_filter_oracle.cc):
the kept input indices must be equal, index for index."""
import ctypes as C

import numpy as np
import pytest

from tests import voxel_filter_oracle as O

pytestmark = pytest.mark.gpu

HIGH = (2.0, 150.0, 15.0)            # trajectory_builder_3d.lua high_resolution_adaptive_voxel_filter
LOW = (4.0, 200.0, float(np.finfo(np.float32).max))   # low_resolution_adaptive_voxel_filter
ADAPTIVE_2D = (0.5, 200.0, 50.0)     # trajectory_builder_2d.lua adaptive_voxel_filter


@pytest.fixture(scope="module")
def S():
    from cartographer_b200 import sensor
    return sensor


def _opts(S, t):
    return S.AdaptiveVoxelFilterOptions(*t)


def _vf(S, pts, res):
    (kept,), stats = S.voxel_filter_batch([pts], [res])
    assert stats["host_syncs"] == 1
    return kept


def _avf(S, pts, t):
    (kept,), stats = S.adaptive_voxel_filter_batch([pts], [_opts(S, t)])
    assert stats["host_syncs"] == 1
    return kept


def _check_vf(S, pts, res):
    want, st = O.voxel_filter(pts, res)
    np.testing.assert_array_equal(_vf(S, pts, res), want)
    return st


def _check_avf(S, pts, t):
    want, st = O.adaptive_voxel_filter(pts, *t)
    np.testing.assert_array_equal(_avf(S, pts, t), want)
    return st


def test_reference_cases(S):
    pts = np.float32([[0, 0, 0], [0.1, -0.1, 0.1], [0.3, -0.1, 0], [0, 0, 0.1]])
    got = S.VoxelFilter(pts, 0.3)
    assert len(got) == 2 and any((got == pts[2]).all(1))
    _check_vf(S, pts, 0.3)
    z = np.float32(0.1) * np.arange(100, dtype=np.float32)
    pts = np.stack([np.full(100, -100.0), np.full(100, 0.3), z], 1).astype(np.float32)
    got, inten = S.VoxelFilter(pts, 0.3, intensities=z)
    assert len(inten) == len(got) and np.all(got[:, 2] == inten)
    _check_vf(S, pts, 0.3)
    pts = np.float32([[100000, 0, 0], [100000.001, -0.0001, 0.0001], [100000.003, -0.0001, 0],
                      [-200000, 0, 0]])
    got = S.VoxelFilter(pts, 0.01)
    assert len(got) == 2 and any((got == pts[3]).all(1))
    _check_vf(S, pts, 0.01)
    pts = np.tile(np.float32([[-100, 0.3, 0.4]]), (100, 1))
    assert len(S.VoxelFilter(pts, 0.3)) == 1
    _check_vf(S, pts, 0.3)


def test_keys_ties_signs_and_wraparound(S):
    pts = np.float32([[0.5, -0.5, 1.5], [-1.5, 2.5, -2.5], [0.49999997, -0.49999997, 0],
                      [0.0, 0.0, -1.0], [0.0, 0.0, -1.0], [3.0, -1.0, 2.0**21], [3.0, 0.0, 0.0],
                      [1e30, -1e30, 3e9], [0.0, 0.0, 0.0], [-3e9, 1e19, 0.0]])
    for res in (1.0, 0.5, 0.1, 1e-3):
        _check_vf(S, pts, res)


def test_scans_2d_and_3d(S):
    rng = np.random.RandomState(7)
    for seed in range(50):
        scan = O.planar_scan(seed)
        res = float(np.float32(10 ** rng.uniform(-2, np.log10(4.0))))
        _check_vf(S, scan, res)
        kept = _vf(S, scan, 0.025)
        _check_avf(S, scan[kept], ADAPTIVE_2D)
        _, inten = S.AdaptiveVoxelFilter(scan, _opts(S, ADAPTIVE_2D),
                                         intensities=np.arange(len(scan), dtype=np.float32))
        np.testing.assert_array_equal(inten, O.adaptive_voxel_filter(scan, *ADAPTIVE_2D)[0])
    for seed in range(50):
        scan = O.box_room_scan(seed)
        res = float(np.float32(10 ** rng.uniform(-2, np.log10(4.0))))
        _check_vf(S, scan, res)
        _check_vf(S, scan, 0.15)
        kept = _vf(S, scan, 0.15)
        for t in (HIGH, LOW):
            _check_avf(S, scan[kept], t)


def test_single_voxel_rejections(S):
    # 30 000 and 300 000 calls in one voxel reject 1 and 12 draws; 10^6 rejects more than the
    # 64 shifts each call tests, so the device steps the rest of the cloud call by call
    for n, least in ((30000, 1), (300000, 10), (1000000, 64)):
        pts = np.random.RandomState(n).uniform(0.0, 0.9, (n, 3)).astype(np.float32)
        st = _check_vf(S, pts, 2.0)
        assert st["rejections"] >= least, st


def test_empty_one_point_range_edge_and_large(S):
    for pts in (np.zeros((0, 3), np.float32), np.float32([[1, 2, 3]])):
        _check_vf(S, pts, 0.1)
        _check_avf(S, pts, ADAPTIVE_2D)
        _check_avf(S, pts, (0.5, 0.0, 50.0))
    edge = np.float32([[3, 4, 0], [3, 4, 0.01], [0, 0, 5], [-5, 0, 0], [0.5, 0.5, 0.5]])
    assert list(_avf(S, edge, (1.0, 10.0, 5.0))) == [0, 2, 3, 4]
    _check_avf(S, edge, (1.0, 2.0, 5.0))
    big = np.random.RandomState(1).uniform(-3e5, 3e5, (5000, 3)).astype(np.float32)
    _check_vf(S, big, 0.01)
    _check_avf(S, big, (0.5, 4000.0, 1e6))


def test_adaptive_branches_at_scale(S):
    scan = O.box_room_scan(3)
    cases = {
        "early return": (2.0, 70000.0, 1e9),
        "max_length enough": (0.05, 100.0, 1e9),
        "halving then bisection": (64.0, 3000.0, 1e9),
        "float min_num_points": (2.0, 1500.5, 1e9),
    }
    seen = {}
    for name, t in cases.items():
        seen[name] = _check_avf(S, scan, t)
    # every point twice: never 70 000 distinct voxels, but more points than that
    seen["nothing qualifies"] = _check_avf(S, np.vstack([scan, scan]), (1.0, 70000.0, 1e9))
    assert seen["early return"]["trials"] == 0
    assert seen["max_length enough"]["trials"] == 1
    assert seen["halving then bisection"]["trials"] > 3
    assert seen["nothing qualifies"]["length"] == np.float32(1.0) / 128


def test_batch_equals_one_by_one(S):
    rng = np.random.RandomState(11)
    clouds = [O.box_room_scan(100 + i, rings=16, azimuths=512) for i in range(4)] + \
        [O.planar_scan(200 + i) for i in range(4)] + [np.zeros((0, 3), np.float32),
                                                     np.float32([[1, 1, 1]])]
    res = [float(np.float32(10 ** rng.uniform(-2, 0.6))) for _ in clouds]
    got, st = S.voxel_filter_batch(clouds, res)
    assert st["host_syncs"] == 1
    for c, r, g in zip(clouds, res, got):
        np.testing.assert_array_equal(g, O.voxel_filter(c, r)[0])
    opts = [S.AdaptiveVoxelFilterOptions(*t) for t in
            (HIGH, LOW, ADAPTIVE_2D, (64.0, 3000.0, 1e9), (1.0, 65000.0, 8.0), (2.0, 10.0, 1e9),
             (0.5, 500.0, 50.0), (8.0, 2.0, 1e9), (0.5, 1.0, 1.0), HIGH)]
    got, st = S.adaptive_voxel_filter_batch(clouds, opts)
    trials = 0
    for c, o, g in zip(clouds, opts, got):
        want, ost = O.adaptive_voxel_filter(c, *o)
        trials += ost["trials"]
        np.testing.assert_array_equal(g, want)
        np.testing.assert_array_equal(S.adaptive_voxel_filter_batch([c], [o])[0][0], want)
    assert trials > 10 and st["host_syncs"] == 1 and st["device_ms"] > 0


def test_refused_calls_leave_outputs_untouched(S):
    from cartographer_b200 import _lib
    pts = O.planar_scan(1)
    S.voxel_filter_batch([pts], [0.05])          # a device context exists
    bad = pts.copy()
    bad[10, 0] = np.nan
    counts = np.array([len(bad)], np.int32)
    ptrs = (C.POINTER(C.c_float) * 1)(_lib.ptr(bad, C.c_float))
    out = np.full(len(bad), -7, np.int32)
    nk = np.full(1, -7, np.int32)
    res = np.float32([0.05])
    st = _lib.lib().csm_voxel_filter_batch(ptrs, _lib.ptr(counts, C.c_int32),
                                           _lib.ptr(res, C.c_float), 1, 0,
                                           _lib.ptr(out, C.c_int32), _lib.ptr(nk, C.c_int32), None)
    assert st == 1 and np.all(out == -7) and np.all(nk == -7)
    with pytest.raises(_lib.CsmError):
        S.adaptive_voxel_filter_batch([pts], [S.AdaptiveVoxelFilterOptions(0.0, 10.0, 50.0)])
