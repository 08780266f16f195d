"""The device OutlierRemovingPointsProcessor (csm_outlier_remover_*) against the CPU restatement
(tests/outlier_removal_oracle.cc): the voxels after phase 1 and after phase 2 and every batch's
kept indices must be equal, count for count and index for index."""
import functools

import numpy as np
import pytest

from benchmarks import synthetic
from tests import outlier_removal_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def P():
    from cartographer_b200 import points_processing
    return points_processing


@functools.lru_cache(maxsize=None)
def _scans(seed=3, num_scans=10):
    return synthetic.moving_box_scans(seed, num_scans)


def _chunks(seq, size):
    return [seq[i:i + size] for i in range(0, len(seq), size)] if seq else [[]]


def _device(P, batches, voxel_size, limit, per_call=None, remover=None):
    r = remover or P.OutlierRemover(voxel_size, limit)
    groups = _chunks(list(batches), per_call or max(1, len(batches)))
    for g in groups:
        st = r.add_hits([p for _, p in g])
        assert st["host_syncs"] == (1 if sum(len(p) for _, p in g) else 0)
    hits = r.voxels()
    for g in groups:
        st = r.count_rays([o for o, _ in g], [p for _, p in g])
        assert st["host_syncs"] == (1 if sum(len(p) for _, p in g) else 0)
    rays = r.voxels()
    kept = []
    for g in groups:
        k, st = r.filter([p for _, p in g])
        assert st["host_syncs"] == (1 if sum(len(p) for _, p in g) else 0)
        kept += k
    return hits, rays, kept, r


def _assert_equal(got, want):
    for a, b in zip(got[0], want[0]):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(got[1], want[1]):
        np.testing.assert_array_equal(a, b)
    assert len(got[2]) == len(want[2])
    for a, b in zip(got[2], want[2]):
        np.testing.assert_array_equal(a, b)


@functools.lru_cache(maxsize=None)
def _oracle(voxel_size, limit, seed=3, num_scans=10):
    return O.run(_scans(seed, num_scans), voxel_size, limit)


@pytest.mark.parametrize("voxel_size", [0.05, 0.1, 0.15])
@pytest.mark.parametrize("limit", [3.0, 0.5, 0.0])
def test_moving_box_trajectory(P, voxel_size, limit):
    want = _oracle(voxel_size, limit)
    got = _device(P, _scans(), voxel_size, limit)
    _assert_equal(got[:3], want)
    total = sum(len(p) for _, p in _scans())
    kept = sum(len(k) for k in got[2])
    assert kept < total                          # removals happen
    if limit == 3.0:
        assert kept > total // 2
        assert got[1][2].max() > 0               # rays were counted


def test_grouping_of_batches_into_calls(P):
    want = _oracle(0.1, 3.0)
    for per_call in (1, 3, 10):
        _assert_equal(_device(P, _scans(), 0.1, 3.0, per_call=per_call)[:3], want)


def test_map_grows_from_a_small_start_over_hundreds_of_batches(P):
    batches = []
    for o, p in _scans():
        batches += [(o, p[i:i + 256]) for i in range(0, len(p), 256)]
    assert len(batches) >= 300
    r = P.OutlierRemover(0.05, 3.0)
    start = r.info()["slots"]
    got = _device(P, batches, 0.05, 3.0, per_call=1, remover=r)
    info = r.info()
    assert info["slots"] >= 8 * start and 2 * info["voxels"] <= info["slots"]
    assert info["voxels"] == len(got[0][1])
    _assert_equal(got[:3], O.run(batches, 0.05, 3.0))


def test_cube_faces(P):
    from cartographer_b200._lib import CsmError
    inside = np.float32([[-8192, 0, 0], [8191, 0, 0], [0, -8192, 8191], [0, 8191, -8192],
                         [8191.49, -8192.5 + 0.01, 0]])
    r = P.OutlierRemover(1.0, 3.0)
    o = O.Processor(1.0, 3.0)
    r.add_hits([inside])
    assert o.add_hits(inside)
    before = r.voxels()
    for bad in ([8192, 0, 0], [0, -8193, 0], [0, 0, 8191.5], [-8192.5, 0, 0]):
        with pytest.raises(CsmError) as e:
            r.add_hits([np.float32([[1, 2, 3], bad])])
        assert e.value.status == 1
        assert not o.add_hits(np.float32([[1, 2, 3], bad]))
    after = r.voxels()
    for a, b in zip(before, after):
        np.testing.assert_array_equal(a, b)
    assert r.info()["phase"] == 1
    for a, b in zip(after, o.voxels()):
        np.testing.assert_array_equal(a, b)
    # rays from far outside the cube still count in it; phase 3 reads voxels outside as {0, 0}
    rays = [(np.float32([-9000.0, 0.0, 0.0]), inside), (np.float32([0, 0, 0]), inside)]
    r.count_rays([o_ for o_, _ in rays], [p for _, p in rays])
    for org, p in rays:
        assert o.count_rays(org, p)
    for a, b in zip(r.voxels(), o.voxels()):
        np.testing.assert_array_equal(a, b)
    pts = np.concatenate([inside, np.float32([[9000, 0, 0], [5, 5, 5]])])
    (k,), _ = r.filter([pts])
    np.testing.assert_array_equal(k, o.filter(pts))


def test_far_origin(P):
    scans = _scans()[:2]
    batches = [(o + np.float32([700.0, -450.0, 120.0]), p) for o, p in scans]
    _assert_equal(_device(P, batches, 0.25, 3.0)[:3], O.run(batches, 0.25, 3.0))


def test_narrowed_voxels_of_large_coordinates(P):
    # lround's 64-bit result narrowed to int: 2^34 + 2048 -> 2048 at 0.25 m, 4e30 -> LONG_MIN -> 0
    pts = np.float32([[2.0**32 + 512, 0.0, 0.0], [1e30, 0.5, 0.0], [128.0, 0.0, 0.0],
                      [0.0, 0.5, 0.0], [-(2.0**33), 1.0, 2.0]])
    r = P.OutlierRemover(0.25, 3.0)
    o = O.Processor(0.25, 3.0)
    r.add_hits([pts])
    assert o.add_hits(pts)
    for a, b in zip(r.voxels(), o.voxels()):
        np.testing.assert_array_equal(a, b)
    (k,), _ = r.filter([pts])                  # phase 2 may be empty
    np.testing.assert_array_equal(k, o.filter(pts))


def test_absorbed_step_is_refused(P):
    from cartographer_b200._lib import CsmError
    r = P.OutlierRemover(1e-6, 3.0)
    o = O.Processor(1e-6, 3.0)
    pts = np.float32([[1e-3, 0, 0], [0, 2e-3, 0]])
    r.add_hits([pts])
    assert o.add_hits(pts)
    edge = np.float32([[32.0, 0, 0]])                 # x stops growing at exactly 32
    longer = np.float32([[np.nextafter(np.float32(32), np.float32(64)), 0, 0]])
    with pytest.raises(CsmError) as e:
        r.count_rays([[0, 0, 0], [0, 0, 0]], [pts, longer])
    assert e.value.status == 1 and r.info()["phase"] == 1
    assert not o.count_rays([0, 0, 0], np.concatenate([pts, longer]))
    r.count_rays([[0, 0, 0], [0, 0, 0]], [pts, edge])
    assert o.count_rays([0, 0, 0], pts) and o.count_rays([0, 0, 0], edge)
    for a, b in zip(r.voxels(), o.voxels()):
        np.testing.assert_array_equal(a, b)


def test_empty_batches_and_calls(P):
    scans = _scans()[:3]
    e = np.zeros((0, 3), np.float32)
    batches = [(scans[0][0], e), scans[0], (scans[1][0], e), scans[1], scans[2], (scans[2][0], e)]
    r = P.OutlierRemover(0.1, 3.0)
    assert r.add_hits([])["host_syncs"] == 0
    got = _device(P, batches, 0.1, 3.0, remover=r)
    assert [len(k) for k in got[2]][0] == 0 and len(got[2]) == 6
    _assert_equal(got[:3], O.run(batches, 0.1, 3.0))
    k, st = r.filter([])
    assert k == [] and st["host_syncs"] == 0


def test_out_of_order_calls_are_refused(P):
    from cartographer_b200._lib import CsmError
    o, p = _scans()[0]
    r = P.OutlierRemover(0.1, 3.0)
    r.add_hits([p])
    r.count_rays([o], [p])
    with pytest.raises(CsmError) as e:
        r.add_hits([p])
    assert e.value.status == 1
    r.filter([p])
    with pytest.raises(CsmError):
        r.count_rays([o], [p])
    with pytest.raises(CsmError):
        r.add_hits([p])
    assert r.info()["phase"] == 3
    # phase 2 may be empty: filtering right after the hits is in order
    q = P.OutlierRemover(0.1, 3.0)
    q.add_hits([p])
    (k,), _ = q.filter([p])
    ref = O.Processor(0.1, 3.0)
    assert ref.add_hits(p)
    np.testing.assert_array_equal(k, ref.filter(p))


def test_two_independent_processors(P):
    a, b = P.OutlierRemover(0.1, 3.0), P.OutlierRemover(0.15, 0.5)
    scans = _scans()
    for o, p in scans:
        a.add_hits([p])
        b.add_hits([p])
    for o, p in scans:
        b.count_rays([o], [p])
        a.count_rays([o], [p])
    ka = [a.filter([p])[0][0] for _, p in scans]
    kb = [b.filter([p])[0][0] for _, p in scans]
    wa, wb = _oracle(0.1, 3.0), _oracle(0.15, 0.5)
    for x, y in zip(ka, wa[2]):
        np.testing.assert_array_equal(x, y)
    for x, y in zip(kb, wb[2]):
        np.testing.assert_array_equal(x, y)
    for x, y in zip(a.voxels(), wa[1]):
        np.testing.assert_array_equal(x, y)


def test_pipeline_stage(P):
    scans = _scans()[:4]
    want = O.run(scans, 0.1, 3.0)[2]
    stage = P.OutlierRemovingPointsProcessor(0.1)
    assert stage.kConfigurationFileActionName == "voxel_filter_and_remove_moving_objects"
    results = []
    for _ in range(3):
        for o, p in scans:
            stage.Process(P.PointsBatch(p, o, intensities=np.arange(len(p), dtype=np.float32),
                                        colors=np.repeat(np.arange(len(p), dtype=np.float32)[:, None],
                                                         3, 1)))
        results.append(stage.Flush())
    assert results == [P.FlushResult.kRestartStream] * 2 + [P.FlushResult.kFinished]
    for batch, (o, p), k in zip(stage.output, scans, want):
        np.testing.assert_array_equal(batch.points, p[k])
        np.testing.assert_array_equal(batch.intensities, k.astype(np.float32))
        np.testing.assert_array_equal(batch.colors[:, 1], k.astype(np.float32))


def test_config5_size(P):
    """200 batches of 65,536 points (64 rings x 1024 azimuths), in calls of 20 batches."""
    base = synthetic.moving_box_scans(5, 4, rings=64, azimuths=1024, max_range=8.0)
    batches = []
    for k in range(200):
        o, p = base[k % len(base)]
        batches.append((o, np.resize(p, (65536, 3))))
    got = _device(P, batches, 0.15, 3.0, per_call=20)
    _assert_equal(got[:3], O.run(batches, 0.15, 3.0))
