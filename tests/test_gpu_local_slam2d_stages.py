"""2D local SLAM on the device stage by stage (csm_local_slam2d_* through local_slam.py) against
the CPU chain of tests/local_slam2d_chain.py: every read-back hook bit for bit with the float32
restatement, the voxel filters and the insert, the real-time matcher bit for bit and the
refinement within 1e-7 of the oracle, at the inputs where the kernels go wrong."""
import gc
import math

import numpy as np
import pytest

from benchmarks import synthetic
from benchmarks.bench_insert2d import trajectory
from cartographer_b200 import local_slam as L
from cartographer_b200 import scan_matching as sm
from cartographer_b200 import sensor
from cartographer_b200._lib import CsmError
from tests import insert2d_oracle as I
from tests import local_slam2d_chain as K
from tests import local_slam2d_oracle as O
from tests import voxel_filter_oracle as VO

pytestmark = pytest.mark.gpu

F = np.float32
IDENT = L.rigid3f((0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))


def _tilted(rng, reach, roll=0.3, pitch=0.3):
    yaw = rng.uniform(-math.pi, math.pi)
    q = K.quat_mul64((math.cos(yaw / 2), 0, 0, math.sin(yaw / 2)),
                     K.quat_mul64((math.cos(rng.uniform(-pitch, pitch) / 2), 0,
                                   math.sin(rng.uniform(-pitch, pitch) / 2), 0),
                                  (math.cos(rng.uniform(-roll, roll) / 2),
                                   math.sin(rng.uniform(-roll, roll) / 2), 0, 0)))
    return L.rigid3f(rng.uniform(-reach, reach, 3), L._quatd_normalized(q))


def _flat(poses):
    return np.stack([L._flat(p) for p in poses])


def _bits(a, b):
    a, b = np.asarray(a, np.float32).reshape(-1, 3), np.asarray(b, np.float32).reshape(-1, 3)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _accumulate(slam, hits, origins, oi, poses, pi):
    st = slam.accumulate(hits, origins, oi, _flat(poses), pi)
    assert st["host_syncs"] == 0
    return st


def _check_accumulated(slam, want_r, want_m):
    assert _bits(slam.read(L.ACCUMULATED_RETURNS), want_r)
    assert _bits(slam.read(L.ACCUMULATED_MISSES), want_m)


def _opts(**kw):
    return L.LocalTrajectoryBuilderOptions2D(**kw)


# ---- a. accumulate ----
@pytest.mark.parametrize("per_point", [False, True])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 65537])
def test_accumulate_sizes_origins_and_poses(n, per_point):
    rng = np.random.RandomState(n + 7 * per_point)
    o = _opts(min_range=0.3, max_range=30.0, missing_data_ray_length=5.0)
    for num_origins in (1, 7, 16):
        slam = L.LocalSlam2D(o)
        origins = rng.uniform(-0.5, 0.5, (num_origins, 3)).astype(np.float32)
        oi = rng.randint(0, num_origins, n).astype(np.int32)
        num_poses = n if per_point else 1
        poses = [_tilted(rng, 20.0) for _ in range(min(num_poses, 64))]
        pi = (rng.randint(0, len(poses), n) if per_point else np.zeros(n)).astype(np.int32)
        d = rng.normal(size=(n, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        hits = (origins[oi] + d * rng.uniform(0.0, 45.0, (n, 1))).astype(np.float32)
        _accumulate(slam, hits, origins, oi, poses, pi)
        want = O.accumulate(hits, origins, oi, poses, pi, 0.3, 30.0, 5.0) if n < 5000 else \
            K.accumulate(hits, origins, oi, poses, pi, 0.3, 30.0, 5.0)
        _check_accumulated(slam, *want)
        slam.close()


def _range32(hit, origin, pose):
    """The float32 range the restatement computes for one hit."""
    o = L.rigid3f_apply(pose, origin)
    p = L.rigid3f_apply(pose, hit)
    dd = [p[k] - o[k] for k in range(3)]
    return F(np.sqrt((dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2]))


def _hits_at_range(target, origin, pose, rng):
    """Hits whose float32 range is exactly `target` and one ulp below and above it, found by
    stepping a hit's coordinates one ulp at a time along seeded directions."""
    target = F(target)
    wanted = {np.nextafter(target, F(-1)): None, target: None, np.nextafter(target, F(1e9)): None}
    for _ in range(50):
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        base = (np.asarray(origin, np.float64) + d * float(target)).astype(F)
        for k in range(-300, 301):
            for axis in range(3):
                h = base.copy()
                h[axis] = h[axis] + F(k) * np.spacing(h[axis])
                r = _range32(h, origin, pose)
                if r in wanted and wanted[r] is None:
                    wanted[r] = h
        if all(v is not None for v in wanted.values()):
            return [wanted[r] for r in sorted(wanted)]
    raise AssertionError(wanted)


def test_accumulate_range_edges_zero_ranges_and_signed_zeros():
    rng = np.random.RandomState(3)
    min_range, max_range = 0.25, 30.0
    origins = np.array([[0.1, -0.2, 0.05], [-0.0, 0.0, -0.0], [1e3, -2e3, 5.0]], np.float32)
    poses = [_tilted(rng, 5.0), L.rigid3f((-0.0, 0.0, -0.0), (1.0, 0.0, -0.0, 0.0)),
             _tilted(rng, 5e3), _tilted(rng, 1e4)]
    hits, oi, pi = [], [], []
    for p in range(len(poses)):
        for o in range(len(origins)):
            if p < 2 and o < 2:    # exact thresholds are reachable near the origin only
                for target in (min_range, max_range):
                    for h in _hits_at_range(target, origins[o], poses[p], rng):
                        hits.append(h)
                        oi.append(o)
                        pi.append(p)
            d = rng.normal(size=(20, 3))     # 10^3 to 10^4 m coordinates around the thresholds
            d /= np.linalg.norm(d, axis=1, keepdims=True)
            for h in origins[o] + d * rng.choice([min_range, max_range], (20, 1)):
                hits.append(h.astype(np.float32))
                oi.append(o)
                pi.append(p)
            hits.append(origins[o].copy())            # zero range
            oi.append(o)
            pi.append(p)
            hits.append(np.array([-0.0, 3.0, -0.0], np.float32))
            oi.append(o)
            pi.append(p)
    hits = np.array(hits, np.float32)
    oi, pi = np.array(oi, np.int32), np.array(pi, np.int32)
    for mn, ray in ((min_range, 5.0), (0.0, 5.0), (min_range, 1e6), (0.0, 3e4)):
        o = _opts(min_range=mn, max_range=max_range, missing_data_ray_length=ray)
        slam = L.LocalSlam2D(o)
        _accumulate(slam, hits, origins, oi, poses, pi)
        want = O.accumulate(hits, origins, oi, poses, pi, mn, max_range, ray)
        _check_accumulated(slam, *want)
        if mn == 0.0:        # the zero-range hits are kept as returns at their origin
            assert len(want[0]) > len(O.accumulate(hits, origins, oi, poses, pi, 1e-30,
                                                   max_range, ray)[0])
        slam.close()


# ---- b. accumulation across calls ----
def _scan(rng, n, kind, origins):
    oi = rng.randint(0, len(origins), n).astype(np.int32)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    lo, hi = {"returns": (1.0, 25.0), "misses": (35.0, 80.0), "mixed": (0.0, 45.0)}[kind]
    hits = (origins[oi] + d * rng.uniform(lo, hi, (n, 1))).astype(np.float32)
    return hits, oi


@pytest.mark.parametrize("sizes", [
    [(1, "returns"), (100000, "mixed"), (7, "misses")],
    [(1, "misses"), (100000, "mixed"), (7, "returns"), (300000, "mixed"), (2, "misses")],
])
def test_accumulation_grows_while_not_fresh(sizes):
    rng = np.random.RandomState(len(sizes))
    o = _opts(min_range=0.2, num_accumulated_range_data=len(sizes))
    slam = L.LocalSlam2D(o)
    origins = rng.uniform(-0.3, 0.3, (5, 3)).astype(np.float32)
    for round_ in range(2):
        want_r, want_m = [], []
        for n, kind in sizes:
            hits, oi = _scan(rng, n, kind, origins)
            poses = [_tilted(rng, 3.0) for _ in range(4)]
            pi = rng.randint(0, 4, n).astype(np.int32)
            flat = _flat(poses)
            slam.accumulate(hits, origins, oi, flat, pi)
            r, m = K.accumulate(hits, origins, oi, poses, pi, 0.2, 30.0, 5.0)
            want_r.append(r)
            want_m.append(m)
            hits[:] = np.nan       # the caller reuses its arrays at once
            oi[:] = -1
            flat[:] = np.nan
            pi[:] = -1
            del hits, oi, flat, pi
            gc.collect()
        _check_accumulated(slam, np.concatenate(want_r), np.concatenate(want_m))
        T = L.rigid3f((0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))
        if round_ == 0:           # a dropped match: every return cropped away
            tg = L.rigid3f((0.0, 0.0, 100.0), (1.0, 0.0, 0.0, 0.0))
            res, st = slam.match(L._flat(tg), (0, 0, 0), (0, 0, 0), None)
            assert res.status == L.DROPPED_EMPTY_RETURNS and st["host_syncs"] == 1
            assert len(slam.read(L.ACCUMULATED_RETURNS)) == 0
        else:
            res, _ = slam.match(L._flat(T), (0, 0, 0), (0, 0, 0), None)
            assert res.status == L.MATCHED
            assert _bits(slam.read(L.CROPPED_RETURNS),
                         O.crop(np.concatenate(want_r), o.min_z, o.max_z))
            assert _bits(slam.read(L.CROPPED_MISSES),
                         O.crop(np.concatenate(want_m), o.min_z, o.max_z))
    # an accumulation after a match starts fresh, and its crop sees only its own points
    hits, oi = _scan(rng, 10, "mixed", origins)
    slam.accumulate(hits, origins, oi, _flat([IDENT]), np.zeros(10, np.int32))
    r, m = O.accumulate(hits, origins, oi, [IDENT], [0] * 10, 0.2, 30.0, 5.0)
    _check_accumulated(slam, r, m)
    res, _ = slam.match(L._flat(IDENT), (0, 0, 0), (0, 0, 0), None)
    assert _bits(slam.read(L.CROPPED_RETURNS), O.crop(r, -0.8, 2.0))
    assert _bits(slam.read(L.CROPPED_MISSES), O.crop(m, -0.8, 2.0))
    slam.close()


# ---- c. the gravity crop ----
def _points_at_z(T, z, rng):
    """Points whose z after T is exactly z and one ulp either side (searched an ulp at a
    time around seeded points of the accumulation frame)."""
    z = F(z)
    wanted = {np.nextafter(z, F(-1e9)): None, z: None, np.nextafter(z, F(1e9)): None}
    Tinv = L.rigid3f_inverse(T)
    for _ in range(50):
        xy = rng.uniform(-2.0, 2.0, 2)
        base = np.array(L.rigid3f_apply(Tinv, (F(xy[0]), F(xy[1]), z)), np.float32)
        for k in range(-300, 301):
            for axis in (2, 0, 1):
                p = base.copy()
                p[axis] = p[axis] + F(k) * np.spacing(p[axis])
                got = L.rigid3f_apply(T, p)[2]
                if got in wanted and wanted[got] is None:
                    wanted[got] = p
        if all(v is not None for v in wanted.values()):
            return [wanted[v] for v in sorted(wanted)]
    raise AssertionError(wanted)


def test_gravity_crop_edges():
    rng = np.random.RandomState(5)
    o = _opts(min_range=0.0, max_range=1e4, min_z=-0.8, max_z=2.0)
    slam = L.LocalSlam2D(o)
    T = _tilted(rng, 2.0, roll=0.2, pitch=0.2)
    pts = []
    for _ in range(4):
        pts += _points_at_z(T, -0.8, rng) + _points_at_z(T, 2.0, rng)
    pts = np.array(pts, np.float32)
    # a first, larger scan leaves stale entries past the next scan's counts
    big = rng.uniform(-10, 10, (5000, 3)).astype(np.float32)
    slam.accumulate(big, np.zeros((1, 3), np.float32), np.zeros(5000, np.int32),
                    _flat([IDENT]), np.zeros(5000, np.int32))
    slam.match(L._flat(IDENT), (0, 0, 0), (0, 0, 0), None)
    # misses whose placed point goes in and out of the crop one at a time
    o2 = _opts(min_range=0.0, max_range=30.0, min_z=-0.8, max_z=2.0)
    slam2 = L.LocalSlam2D(o2)
    for s in (slam, slam2):
        s.accumulate(big[:100], np.zeros((1, 3), np.float32), np.zeros(100, np.int32),
                     _flat([IDENT]), np.zeros(100, np.int32))
        s.match(L._flat(IDENT), (0, 0, 0), (0, 0, 0), None)
    n = len(pts)
    slam.accumulate(pts, np.zeros((1, 3), np.float32), np.zeros(n, np.int32), _flat([IDENT]),
                    np.zeros(n, np.int32))
    r, m = O.accumulate(pts, [[0, 0, 0]], [0] * n, [IDENT], [0] * n, 0.0, 1e4, 5.0)
    assert len(m) == 0
    res, _ = slam.match(L._flat(T), (0, 0, 0), (0, 0, 0), None)
    want = O.crop(O.transform(r, T), -0.8, 2.0)
    assert len(want) == 2 * n // 3
    assert _bits(slam.read(L.CROPPED_RETURNS), want)
    assert len(slam.read(L.CROPPED_MISSES)) == 0                       # no misses at all
    # misses alternately in and out of the crop, behind a few returns
    k = 40
    z = np.where(np.arange(k) % 2 == 0, 0.5, 40.0)
    hits = np.stack([rng.uniform(-100, 100, k), rng.uniform(-100, 100, k), z * 10], 1)
    hits = np.vstack([hits, [[1, 0, 0], [0, 1, 0.5]]]).astype(np.float32)
    oi = np.zeros(len(hits), np.int32)
    slam2.accumulate(hits, np.zeros((1, 3), np.float32), oi, _flat([IDENT]), oi)
    r, m = O.accumulate(hits, [[0, 0, 0]], oi, [IDENT], oi, 0.0, 30.0, 5.0)
    res, _ = slam2.match(L._flat(T), (0, 0, 0), (0, 0, 0), None)
    wm = O.crop(O.transform(m, T), -0.8, 2.0)
    assert 0 < len(wm) < len(m)
    assert _bits(slam2.read(L.CROPPED_MISSES), wm)
    assert _bits(slam2.read(L.CROPPED_RETURNS), O.crop(O.transform(r, T), -0.8, 2.0))
    # no returns left: dropped, with empty hooks and nothing to insert
    hits = np.float32([[1.0, 0.0, 10.0], [0.0, -3.0, 9.0], [100.0, 0.0, 0.0], [0.0, 90.0, 1.0],
                       [50.0, 50.0, 300.0]])      # returns above max_z; misses in and out
    oi = np.zeros(len(hits), np.int32)
    slam2.accumulate(hits, np.zeros((1, 3), np.float32), oi, _flat([IDENT]), oi)
    r, m = O.accumulate(hits, [[0, 0, 0]], oi, [IDENT], oi, 0.0, 30.0, 5.0)
    res, st = slam2.match(L._flat(T), (0, 0, 0), (0, 0, 0), None)
    assert res.status == L.DROPPED_EMPTY_RETURNS and st["host_syncs"] == 1
    assert len(slam2.read(L.CROPPED_RETURNS)) == 0
    wm = O.crop(O.transform(m, T), -0.8, 2.0)
    assert len(wm) == 2 and _bits(slam2.read(L.CROPPED_MISSES), wm)
    for which in (L.FILTERED_RETURNS, L.FILTERED_MISSES, L.FILTERED, L.LOCAL_RETURNS,
                  L.LOCAL_MISSES, L.ACCUMULATED_RETURNS, L.ACCUMULATED_MISSES):
        assert len(slam2.read(which)) == 0
    g = sm.RealTimeGrid2D.empty(*sm.create_grid_limits((0, 0), 0.05))
    with pytest.raises(CsmError):
        slam2.insert(L._flat(L.embed3d_f((0.0, 0.0, 0.0))), [g])
    g.close()
    slam.close()
    slam2.close()


# ---- d. the filters through the mask ----
def _filter_case(returns, misses, voxel, adaptive):
    """Accumulates returns (identity pose, origin 0) and misses, matches without a grid and
    checks FILTERED_RETURNS, FILTERED_MISSES and FILTERED index for index.  -> the result and
    the adaptive filter's stats."""
    o = _opts(min_range=0.0, max_range=100.0, min_z=-1e6, max_z=1e6, voxel_filter_size=voxel,
              missing_data_ray_length=5.0)
    o.adaptive_voxel_filter_options = sensor.AdaptiveVoxelFilterOptions(*adaptive)
    slam = L.LocalSlam2D(o)
    hits = np.vstack([returns, misses]).astype(np.float32)
    n = len(hits)
    z = np.zeros(n, np.int32)
    slam.accumulate(hits, np.zeros((1, 3), np.float32), z, _flat([IDENT]), z)
    res, st = slam.match(L._flat(IDENT), (0, 0, 0), (1.0, 2.0, 0.3), None)
    r, m = K.accumulate(hits, [[0, 0, 0]], z, [IDENT], z, 0.0, 100.0, 5.0)
    cr, cm = K.transform(r, IDENT), K.transform(m, IDENT)
    assert _bits(slam.read(L.CROPPED_RETURNS), cr)
    kr, km, ka, ast = K.filters(cr, cm, o)
    assert _bits(slam.read(L.FILTERED_RETURNS), cr[kr])
    assert _bits(slam.read(L.FILTERED_MISSES), cm[km])
    assert _bits(slam.read(L.FILTERED), cr[kr][ka])
    assert (res.num_returns, res.num_misses, res.num_filtered) == (len(kr), len(km), len(ka))
    want_status = L.MATCHED if len(ka) else L.DROPPED_EMPTY_FILTERED
    assert res.status == want_status and st["host_syncs"] == 2
    if want_status == L.MATCHED:
        assert np.array_equal(np.array(res.pose_estimate[:]), [1.0, 2.0, 0.3])
    slam.close()
    return res, ast, len(kr), len(cr)


def _dup_cloud(rng, n, spread, copies=3):
    """n distinct returns, each repeated `copies` times in shuffled order: the voxel filter
    keeps one of each, and masks the rest out of the adaptive filter."""
    base = rng.uniform(-spread, spread, (n, 3)).astype(np.float32)
    base[:, 2] *= 0.05
    cloud = np.repeat(base, copies, 0)
    return cloud[rng.permutation(len(cloud))]


def test_filters_through_the_mask_branch_by_branch():
    rng = np.random.RandomState(9)
    misses = np.tile(np.float32([[160.0, 0, 0]]), (5, 1))
    misses = np.vstack([misses, rng.uniform(120, 200, (50, 3))]).astype(np.float32)
    seen = {}
    # at most min_num_points kept: the range-filtered cloud (the mask is all that filters)
    _, seen["early"], nk, nc = _filter_case(_dup_cloud(rng, 150, 10.0), misses, 0.025,
                                            (0.5, 200.0, 50.0))
    assert seen["early"]["trials"] == 0 and nk < nc
    # max_length is enough
    _, seen["enough"], _, _ = _filter_case(_dup_cloud(rng, 2000, 15.0), misses, 0.025,
                                           (0.5, 200.0, 50.0))
    assert seen["enough"]["trials"] == 1
    # halving, then the bisection
    _, seen["bisection"], _, _ = _filter_case(_dup_cloud(rng, 3000, 3.0), misses, 0.01,
                                              (8.0, 900.0, 50.0))
    assert seen["bisection"]["trials"] > 3
    # the give-up path: more points than min_num_points, never that many voxels
    g = np.stack(np.meshgrid(np.arange(30), np.arange(30), [0], indexing="ij"), -1)
    grid = (g.reshape(-1, 3) * 1e-3).astype(np.float32)
    _, seen["give up"], nk, _ = _filter_case(np.repeat(grid, 2, 0), misses, 1e-4,
                                             (0.5, 800.0, 50.0))
    assert seen["give up"]["length"] == np.float32(0.5) / 128 and nk == 900
    # max_range cuts kept points
    cloud = _dup_cloud(rng, 400, 30.0)
    res, _, _, _ = _filter_case(cloud, misses, 0.025, (0.5, 1000.0, 20.0))
    assert 0 < res.num_filtered < res.num_returns
    # nothing within max_range: DROPPED_EMPTY_FILTERED
    far = _dup_cloud(rng, 100, 10.0) + np.float32([60.0, 0.0, 0.0])
    res, _, _, _ = _filter_case(far, misses, 0.025, (0.5, 200.0, 20.0))
    assert res.status == L.DROPPED_EMPTY_FILTERED


def _rejections(k_max):
    """Rejections of uniform_int_distribution(1, k) for k = 2 .. k_max on one minstd_rand0
    stream (the adaptive filter's draws in a single voxel)."""
    raw = VO.generator(4 * k_max)
    pos = rejected = 0
    for k in range(2, k_max + 1):
        _, used = VO.uniform(k, raw[pos:pos + 64])
        pos += used
        rejected += used - 1
    return rejected


def test_single_voxel_rejections_under_the_mask():
    """~3e5 distinct returns plus masked duplicates in one max_length voxel: the adaptive
    filter's draws reject (checked on the CPU stream first), and the masked points draw
    nothing.  Then 3e5 returns in one voxel of the first, unmasked filter."""
    rng = np.random.RandomState(21)
    n = 300000
    assert _rejections(n) >= 10
    base = rng.uniform(0.0, 0.2, (n, 3)).astype(np.float32)
    dup = base[rng.randint(0, n, 60000)]
    cloud = np.vstack([base, dup])[rng.permutation(n + 60000)]
    misses = np.float32([[180.0, 0.0, 0.0]])
    _, st, nk, nc = _filter_case(cloud, misses, 1e-4, (1.0, 400000.0, 50.0))
    assert nc == n + 60000 and n - 100 < nk < n + 1 and st["trials"] == 0
    _, st, nk, _ = _filter_case(cloud, misses, 1e-4, (1.0, 100.0, 50.0))
    assert st["trials"] > 1 and nk == n - 5     # the first trial: one voxel of every point
    res, _, nk, _ = _filter_case(base, misses, 2.0, (0.5, 200.0, 50.0))
    assert nk == 1 and VO.voxel_filter(base, 2.0)[1]["rejections"] >= 10


# ---- e. the match ----
@pytest.fixture(scope="module")
def world():
    spec, occ = synthetic.make_grid2d(3, size_cells=600)
    poses = trajectory(occ, spec, np.random.RandomState(4), 12)
    return spec, occ, poses


@pytest.mark.parametrize("online", [False, True])
def test_match_against_the_oracle(oracle, world, online):
    spec, occ, poses = world
    o = _opts(min_range=0.2, use_online_correlative_scan_matching=online)
    slam = L.LocalSlam2D(o)
    grid = sm.RealTimeGrid2D(spec)
    og = oracle.Grid2D(spec.cells, spec.resolution, spec.max_x, spec.max_y)
    rng = np.random.RandomState(2)
    for k, pose in enumerate(poses[:6]):
        pts = synthetic.cast_scan(occ, spec, pose, beams=541, max_range=30.0, seed=k)
        pts[:, 2] = rng.uniform(-1.0, 2.5, len(pts))
        n = len(pts)
        z = np.zeros(n, np.int32)
        slam.accumulate(pts, np.zeros((1, 3), np.float32), z, _flat([IDENT]), z)
        pred = np.asarray(pose, np.float64) + rng.uniform(-0.05, 0.05, 3)
        r, m = K.accumulate(pts, [[0, 0, 0]], z, [IDENT], z, 0.2, 30.0, 5.0)
        cr, cm = O.crop(K.transform(r, IDENT), -0.8, 2.0), O.crop(K.transform(m, IDENT), -0.8, 2.0)
        kr, km, ka, _ = K.filters(cr, cm, o)
        filtered = cr[kr][ka]
        if k == 0:
            res, st = slam.match(L._flat(IDENT), (0, 0, 0), pred, None)
            assert res.matched_submap == 0 and st["host_syncs"] == 2
            assert np.array(res.pose_estimate[:]).tobytes() == pred.tobytes()
        else:
            res, st = slam.match(L._flat(IDENT), (0, 0, 0), pred, grid)
            assert res.matched_submap == 1 and st["host_syncs"] == 3 + online
            initial = pred
            if online:
                ro = o.real_time_correlative_scan_matcher_options
                rt = oracle.rt2d_match(og, filtered, pred, ro.linear_search_window,
                                       ro.angular_search_window, ro.translation_delta_cost_weight,
                                       ro.rotation_delta_cost_weight)
                assert np.float32(res.rt_score) == np.float32(rt["score"])
                initial = rt["pose"]
            c = o.ceres_scan_matcher_options
            ceres = oracle.ceres2d_match(og, filtered, pred[:2], initial, c.occupied_space_weight,
                                         c.translation_weight, c.rotation_weight,
                                         c.use_nonmonotonic_steps, c.max_num_iterations)
            got = np.array(res.pose_estimate[:])
            assert np.abs(got - ceres["pose"]).max() <= 1e-7
            assert res.ceres.iterations == ceres["iterations"]
            assert sm.CERES_TERMINATION[res.ceres.termination] == ceres["termination"]
            # the real-time pose is where the refinement starts
            assert res.ceres.initial_cost == pytest.approx(ceres["initial_cost"], rel=1e-9)
        assert res.status == L.MATCHED
        assert (res.num_returns, res.num_misses, res.num_filtered) == (len(kr), len(km), len(ka))
        assert _bits(slam.read(L.FILTERED), filtered)
    grid.close()
    slam.close()


# ---- f. the insert ----
def _insert_case(returns, misses, pose2d, grids_origins, free_space=True, resolution=0.05):
    """Matches (no grid) and inserts returns / misses (identity accumulation and gravity) into
    fresh grids at `grids_origins`, against the oracle inserter."""
    o = _opts(min_range=0.0, max_range=100.0, min_z=-1e6, max_z=1e6, voxel_filter_size=1e-6,
              missing_data_ray_length=5.0)
    o.adaptive_voxel_filter_options = sensor.AdaptiveVoxelFilterOptions(0.5, 1e9, 1e9)
    o.submaps_options = sm.SubmapsOptions2D(
        resolution=resolution,
        probability_grid_range_data_inserter_options=sm.ProbabilityGridRangeDataInserterOptions2D(
            0.55, 0.49, free_space))
    slam = L.LocalSlam2D(o)
    hits = np.vstack([returns, misses]).astype(np.float32)
    n = len(hits)
    z = np.zeros(n, np.int32)
    origin = np.float32([0.0, 0.0, 0.0])
    slam.accumulate(hits, origin[None], z, _flat([IDENT]), z)
    res, _ = slam.match(L._flat(IDENT), origin, (0.0, 0.0, 0.0), None)
    assert res.status == L.MATCHED
    vr, vm = slam.read(L.FILTERED_RETURNS), slam.read(L.FILTERED_MISSES)
    pose3f = L.embed3d_f(pose2d)
    grids, oras = [], []
    for go in grids_origins:
        grids.append(sm.RealTimeGrid2D.empty(*sm.create_grid_limits(go, resolution)))
        oras.append(I.Grid.create_grid(go, resolution))
    org, st = slam.insert(L._flat(pose3f), grids)
    assert st["host_syncs"] == 2
    want_org = np.array(L.rigid3f_apply(pose3f, L.rigid3f_apply(IDENT, origin)), np.float32)
    assert org.tobytes() == want_org.tobytes()
    lr, lm = K.transform(vr, pose3f), K.transform(vm, pose3f)
    assert _bits(slam.read(L.LOCAL_RETURNS), lr) and _bits(slam.read(L.LOCAL_MISSES), lm)
    ins = I.Inserter(0.55, 0.49, free_space)
    for g, og in zip(grids, oras):
        ins.insert(want_org, lr, og, lm)
        s = g.read()
        assert (s.resolution, s.max_x, s.max_y) == og.limits[:3]
        assert s.known_cells_box == og.known_box
        np.testing.assert_array_equal(s.cells, og.cells)
        g.close()
    slam.close()
    return lr, lm, oras


def _far(rng, n):
    """Hits beyond max_range in every direction: misses 5 m out."""
    d = rng.normal(size=(n, 3))
    d[:, 2] *= 0.1
    return (d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(120, 200, (n, 1))
            ).astype(np.float32)


def test_insert_cell_borders_limits_and_signed_zero_box():
    res = 0.05
    lim = sm.create_grid_limits((0.0, 0.0), res)
    max_x, max_y = F(lim[1]), F(lim[2])
    k = np.arange(-40, 41, dtype=np.float32)
    border = np.stack([k * F(res), k[::-1] * F(res), np.zeros_like(k)], 1)   # cell borders
    limits = np.float32([[max_x, max_y, 0], [max_x, 0, 0], [0, max_y, 0],
                         [np.nextafter(max_x, F(0)), max_y, 0]])
    for zero in (F(0.0), F(-0.0)):
        # every x >= 0, so the box's min x is the signed zero itself
        pts = np.vstack([border[border[:, 0] >= 0], limits,
                         np.float32([[zero, 1.0, 0], [zero, -1.0, 0]])])
        for ident in ((0.0, 0.0, 0.0), (-0.0, -0.0, -0.0)):
            lr, _, _ = _insert_case(pts, np.zeros((0, 3), np.float32), ident, [(0, 0)])
            # Embed3D adds the translation to a rotated +0.0, so a -0.0 input reaches the
            # box as +0.0
            assert lr[:, 0].min() == 0.0 and not np.signbit(lr[lr[:, 0] == 0, 0]).any()
    # one and two handles, misses and returns on both signs
    rng = np.random.RandomState(1)
    r = rng.uniform(-2.4, 2.4, (300, 3)).astype(np.float32)
    m = _far(rng, 100)
    _insert_case(r, m, (0.3, -0.2, 0.4), [(0, 0)])
    _insert_case(r, m, (0.3, -0.2, 0.4), [(0, 0), (1.0, -1.5)])
    _insert_case(r, m, (0.3, -0.2, 0.4), [(0, 0), (1.0, -1.5)], free_space=False)


@pytest.mark.parametrize("side", ["-x", "+x", "-y", "+y", "all"])
def test_insert_growth_on_every_side(side):
    rng = np.random.RandomState(len(side))
    far = {"-x": (-40.0, 0.0), "+x": (40.0, 0.0), "-y": (0.0, -40.0), "+y": (0.0, 40.0)}
    ends = [far[side]] if side != "all" else list(far.values())
    r = [rng.uniform(-1, 1, (50, 3))]
    for e in ends:   # 40 m from a 5 m grid: several doublings in one insert
        r.append(np.float32([[e[0], e[1], 0.0]]) + rng.uniform(-0.5, 0.5, (20, 3)))
    r = np.vstack(r).astype(np.float32)
    r[:, 2] = 0.0
    m = np.zeros((0, 3), np.float32)
    _, _, oras = _insert_case(r, m, (0.1, 0.2, -0.3), [(0, 0), (0.5, 0.5)])
    assert oras[0].limits[3] >= 800 or oras[0].limits[4] >= 800


def test_insert_one_return_and_misses():
    rng = np.random.RandomState(4)
    m = _far(rng, 200)
    _insert_case(np.float32([[0.5, 0.5, 0.0]]), m, (-0.2, 0.1, 1.0), [(0, 0), (0.3, 0.3)])
    _insert_case(np.float32([[0.5, 0.5, 0.0]]), m, (-0.2, 0.1, 1.0), [(0, 0)], free_space=False)


# ---- g. a long run on the chain ----
def _assert_grid(dev, ora):
    s = dev.read()
    assert (s.resolution, s.max_x, s.max_y) == ora.limits[:3]
    assert s.known_cells_box == ora.known_box
    np.testing.assert_array_equal(s.cells, ora.cells)


@pytest.mark.parametrize("online,accumulate", [(False, 1), (True, 1), (False, 3), (True, 3)])
def test_long_run_against_the_chain(oracle, online, accumulate):
    n_scans = 300
    spec, occ = synthetic.make_grid2d(3, size_cells=1000)
    traj = trajectory(occ, spec, np.random.RandomState(11), n_scans + 2)
    o = _opts(min_range=0.2, num_accumulated_range_data=accumulate,
              use_online_correlative_scan_matching=online)
    o.submaps_options = sm.SubmapsOptions2D(num_range_data=12)
    o.motion_filter_options = L.MotionFilterOptions(0.0, 0.0, 0.0)   # every scan is inserted
    ex_b, ex_c = K.TiltedExtrapolator(traj), K.TiltedExtrapolator(traj)
    b = L.LocalTrajectoryBuilder2D(o, ex_b)
    chain = K.Chain(o, ex_c, oracle)
    seen = []
    match = b.slam.match
    b.slam.match = lambda *a: (seen.append(np.array(a[2], np.float64)), match(*a))[1]
    origins = np.float32([[0.0, 0.0, 0.0], [0.05, -0.02, 0.1], [-0.03, 0.04, -0.05]])
    rng = np.random.RandomState(8)
    matched = finished = 0
    for k in range(n_scans):
        time = (k + 1) * 0.1
        pts = synthetic.cast_scan(occ, spec, traj[k + 1], beams=361, max_range=30.0, seed=k)
        pts[:, 2] = rng.uniform(-1.2, 2.6, len(pts))
        t = np.linspace(-0.05, 0.0, len(pts), dtype=np.float32)
        t[rng.rand(len(t)) < 0.1] = np.float32(-0.05)          # repeated and unsorted times
        t[-1] = 0.0
        hw = np.concatenate([pts.astype(np.float32), t[:, None]], 1)
        oi = rng.randint(0, 3, len(hw)).astype(np.int32)
        seen.clear()
        got = b.AddRangeData(time, hw, origins, oi)
        want = chain.add(time, hw, origins, oi)
        if want["status"] is None:
            assert got is None
            _check_accumulated(b.slam, want["accumulated_returns"], want["accumulated_misses"])
            continue
        assert _bits(b.slam.read(L.CROPPED_RETURNS), want["cropped_returns"])
        assert _bits(b.slam.read(L.CROPPED_MISSES), want["cropped_misses"])
        if want["status"] != "matched":
            assert got is None
            continue
        matched += 1
        assert got is not None
        assert _bits(b.slam.read(L.FILTERED_RETURNS), want["filtered_returns"])
        assert _bits(b.slam.read(L.FILTERED_MISSES), want["filtered_misses"])
        assert _bits(b.slam.read(L.FILTERED), want["filtered"])
        (pred,) = seen
        assert np.abs(pred - want["prediction"]).max() <= 1e-12
        rt, ceres = K.match(oracle, o, want["grid"], want["filtered"], pred)
        if ceres is None:
            assert got.pose_estimate_2d.tobytes() == pred.tobytes()
        else:
            assert np.abs(got.pose_estimate_2d - ceres["pose"]).max() <= 1e-7
            assert got.ceres_summary["iterations"] == ceres["iterations"]
            assert got.ceres_summary["termination"] == ceres["termination"]
            if rt is not None:
                assert np.float32(got.rt_score) == np.float32(rt["score"])
        chain.finish(want, L.embed3d_f(got.pose_estimate_2d))
        assert got.insertion_result is not None
        assert np.array(got.range_data_in_local_origin, np.float32).tobytes() == \
            want["local_origin"].tobytes()
        assert _bits(b.slam.read(L.LOCAL_RETURNS), want["local_returns"])
        assert _bits(b.slam.read(L.LOCAL_MISSES), want["local_misses"])
        subs = b.active_submaps.submaps()
        assert len(subs) == len(chain.submaps.submaps)
        for s, c in zip(subs, chain.submaps.submaps):
            assert (s.num_range_data, s.insertion_finished) == (c.num_range_data,
                                                                 c.insertion_finished)
            assert s.local_pose == c.local_pose
            _assert_grid(s.grid, c.grid)
        finished += want["event"]["finished"] is not None
    assert matched >= n_scans // accumulate - 2 and finished >= 2
    b.close()
