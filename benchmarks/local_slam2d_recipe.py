"""The recipe for 2D local SLAM: the same scans pushed through the existing single-stage public
calls (voxel_filter_batch, adaptive_voxel_filter_batch, RealTimeCorrelativeScanMatcher2D
.MatchBatch, CeresScanMatcher2D.Match, MotionFilter, ActiveSubmaps2D.InsertRangeData), with the
per-point transforms in vectorised float32 numpy in the reference's operation order.  Shared by
tests/test_gpu_local_slam2d.py, benchmarks/bench_local_slam2d.py and smoke()."""
import math

import numpy as np

from benchmarks import synthetic
from benchmarks.bench_insert2d import trajectory
from cartographer_b200 import local_slam as L
from cartographer_b200 import scan_matching as sm
from cartographer_b200 import sensor

F = np.float32


def _columns(p):
    p = np.asarray(p, np.float32).reshape(-1, 3)
    return (p[:, 0], p[:, 1], p[:, 2])


def transform(points, rigid):
    """TransformPointCloud: every point through one Rigid3f, elementwise as rigid3f.h does."""
    return np.stack(L.rigid3f_apply(rigid, _columns(points)), 1).astype(np.float32).reshape(-1, 3)


def crop(points, min_z, max_z):
    p = np.asarray(points, np.float32).reshape(-1, 3)
    return p[(F(min_z) <= p[:, 2]) & (p[:, 2] <= F(max_z))]


def accumulate(hits, origins, origin_index, poses, pose_index, min_range, max_range,
               missing_data_ray_length):
    """AddRangeData's loop (:163-186) over one scan, every point with its own pose."""
    pi = np.asarray(pose_index)
    t = [np.array([p[0][k] for p in poses], np.float32)[pi] for k in range(3)]
    q = [np.array([p[1][k] for p in poses], np.float32)[pi] for k in range(4)]
    o = np.asarray(origins, np.float32).reshape(-1, 3)[np.asarray(origin_index)]
    org = L.rigid3f_apply((t, q), _columns(o))
    hit = L.rigid3f_apply((t, q), _columns(hits))
    d = [hit[k] - org[k] for k in range(3)]
    rng = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]).astype(np.float32)
    keep = rng >= F(min_range)
    ret = keep & (rng <= F(max_range))
    mis = keep & ~(rng <= F(max_range))
    with np.errstate(divide="ignore", invalid="ignore"):
        s = F(missing_data_ray_length) / rng
    miss = [org[k] + s * d[k] for k in range(3)]
    returns = np.stack([hit[k][ret] for k in range(3)], 1).astype(np.float32).reshape(-1, 3)
    misses = np.stack([miss[k][mis] for k in range(3)], 1).astype(np.float32).reshape(-1, 3)
    return returns, misses


TILT = 0.01   # rad of roll between the tracking frame and gravity


def _quat_yaw(a):
    return (math.cos(a / 2), 0.0, 0.0, math.sin(a / 2))


class FakeExtrapolator:
    """Replays a trajectory: poses at times k * dt, linear in x, y and yaw between them, with
    a constant roll tilt that EstimateGravityOrientation undoes."""

    def __init__(self, poses, dt=0.1):
        self.poses, self.dt = poses, dt
        self.last_pose_time = -1e9
        self.last_extrapolated = -1e9
        self.added = []

    def _at(self, t):
        u = min(max(t / self.dt, 0.0), len(self.poses) - 1.0)
        k = min(int(u), len(self.poses) - 2)
        f = u - k
        a, b = self.poses[k], self.poses[k + 1]
        p = a + f * (b - a)
        tilt = (math.cos(TILT / 2), math.sin(TILT / 2), 0.0, 0.0)
        return ((float(p[0]), float(p[1]), 0.0), L._quatd_mul(_quat_yaw(float(p[2])), tilt))

    def ExtrapolatePose(self, t):
        self.last_extrapolated = max(self.last_extrapolated, t)
        return self._at(t)

    def EstimateGravityOrientation(self, t):
        return (math.cos(TILT / 2), -math.sin(TILT / 2), 0.0, 0.0)

    def AddPose(self, t, pose):
        self.last_pose_time = t
        self.added.append((t, pose))

    def GetLastPoseTime(self):
        return self.last_pose_time

    def GetLastExtrapolatedTime(self):
        return self.last_extrapolated


def world(n_scans, seed=11):
    spec, occ = synthetic.make_grid2d(3, size_cells=1000)
    rng = np.random.RandomState(seed)
    return spec, occ, trajectory(occ, spec, rng, n_scans + 2)


def scan_at(spec, occ, pose, seed, beams=1081):
    """One scan in the sensor frame with per-point times, the last point at 0."""
    pts = synthetic.cast_scan(occ, spec, pose, beams=beams, max_range=30.0, seed=seed)
    t = np.linspace(-0.05, 0.0, len(pts), dtype=np.float32)
    return np.concatenate([pts.astype(np.float32), t[:, None]], 1)


class Recipe:
    """The same builder glued from the existing public calls."""

    def __init__(self, options, extrapolator):
        self.o = options
        self.ex = extrapolator
        self.submaps = sm.ActiveSubmaps2D(options.submaps_options)
        self.mf = L.MotionFilter(options.motion_filter_options)
        self.rt = sm.RealTimeCorrelativeScanMatcher2D(
            options.real_time_correlative_scan_matcher_options)
        self.ceres = sm.CeresScanMatcher2D(options.ceres_scan_matcher_options)
        self.num = 0
        self.ret, self.mis = [], []
        self._poses = L.LocalTrajectoryBuilder2D._poses.__get__(self)
        self.extrapolator = extrapolator

    def add(self, time, hw, origins, oi):
        o = self.o
        table, _, index = self._poses(time, hw[:, 3])
        r, m = accumulate(hw[:, :3], origins, oi, table, index, o.min_range, o.max_range,
                          o.missing_data_ray_length)
        if self.num == 0:
            self.ret, self.mis = [], []
        self.ret.append(r)
        self.mis.append(m)
        self.num += 1
        if self.num < o.num_accumulated_range_data:
            return None
        self.num = 0
        gq = tuple(float(c) for c in self.ex.EstimateGravityOrientation(time))
        last = table[index[-1]]
        T = L.rigid3f_mul(((L.F(0),) * 3, tuple(L.F(c) for c in gq)), L.rigid3f_inverse(last))
        ret = crop(transform(np.concatenate(self.ret), T), o.min_z, o.max_z)
        mis = crop(transform(np.concatenate(self.mis), T), o.min_z, o.max_z)
        out = dict(ret=ret, mis=mis)
        if len(ret) == 0:
            out["status"] = L.DROPPED_EMPTY_RETURNS
            return out
        (kr, km), _ = sensor.voxel_filter_batch([ret, mis], o.voxel_filter_size)
        vret, vmis = ret[kr], mis[km]
        (ka,), _ = sensor.adaptive_voxel_filter_batch([vret], o.adaptive_voxel_filter_options)
        filtered = vret[ka]
        out.update(vret=vret, vmis=vmis, filtered=filtered)
        if len(filtered) == 0:
            out["status"] = L.DROPPED_EMPTY_FILTERED
            return out
        out["status"] = L.MATCHED
        gravity = ((0.0, 0.0, 0.0), gq)
        p3 = self.ex.ExtrapolatePose(time)
        pred = L.project2d(L.rigid3d_mul((tuple(p3[0]), tuple(p3[1])), L.rigid3d_inverse(gravity)))
        subs = self.submaps.submaps()
        pose2d = pred
        if subs:
            init = pred
            if o.use_online_correlative_scan_matching:
                _, poses, _ = self.rt.MatchBatch([pred], [filtered], subs[0].grid)
                init = poses[0]
            pose2d, summary = self.ceres.Match(pred[:2], init, filtered, subs[0].grid)
            out["summary"] = summary
        out["pose2d"] = np.asarray(pose2d, np.float64)
        pe = L.rigid3d_mul(L.embed3d(pose2d), gravity)
        self.ex.AddPose(time, pe)
        p3f = L.embed3d_f(pose2d)
        origin = np.array(L.rigid3f_apply(p3f, L.rigid3f_apply(T, last[0])), np.float32)
        out["similar"] = self.mf.IsSimilar(time, pe)
        if not out["similar"]:
            self.submaps.InsertRangeData(origin, transform(vret, p3f), transform(vmis, p3f))
        return out


def grids_equal(a, b):
    sa, sb = a.submaps(), b.submaps()
    assert len(sa) == len(sb)
    for x, y in zip(sa, sb):
        gx, gy = x.grid.read(), y.grid.read()
        assert np.array_equal(gx.cells, gy.cells)
        assert (gx.resolution, gx.max_x, gx.max_y) == (gy.resolution, gy.max_x, gy.max_y)
        assert gx.known_cells_box == gy.known_cells_box
        assert x.num_range_data == y.num_range_data
        assert x.insertion_finished == y.insertion_finished


def run(options, n_scans, tweak=None):
    """The builder and the recipe side by side over n_scans scans; every scan's result is
    checked equal (AssertionError otherwise).  -> (builder, matched, dropped, inserted)."""
    spec, occ, traj = world(n_scans)
    ex_a, ex_b = FakeExtrapolator(traj), FakeExtrapolator(traj)
    b = L.LocalTrajectoryBuilder2D(options, ex_a)
    rec = Recipe(options, ex_b)
    origins = np.zeros((1, 3), np.float32)
    matched = dropped = inserted = 0
    for k in range(n_scans):
        time = (k + 1) * 0.1
        hw = scan_at(spec, occ, traj[k + 1], seed=k)
        if tweak:
            hw = tweak(k, hw)
        oi = np.zeros(len(hw), np.int32)
        got = b.AddRangeData(time, hw, origins, oi)
        want = rec.add(time, hw, origins, oi)
        if want is None:
            assert got is None
            continue
        st = b.last_stats["match"]
        assert st["host_syncs"] <= 4
        if want["status"] != L.MATCHED:
            assert got is None
            dropped += 1
            assert np.array_equal(b.slam.read(L.CROPPED_RETURNS), want["ret"])
            continue
        matched += 1
        assert got is not None
        assert np.array_equal(got.pose_estimate_2d, want["pose2d"]), k
        assert np.array_equal(b.slam.read(L.FILTERED), want["filtered"])
        assert np.array_equal(b.slam.read(L.FILTERED_RETURNS), want["vret"])
        assert np.array_equal(b.slam.read(L.FILTERED_MISSES), want["vmis"])
        has_grid = "summary" in want
        expect_syncs = 2 + has_grid + (has_grid and options.use_online_correlative_scan_matching)
        assert st["host_syncs"] == expect_syncs
        if has_grid:
            assert got.ceres_summary == want["summary"]
        assert (got.insertion_result is None) == want["similar"]
        if not want["similar"]:
            inserted += 1
            assert b.last_stats["insert"]["host_syncs"] == 2
        grids_equal(b.active_submaps, rec.submaps)
    assert ex_a.added == ex_b.added
    return b, matched, dropped, inserted
