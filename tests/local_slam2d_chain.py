"""One scan of 2D local SLAM through the CPU references alone: the parity reference of the
device stages (tests/test_gpu_local_slam2d_stages.py).

Nothing here comes from the device or from local_slam.py's pose code.  The stages are

  range_data_poses      a float64 restatement of local_trajectory_builder_2d.cc:141-160, one
                        extrapolator call per point;
  accumulate / crop     tests/local_slam2d_oracle.py (float32, the reference's order), on
                        whole columns of points (checked equal to the scalar form);
  voxel filters         tests/voxel_filter_oracle.py;
  match                 oracle.pyoracle.rt2d_match and ceres2d_match;
  insert                tests/active_submaps2d_oracle.py over tests/insert2d_oracle.py.

Ceres parity is 1e-7, not bit for bit, so `Chain` takes the device's pose of each scan as the
pose it inserts with and carries forward, after the caller has checked it against the chain's.

The float64 functions (`geometry64`, `transform64`) restate the per-point geometry with rotation
matrices, so that the float32 restatement is checked against something that does not copy its
operation order.  F32_GEOMETRY_ULPS bounds their distance in float32 ulps of the largest
magnitude in play."""
import math

import numpy as np

from cartographer_b200.local_slam import rigid3f_apply, rigid3f_inverse, rigid3f_mul
from tests import active_submaps2d_oracle as A
from tests import local_slam2d_oracle as O
from tests import voxel_filter_oracle as VO

F = np.float32
F32_GEOMETRY_ULPS = 8


# ---- float64 geometry ----
def rotation64(q):
    """The matrix of v -> v + 2w (u x v) + 2 u x (u x v) (u = q.vec), the map Eigen's
    _transformVector evaluates, for any quaternion q = (w, x, y, z); a unit q gives its
    rotation matrix."""
    w, x, y, z = (float(c) for c in q)
    K = np.array([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]])
    return np.eye(3) + 2.0 * w * K + 2.0 * (K @ K)


def transform64(points, rigid):
    """Every point through rigid = (t(3), q(4)) in float64: R p + t."""
    t, q = rigid
    p = np.asarray(points, np.float64).reshape(-1, 3)
    return p @ rotation64(q).T + np.asarray(t, np.float64)


def ulp32(x):
    """The float32 ulp of |x| (elementwise), at least that of the smallest normal."""
    a = np.maximum(np.abs(np.asarray(x, np.float64)), np.finfo(np.float32).tiny)
    return np.spacing(a.astype(np.float32)).astype(np.float64)


def geometry64(hits, origins, origin_index, poses, pose_index, missing_data_ray_length):
    """AddRangeData's per-point geometry (:165-185) in float64: the hit and its origin in the
    tracking frame, the range and the miss point.  -> dict of hit, origin, range, miss and
    `scale`, each point's largest coordinate magnitude (the float32 ulp unit)."""
    hits = np.asarray(hits, np.float32).reshape(-1, 3)
    origins = np.asarray(origins, np.float32).reshape(-1, 3)
    n = len(hits)
    hit, org = np.zeros((n, 3)), np.zeros((n, 3))
    pi = np.asarray(pose_index)
    oi = np.asarray(origin_index)
    for k in np.unique(pi):
        sel = pi == k
        hit[sel] = transform64(hits[sel], poses[k])
        org[sel] = transform64(origins[oi[sel]], poses[k])
    d = hit - org
    rng = np.sqrt((d * d).sum(1))
    with np.errstate(divide="ignore", invalid="ignore"):
        miss = org + (float(F(missing_data_ray_length)) / rng)[:, None] * d
    t = np.array([np.abs(np.asarray(poses[k][0], np.float64)).max() for k in pi]).reshape(n)
    scale = np.maximum.reduce([np.abs(hit).max(1), np.abs(org).max(1), t,
                               np.abs(hits.astype(np.float64)).max(1),
                               np.abs(origins[oi].astype(np.float64)).max(1)])
    return dict(hit=hit, origin=org, range=rng, miss=miss, scale=scale)


# ---- range_data_poses ----
def range_data_poses(extrapolator, time, point_times):
    """local_trajectory_builder_2d.cc:141-160: for each point, its time clamped to
    GetLastExtrapolatedTime, ExtrapolatePose there, cast to float.  -> a list of (t, q)
    float32 tuples, one per point."""
    out = []
    for pt in np.asarray(point_times, np.float32).tolist():
        tp = time + pt
        last = extrapolator.GetLastExtrapolatedTime()
        if tp < last:
            tp = last
        t, q = extrapolator.ExtrapolatePose(tp)
        out.append((tuple(F(c) for c in t), tuple(F(c) for c in q)))
    return out


def quat_mul64(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return (w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
            w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2)


def prediction64(pose3d, gravity_q):
    """Project2D(pose * Rigid3d::Rotation(gravity).inverse()) (:197-200) in float64 with
    matrices: x, y and the yaw of the composed rotation applied to UnitX."""
    g = gravity_q
    inv = (g[0], -g[1], -g[2], -g[3])
    n2 = sum(c * c for c in g)
    R = rotation64(quat_mul64(pose3d[1], tuple(c / n2 for c in inv)))
    return np.array([pose3d[0][0], pose3d[0][1], math.atan2(R[1, 0], R[0, 0])])


def to_gravity64(gravity_q, last_pose):
    """gravity_alignment * range_data_poses.back().inverse() (:208-210) in float64: (R, t)."""
    Rg = rotation64(gravity_q)
    Rl = rotation64(last_pose[1])
    t = np.asarray(last_pose[0], np.float64)
    R = Rg @ Rl.T
    return R, -(R @ t)


# ---- the float32 restatement on whole columns (large clouds) ----
def _columns(points):
    p = np.asarray(points, np.float32).reshape(-1, 3)
    return (p[:, 0], p[:, 1], p[:, 2])


def accumulate(hits, origins, origin_index, poses, pose_index, min_range, max_range,
               missing_data_ray_length):
    """local_slam2d_oracle.accumulate with every scalar a column of points: the same float32
    operations in the same order, elementwise."""
    pi = np.asarray(pose_index)
    t = tuple(np.array([p[0][k] for p in poses], np.float32)[pi] for k in range(3))
    q = tuple(np.array([p[1][k] for p in poses], np.float32)[pi] for k in range(4))
    o = np.asarray(origins, np.float32).reshape(-1, 3)[np.asarray(origin_index)]
    with np.errstate(divide="ignore", invalid="ignore"):
        org = rigid3f_apply((t, q), _columns(o))
        hit = rigid3f_apply((t, q), _columns(hits))
        d = [hit[k] - org[k] for k in range(3)]
        rng = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]).astype(np.float32)
        keep = rng >= F(min_range)
        ret = keep & (rng <= F(max_range))
        mis = keep & ~(rng <= F(max_range))
        s = F(missing_data_ray_length) / rng
        miss = [org[k] + s * d[k] for k in range(3)]
    returns = np.stack([hit[k][ret] for k in range(3)], 1).astype(np.float32).reshape(-1, 3)
    misses = np.stack([miss[k][mis] for k in range(3)], 1).astype(np.float32).reshape(-1, 3)
    return returns, misses


def transform(points, rigid):
    """local_slam2d_oracle.transform on columns."""
    return np.stack(rigid3f_apply(rigid, _columns(points)), 1).astype(np.float32).reshape(-1, 3)


# ---- the per-scan chain ----
def filters(cropped_returns, cropped_misses, options):
    """VoxelFilter of both clouds and AdaptiveVoxelFilter of the filtered returns:
    (kept returns, kept misses, adaptive kept) indices and the adaptive filter's stats."""
    vs = float(F(options.voxel_filter_size))
    kr, _ = VO.voxel_filter(cropped_returns, vs)
    km, _ = VO.voxel_filter(cropped_misses, vs)
    a = options.adaptive_voxel_filter_options
    ka, st = VO.adaptive_voxel_filter(cropped_returns[kr], a.max_length, a.min_num_points,
                                      a.max_range)
    return kr, km, ka, st


def oracle_grid(pyoracle, grid):
    """The oracle's record of an insert2d_oracle.Grid (the cells the matchers read)."""
    res, max_x, max_y, _, _ = grid.limits
    return pyoracle.Grid2D(grid.cells, res, max_x, max_y)


def match(pyoracle, options, grid, filtered, prediction):
    """ScanMatch (:65-102) on the oracle: (real-time result or None, Ceres result), or
    (None, None) without a grid."""
    if grid is None:
        return None, None
    og = oracle_grid(pyoracle, grid)
    initial = np.asarray(prediction, np.float64)
    rt = None
    if options.use_online_correlative_scan_matching:
        r = options.real_time_correlative_scan_matcher_options
        rt = pyoracle.rt2d_match(og, filtered, prediction, r.linear_search_window,
                                 r.angular_search_window, r.translation_delta_cost_weight,
                                 r.rotation_delta_cost_weight)
        initial = rt["pose"]
    c = options.ceres_scan_matcher_options
    ceres = pyoracle.ceres2d_match(og, filtered, np.asarray(prediction)[:2], initial,
                                   c.occupied_space_weight, c.translation_weight,
                                   c.rotation_weight, c.use_nonmonotonic_steps,
                                   c.max_num_iterations)
    return rt, ceres


class Chain:
    """LocalTrajectoryBuilder2D's stages on the CPU references, scan by scan.  add() takes what
    the builder's AddRangeData takes; finish() the device's 2D pose of a matched scan."""

    def __init__(self, options, extrapolator, pyoracle):
        self.o = options
        self.ex = extrapolator
        self.pyoracle = pyoracle
        s = options.submaps_options
        ins = s.probability_grid_range_data_inserter_options
        self.submaps = A.ActiveSubmaps(s.num_range_data, s.resolution, ins.hit_probability,
                                       ins.miss_probability, ins.insert_free_space)
        self.num = 0
        self.returns, self.misses = [], []

    def add(self, time, hits_with_times, origins, origin_index):
        """-> None while accumulating, else a dict of every stage's expected output."""
        o = self.o
        hw = np.asarray(hits_with_times, np.float32).reshape(-1, 4)
        poses = range_data_poses(self.ex, time, hw[:, 3])
        r, m = accumulate(hw[:, :3], origins, origin_index, poses, np.arange(len(hw)),
                          o.min_range, o.max_range, o.missing_data_ray_length)
        if self.num == 0:
            self.returns, self.misses = [], []
        self.returns.append(r)
        self.misses.append(m)
        self.num += 1
        out = dict(accumulated_returns=np.concatenate(self.returns),
                   accumulated_misses=np.concatenate(self.misses))
        if self.num < o.num_accumulated_range_data:
            out["status"] = None
            return out
        self.num = 0
        gq = tuple(float(c) for c in self.ex.EstimateGravityOrientation(time))
        last = poses[-1]
        T = rigid3f_mul(((F(0), F(0), F(0)), tuple(F(c) for c in gq)), rigid3f_inverse(last))
        cr = O.crop(transform(out["accumulated_returns"], T), o.min_z, o.max_z)
        cm = O.crop(transform(out["accumulated_misses"], T), o.min_z, o.max_z)
        out.update(to_gravity=T, gravity=gq, cropped_returns=cr, cropped_misses=cm,
                   ga_origin=rigid3f_apply(T, last[0]))
        if len(cr) == 0:
            out["status"] = "dropped_empty_returns"
            return out
        kr, km, ka, _ = filters(cr, cm, o)
        vret, vmis = cr[kr], cm[km]
        out.update(filtered_returns=vret, filtered_misses=vmis, filtered=vret[ka])
        if len(ka) == 0:
            out["status"] = "dropped_empty_filtered"
            return out
        out["status"] = "matched"
        out["prediction"] = prediction64(self.ex.ExtrapolatePose(time), gq)
        subs = self.submaps.submaps
        out["grid"] = subs[0].grid if subs else None
        return out

    def finish(self, out, pose3f):
        """Inserts a matched scan with the device's Embed3D(pose) (float32 (t, q)): the local
        range data and origin, and the lifecycle event."""
        vret = transform(out["filtered_returns"], pose3f)
        vmis = transform(out["filtered_misses"], pose3f)
        origin = np.array(rigid3f_apply(pose3f, out["ga_origin"]), np.float32)
        out.update(local_returns=vret, local_misses=vmis, local_origin=origin)
        out["event"] = self.submaps.insert_range_data(origin, vret, vmis)
        return out


class TiltedExtrapolator:
    """Replays a trajectory as a PoseExtrapolator would: poses at times k * dt, linear in x, y
    and yaw between them, with a roll and a pitch tilt that EstimateGravityOrientation undoes
    and a z that moves with time.  GetLastExtrapolatedTime is the last ExtrapolatePose time."""

    def __init__(self, poses, dt=0.1, roll=0.03, pitch=-0.02, z=0.05):
        self.poses, self.dt = poses, dt
        self.roll, self.pitch, self.z = roll, pitch, z
        self.last_pose_time = -1e9
        self.last_extrapolated = -1e9
        self.added = []

    def _tilt(self):
        r = (math.cos(self.roll / 2), math.sin(self.roll / 2), 0.0, 0.0)
        p = (math.cos(self.pitch / 2), 0.0, math.sin(self.pitch / 2), 0.0)
        return quat_mul64(p, r)

    def ExtrapolatePose(self, t):
        self.last_extrapolated = t
        u = min(max(t / self.dt, 0.0), len(self.poses) - 1.0)
        k = min(int(u), len(self.poses) - 2)
        f = u - k
        a, b = self.poses[k], self.poses[k + 1]
        p = a + f * (b - a)
        yaw = float(p[2])
        q = quat_mul64((math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)), self._tilt())
        return ((float(p[0]), float(p[1]), self.z * math.sin(7.0 * t)), q)

    def EstimateGravityOrientation(self, t):
        w, x, y, z = self._tilt()
        return (w, -x, -y, -z)

    def AddPose(self, t, pose):
        self.last_pose_time = t
        self.added.append((t, pose))

    def GetLastPoseTime(self):
        return self.last_pose_time

    def GetLastExtrapolatedTime(self):
        return self.last_extrapolated
