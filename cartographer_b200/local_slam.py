"""LocalTrajectoryBuilder2D (mapping/internal/2d/local_trajectory_builder_2d.h) on the device.

The per-point stages (accumulation, gravity alignment, crop, voxel filters, scan matching and
the submap insert) run in one csm_local_slam2d handle with the range data kept in device memory.
The host keeps what the reference computes in double precision with libm: the injected pose
extrapolator, the gravity alignment, Embed3D of the 2D pose, the motion filter and the
ActiveSubmaps2D lifecycle.  Times are seconds (float).
"""
import ctypes as C
import ctypes.util
import math
from dataclasses import dataclass, field

import numpy as np

from ._lib import CsmStats, check, lib, ptr
from .scan_matching import (ActiveSubmaps2D, CeresScanMatcherOptions2D, CsmCeresOptions2D,
                            CsmCeresResult2D, CsmRangeInserterOptions2D, CERES_TERMINATION,
                            RealTimeCorrelativeScanMatcherOptions, SubmapsOptions2D)
from .sensor import AdaptiveVoxelFilterOptions, CsmAdaptiveVoxelFilterOptions

_libm = C.CDLL(ctypes.util.find_library("m"))
_libm.cosf.restype = _libm.sinf.restype = C.c_float
_libm.cosf.argtypes = _libm.sinf.argtypes = [C.c_float]

MATCHED, DROPPED_EMPTY_RETURNS, DROPPED_EMPTY_FILTERED = 0, 1, 2
(ACCUMULATED_RETURNS, ACCUMULATED_MISSES, CROPPED_RETURNS, CROPPED_MISSES, FILTERED_RETURNS,
 FILTERED_MISSES, FILTERED, LOCAL_RETURNS, LOCAL_MISSES) = range(9)


# ---- Eigen's float quaternion / Rigid3f arithmetic (csrc/rigid3f.h), in float32 scalars ----
F = np.float32


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def rotate3f(q, v):
    """Quaternionf * Vector3f (_transformVector); q = (w, x, y, z) float32."""
    qv = (q[1], q[2], q[3])
    uv = _cross(qv, v)
    uv = (uv[0] + uv[0], uv[1] + uv[1], uv[2] + uv[2])
    c = _cross(qv, uv)
    return tuple((v[k] + q[0] * uv[k]) + c[k] for k in range(3))


def rigid3f_apply(r, p):
    """Rigid3f * point: r = (t(3), q(4)) float32."""
    t, q = r
    x = rotate3f(q, tuple(F(c) for c in p))
    return tuple(x[k] + t[k] for k in range(3))


def quatf_mul(a, b):
    """Eigen's SSE quat_product<float> (rigid3f.h QuatMul)."""
    w = (a[0] * b[0] - a[1] * b[1]) + -(a[3] * b[3] + a[2] * b[2])
    x = (a[1] * b[0] - a[3] * b[2]) + (a[2] * b[3] + a[0] * b[1])
    y = (a[2] * b[0] - a[1] * b[3]) + (a[3] * b[1] + a[0] * b[2])
    z = (a[3] * b[0] - a[2] * b[1]) + (a[1] * b[2] + a[0] * b[3])
    return (w, x, y, z)


def quatf_normalized(q):
    n2 = (q[1] * q[1] + q[3] * q[3]) + (q[2] * q[2] + q[0] * q[0])
    if n2 > 0:
        n = F(np.sqrt(n2))
        return tuple(c / n for c in q)
    return q


def rigid3f(t, q):
    return (tuple(F(c) for c in t), tuple(F(c) for c in q))


def rigid3f_inverse(r):
    t, q = r
    qc = (q[0], -q[1], -q[2], -q[3])
    rt = rotate3f(qc, t)
    return ((-rt[0], -rt[1], -rt[2]), qc)


def rigid3f_mul(a, b):
    ta, qa = a
    tb, qb = b
    rt = rotate3f(qa, tb)
    return (tuple(rt[k] + ta[k] for k in range(3)), quatf_normalized(quatf_mul(qa, qb)))


def embed3d_f(pose2d):
    """Embed3D(Rigid2d.cast<float>()): Quaternionf(AngleAxisf(angle, UnitZ)) with libm's
    cosf / sinf of the float half angle."""
    a = F(pose2d[2])
    h = F(0.5) * a
    c, s = F(_libm.cosf(h)), F(_libm.sinf(h))
    return ((F(pose2d[0]), F(pose2d[1]), F(0.0)), (c, s * F(0.0), s * F(0.0), s * F(1.0)))


def _flat(r):
    return np.array(list(r[0]) + list(r[1]), np.float32)


# ---- double Rigid3d arithmetic for the pose the extrapolator and motion filter see ----
# Poses are (t(3), q(4) wxyz) tuples of Python floats.  The expressions follow Eigen's scalar
# paths (_transformVector, the quaternion product, normalized()); Eigen may vectorise the double
# quaternion product with a different summation order, so the last bits of a composed rotation
# can differ from a given build of the reference.
def _quatd_mul(a, b):
    return (a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
            a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1])


def _quatd_normalized(q):
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    return tuple(c / n for c in q) if n > 0 else q


def _quatd_rotate(q, v):
    """Quaterniond * Vector3d: _transformVector (uv = 2 q.vec x v; v + w uv + q.vec x uv)."""
    qv = (q[1], q[2], q[3])
    uv = _cross(qv, v)
    uv = (uv[0] + uv[0], uv[1] + uv[1], uv[2] + uv[2])
    c = _cross(qv, uv)
    return tuple((v[k] + q[0] * uv[k]) + c[k] for k in range(3))


def rigid3d_mul(a, b):
    """Rigid3d * Rigid3d (rigid_transform.h:184-189)."""
    rt = _quatd_rotate(a[1], b[0])
    return (tuple(rt[k] + a[0][k] for k in range(3)), _quatd_normalized(_quatd_mul(a[1], b[1])))


def rigid3d_inverse(r):
    """Rigid3d::inverse (rigid_transform.h:159-163)."""
    t, q = r
    qc = (q[0], -q[1], -q[2], -q[3])
    rt = _quatd_rotate(qc, t)
    return ((-rt[0], -rt[1], -rt[2]), qc)


def embed3d(pose2d):
    """Embed3D(Rigid2d): AngleAxisd(angle, UnitZ) as Eigen builds it (cos / sin of the half
    angle)."""
    h = 0.5 * pose2d[2]
    s = math.sin(h)
    return ((pose2d[0], pose2d[1], 0.0), (math.cos(h), s * 0.0, s * 0.0, s * 1.0))


def project2d(r):
    """Project2D (transform.h:76-80): the translation's x, y and GetYaw (:43-47), atan2 of
    rotation * UnitX."""
    t, q = r
    d = _quatd_rotate(q, (1.0, 0.0, 0.0))
    return np.array([t[0], t[1], math.atan2(d[1], d[0])])


def get_angle(q):
    """transform::GetAngle (transform.h:34-38)."""
    return 2.0 * math.atan2(math.sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), abs(q[0]))


def to_ticks(seconds):
    """common::Time's 100 ns ticks of a time given in seconds (rounded to the nearest tick)."""
    return int(round(seconds * 1e7))


# ---- options ----
@dataclass
class MotionFilterOptions:
    """proto MotionFilterOptions; trajectory_builder_2d.lua's motion_filter."""
    max_time_seconds: float = 5.0
    max_distance_meters: float = 0.2
    max_angle_radians: float = math.radians(1.0)


@dataclass
class LocalTrajectoryBuilderOptions2D:
    """proto LocalTrajectoryBuilderOptions2D with configuration_files/trajectory_builder_2d.lua's
    defaults.  The float fields of the proto are rounded to float32 where they are used."""
    min_range: float = 0.0
    max_range: float = 30.0
    min_z: float = -0.8
    max_z: float = 2.0
    missing_data_ray_length: float = 5.0
    num_accumulated_range_data: int = 1
    voxel_filter_size: float = 0.025
    adaptive_voxel_filter_options: AdaptiveVoxelFilterOptions = field(
        default_factory=lambda: AdaptiveVoxelFilterOptions(0.5, 200.0, 50.0))
    use_online_correlative_scan_matching: bool = False
    real_time_correlative_scan_matcher_options: RealTimeCorrelativeScanMatcherOptions = field(
        default_factory=lambda: RealTimeCorrelativeScanMatcherOptions(
            0.1, math.radians(20.0), 1e-1, 1e-1))
    ceres_scan_matcher_options: CeresScanMatcherOptions2D = field(
        default_factory=lambda: CeresScanMatcherOptions2D(1.0, 10.0, 40.0, False, 20))
    motion_filter_options: MotionFilterOptions = field(default_factory=MotionFilterOptions)
    submaps_options: SubmapsOptions2D = field(default_factory=SubmapsOptions2D)
    use_imu_data: bool = False


class CsmLocalSlamOptions2D(C.Structure):
    _fields_ = [("min_range", C.c_float), ("max_range", C.c_float), ("min_z", C.c_float),
                ("max_z", C.c_float), ("missing_data_ray_length", C.c_float),
                ("voxel_filter_size", C.c_float), ("num_accumulated_range_data", C.c_int32),
                ("use_online_correlative_scan_matching", C.c_int32),
                ("adaptive_voxel_filter", CsmAdaptiveVoxelFilterOptions),
                ("linear_search_window", C.c_double), ("angular_search_window", C.c_double),
                ("translation_delta_cost_weight", C.c_double),
                ("rotation_delta_cost_weight", C.c_double), ("ceres", CsmCeresOptions2D),
                ("inserter", CsmRangeInserterOptions2D)]


class CsmLocalSlamMatch2D(C.Structure):
    _fields_ = [("status", C.c_int32), ("matched_submap", C.c_int32),
                ("num_returns", C.c_int32), ("num_misses", C.c_int32),
                ("num_filtered", C.c_int32), ("reserved", C.c_int32),
                ("pose_estimate", C.c_double * 3), ("rt_score", C.c_double),
                ("ceres", CsmCeresResult2D)]


def c_options(o):
    a = o.adaptive_voxel_filter_options
    rt = o.real_time_correlative_scan_matcher_options
    return CsmLocalSlamOptions2D(
        o.min_range, o.max_range, o.min_z, o.max_z, o.missing_data_ray_length,
        o.voxel_filter_size, int(o.num_accumulated_range_data),
        1 if o.use_online_correlative_scan_matching else 0,
        CsmAdaptiveVoxelFilterOptions(a.max_length, a.min_num_points, a.max_range, 0),
        rt.linear_search_window, rt.angular_search_window, rt.translation_delta_cost_weight,
        rt.rotation_delta_cost_weight, o.ceres_scan_matcher_options._c(),
        o.submaps_options.probability_grid_range_data_inserter_options._c())


class MotionFilter:
    """mapping/internal/motion_filter.cc in double on the host.  Poses are (t(3), q(4) wxyz);
    times are seconds, compared as common::Time's 100 ns ticks against
    FromSeconds(max_time_seconds) (truncated to a tick, as duration_cast does)."""

    def __init__(self, options=None):
        self.options = options or MotionFilterOptions()
        self.num_total = 0
        self.num_different = 0
        self.last_time = None
        self.last_pose = None

    def IsSimilar(self, time, pose):
        self.num_total += 1
        o = self.options
        if (self.num_total > 1 and
                to_ticks(time) - self.last_time <= int(o.max_time_seconds * 1e7) and
                math.sqrt(sum((pose[0][k] - self.last_pose[0][k]) ** 2 for k in range(3)))
                <= o.max_distance_meters and
                get_angle(rigid3d_mul(rigid3d_inverse(pose), self.last_pose)[1])
                <= o.max_angle_radians):
            return True
        self.last_time = to_ticks(time)
        self.last_pose = pose
        self.num_different += 1
        return False


@dataclass
class InsertionResult:
    time: float
    gravity_alignment: tuple
    filtered_gravity_aligned_point_cloud: np.ndarray
    local_pose: tuple
    insertion_submaps: list


@dataclass
class MatchingResult:
    time: float
    local_pose: tuple                 # Rigid3d (t(3), q(4) wxyz)
    range_data_in_local_origin: tuple
    insertion_result: object          # InsertionResult or None (the motion filter said similar)
    pose_estimate_2d: np.ndarray
    ceres_summary: object
    rt_score: float
    stats: dict


class LocalSlam2D:
    """The csm_local_slam2d handle: accumulate / match / insert and the read-back hooks."""

    def __init__(self, options, device=0):
        self._h = C.c_void_p()
        o = c_options(options)
        check(lib().csm_local_slam2d_create(C.byref(o), C.c_int32(device), C.byref(self._h)))

    def accumulate(self, hits, origins, origin_index, poses, pose_index):
        hits = np.ascontiguousarray(hits, np.float32).reshape(-1, 3)
        origins = np.ascontiguousarray(origins, np.float32).reshape(-1, 3)
        oi = np.ascontiguousarray(origin_index, np.int32)
        poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 7)
        pi = np.ascontiguousarray(pose_index, np.int32)
        st = CsmStats()
        check(lib().csm_local_slam2d_accumulate(
            self._h, ptr(hits, C.c_float), C.c_int32(len(hits)), ptr(origins, C.c_float),
            C.c_int32(len(origins)), ptr(oi, C.c_int32), ptr(poses, C.c_float),
            C.c_int32(len(poses)), ptr(pi, C.c_int32), C.byref(st)))
        return st.as_dict()

    def match(self, to_gravity, origin, pose_prediction, grid):
        tg = np.ascontiguousarray(to_gravity, np.float32).reshape(7)
        org = np.ascontiguousarray(origin, np.float32).reshape(3)
        pp = np.ascontiguousarray(pose_prediction, np.float64).reshape(3)
        r = CsmLocalSlamMatch2D()
        st = CsmStats()
        check(lib().csm_local_slam2d_match(
            self._h, ptr(tg, C.c_float), ptr(org, C.c_float), ptr(pp, C.c_double),
            grid._h if grid is not None else None, C.byref(r), C.byref(st)))
        return r, st.as_dict()

    def insert(self, pose, grids):
        p = np.ascontiguousarray(pose, np.float32).reshape(7)
        handles = (C.c_void_p * len(grids))(*[g._h for g in grids])
        org = np.zeros(3, np.float32)
        st = CsmStats()
        check(lib().csm_local_slam2d_insert(self._h, ptr(p, C.c_float), handles,
                                            C.c_int32(len(grids)), ptr(org, C.c_float),
                                            C.byref(st)))
        for g in grids:
            g._info()
        return org, st.as_dict()

    def read(self, which):
        n = C.c_int32()
        check(lib().csm_local_slam2d_read(self._h, C.c_int32(which), None, C.c_int64(0),
                                          C.byref(n)))
        out = np.zeros((n.value, 3), np.float32)
        check(lib().csm_local_slam2d_read(self._h, C.c_int32(which), ptr(out, C.c_float),
                                          C.c_int64(n.value), C.byref(n)))
        return out

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_local_slam2d_destroy(self._h)
            self._h = None

    __del__ = close


class LocalTrajectoryBuilder2D:
    """local_trajectory_builder_2d.cc:65-300 over csm_local_slam2d.  `extrapolator` is a
    PoseExtrapolatorInterface-like object: ExtrapolatePose(t) -> (t(3), q(4) wxyz) doubles,
    EstimateGravityOrientation(t) -> q(4), AddPose(t, pose), GetLastPoseTime(),
    GetLastExtrapolatedTime().  It may be None until the caller has one (the reference then
    returns nullptr)."""

    def __init__(self, options, extrapolator, device=0):
        if options.num_accumulated_range_data < 1:
            raise ValueError("num_accumulated_range_data must be positive")
        self.options = options
        self.extrapolator = extrapolator
        self.slam = LocalSlam2D(options, device)
        self.active_submaps = ActiveSubmaps2D(options.submaps_options, device)
        self.motion_filter = MotionFilter(options.motion_filter_options)
        self.num_accumulated = 0
        self.last_stats = None

    def _poses(self, time, times):
        """range_data_poses (:141-160): one Rigid3f per distinct clamped point time, and each
        point's index into them.  -> (list of (t, q) float32 tuples, flat n x 7 float32 table,
        index)."""
        ex = self.extrapolator
        table, flat, index, seen = [], [], np.zeros(len(times), np.int32), {}
        last = ex.GetLastExtrapolatedTime()
        for i, t in enumerate(times.tolist()):
            tp = time + t
            if tp < last:       # :145-155, the time jumps backwards
                tp = last
            k = seen.get(tp)
            if k is None:
                p = ex.ExtrapolatePose(tp)
                k = seen[tp] = len(table)
                table.append(rigid3f(p[0], p[1]))
                flat.extend(p[0])
                flat.extend(p[1])
                last = ex.GetLastExtrapolatedTime()
            index[i] = k
        return table, np.array(flat, np.float32).reshape(-1, 7), index

    def AddRangeData(self, time, hits_with_times, origins, origin_index):
        """Synchronized range data: hits_with_times (n x 4: x, y, z, relative time <= 0 of the
        last point), origins (m x 3) and each hit's origin_index.  Returns a MatchingResult, or
        None while accumulating, initialising or after a dropped scan."""
        ex = self.extrapolator
        if ex is None:
            return None
        hw = np.asarray(hits_with_times, np.float32).reshape(-1, 4)
        if len(hw) == 0:
            raise ValueError("empty range data")
        if not hw[-1, 3] <= 0:
            raise ValueError("the last point's time must be <= 0")
        if time + float(hw[0, 3]) < ex.GetLastPoseTime():
            return None        # the extrapolator is still initialising (:130-134)
        table, flat, index = self._poses(time, hw[:, 3])
        self.slam.accumulate(hw[:, :3], origins, origin_index, flat, index)
        self.num_accumulated += 1
        if self.num_accumulated < self.options.num_accumulated_range_data:
            return None
        self.num_accumulated = 0
        gq = tuple(float(c) for c in ex.EstimateGravityOrientation(time))
        last = table[index[-1]]
        to_gravity = rigid3f_mul(((F(0), F(0), F(0)), tuple(F(c) for c in gq)),
                                 rigid3f_inverse(last))
        gravity = ((0.0, 0.0, 0.0), gq)
        pred3 = ex.ExtrapolatePose(time)
        prediction = project2d(rigid3d_mul(
            (tuple(pred3[0]), tuple(pred3[1])), rigid3d_inverse(gravity)))
        submaps = self.active_submaps.submaps()
        grid = submaps[0].grid if submaps else None
        r, st = self.slam.match(_flat(to_gravity), last[0], prediction, grid)
        self.last_stats = {"match": st}
        if r.status != MATCHED:
            return None
        pose2d = np.array(r.pose_estimate[:], np.float64)
        pose_estimate = rigid3d_mul(embed3d(pose2d), gravity)
        ex.AddPose(time, pose_estimate)
        pose3f = embed3d_f(pose2d)
        filtered = self.slam.read(FILTERED)
        ga_origin = rigid3f_apply(to_gravity, last[0])
        origin_in_local = np.array(rigid3f_apply(pose3f, ga_origin), np.float32)
        insertion = None
        if not self.motion_filter.IsSimilar(time, pose_estimate):
            ist = {}

            def insert(grids):
                org, st = self.slam.insert(_flat(pose3f), grids)
                assert np.array_equal(org, origin_in_local)
                ist.update(st)
            subs = self.active_submaps.insert_with(origin_in_local, insert)
            self.last_stats["insert"] = ist
            insertion = InsertionResult(time, gq, filtered, pose_estimate, subs)
        summary = None
        if r.matched_submap:
            c = r.ceres
            summary = dict(initial_cost=c.initial_cost, final_cost=c.final_cost,
                           iterations=c.iterations, num_successful_steps=c.num_successful_steps,
                           termination=CERES_TERMINATION[c.termination])
        return MatchingResult(time, pose_estimate, tuple(origin_in_local), insertion, pose2d,
                              summary, r.rt_score, self.last_stats)

    def close(self):
        self.slam.close()
