"""Host-side mirror of cartographer::mapping::scan_matching for the hot path,
over the C ABI (include/csm_abi.h).  Same class / method names, argument meaning
and "no match" convention as the reference; out-parameters become return values.

Reference: cartographer/mapping/internal/2d/scan_matching/
  fast_correlative_scan_matcher_2d.h:112-136, real_time_correlative_scan_matcher_2d.h:53-85.
"""
import ctypes as C
import math
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from ._lib import CsmStats, JOB2D_DTYPE, RESULT2D_DTYPE, check, lib, ptr

# csm_node2d: a branch-and-bound frontier node
NODE2D_DTYPE = np.dtype([("scan", "<i4"), ("xo", "<i4"), ("yo", "<i4"), ("score", "<f4")])


@dataclass
class FastCorrelativeScanMatcherOptions2D:
    """proto/scan_matching/fast_correlative_scan_matcher_options_2d.proto"""
    linear_search_window: float
    angular_search_window: float
    branch_and_bound_depth: int


@dataclass
class RealTimeCorrelativeScanMatcherOptions:
    """proto/scan_matching/real_time_correlative_scan_matcher_options.proto"""
    linear_search_window: float
    angular_search_window: float
    translation_delta_cost_weight: float
    rotation_delta_cost_weight: float


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError("point cloud must be N x 3 float32")
    return a


class DeviceCloud:
    """sensor::PointCloud resident on the device (csm_cloud)."""

    def __init__(self, xyz, device=0):
        xyz = _f32(xyz)
        self.num_points = len(xyz)
        self._h = C.c_void_p()
        check(lib().csm_cloud_create(ptr(xyz, C.c_float), C.c_int32(len(xyz)),
                                     C.c_int32(device), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_cloud_destroy(self._h)
            self._h = None

    __del__ = close


class FastCorrelativeScanMatcher2D:
    """FastCorrelativeScanMatcher2D(grid, options): builds the precomputation grid
    stack on the device (fast_correlative_scan_matcher_2d.cc:188-194).  `grid` is any
    record with cells (uint16 [num_y, num_x]), resolution, max_x, max_y, min_cost,
    max_cost — Grid2D's limits() and correspondence_cost_cells()."""

    def __init__(self, grid, options, device=0):
        self.options = options
        self.device = device
        cells = np.ascontiguousarray(grid.cells, dtype=np.uint16)
        self._h = C.c_void_p()
        check(lib().csm_stack2d_create(
            ptr(cells, C.c_uint16), C.c_int32(cells.shape[1]), C.c_int32(cells.shape[0]),
            C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
            C.c_float(grid.min_cost), C.c_float(grid.max_cost),
            C.c_int32(options.branch_and_bound_depth), C.c_int32(device), C.byref(self._h)))
        self.last_stats = None

    @classmethod
    def from_proto(cls, serialized_grid2d, options, device=0):
        """Builds the matcher straight from a serialized cartographer.mapping.proto.Grid2D
        (csm_stack2d_create_from_proto; Grid2D::Grid2D(const proto::Grid2D&) semantics)."""
        self = cls.__new__(cls)
        self.options, self.device, self.last_stats = options, device, None
        buf = (C.c_uint8 * len(serialized_grid2d)).from_buffer_copy(serialized_grid2d)
        self._h = C.c_void_p()
        check(lib().csm_stack2d_create_from_proto(buf, C.c_int64(len(serialized_grid2d)),
                                                  C.c_int32(options.branch_and_bound_depth),
                                                  C.c_int32(device), C.byref(self._h)))
        return self

    @classmethod
    def _adopt(cls, handle, options, device):
        self = cls.__new__(cls)
        self.options, self.device, self.last_stats = options, device, None
        self._h = C.c_void_p(handle)
        return self

    def update(self, cells):
        """csm_stack2d_update: the submap's grid changed (same limits); rebuild in place."""
        cells = np.ascontiguousarray(cells, dtype=np.uint16)
        check(lib().csm_stack2d_update(self._h, ptr(cells, C.c_uint16)))

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_stack2d_destroy(self._h)
            self._h = None

    __del__ = close

    def _match(self, xyz, initial_pose, full, min_score):
        xyz = _f32(xyz)
        ip = np.ascontiguousarray(initial_pose, dtype=np.float64)
        found = C.c_int32(0)
        score = C.c_float(0.0)
        pose = np.zeros(3, np.float64)
        stats = CsmStats()
        check(lib().csm_match2d(self._h, ptr(xyz, C.c_float), C.c_int32(len(xyz)),
                                ptr(ip, C.c_double), C.c_int32(int(full)),
                                C.c_double(self.options.linear_search_window),
                                C.c_double(self.options.angular_search_window),
                                C.c_float(min_score), C.byref(found), C.byref(score),
                                ptr(pose, C.c_double), C.byref(stats)))
        self.last_stats = stats.as_dict()
        if not found.value:
            return False, None, None
        return True, np.float32(score.value), pose

    def Match(self, initial_pose_estimate, point_cloud, min_score):
        """-> (found, score, pose_estimate[x, y, yaw]); (False, None, None) if no
        score above min_score (strict), fast_correlative_scan_matcher_2d.cc:198-208."""
        return self._match(point_cloud, initial_pose_estimate, False, min_score)

    def MatchFullSubmap(self, point_cloud, min_score):
        """fast_correlative_scan_matcher_2d.cc:210-225."""
        return self._match(point_cloud, (0.0, 0.0, 0.0), True, min_score)

    # -- "visible for testing" hooks ------------------------------------------------
    def precomputation_grid(self, level):
        nx, ny = C.c_int32(), C.c_int32()
        check(lib().csm_stack2d_read_level(self._h, C.c_int32(level), None, C.byref(nx),
                                           C.byref(ny)))
        out = np.empty((ny.value, nx.value), np.uint8)
        check(lib().csm_stack2d_read_level(self._h, C.c_int32(level), ptr(out, C.c_uint8),
                                           C.byref(nx), C.byref(ny)))
        return out

    def score_candidates(self, level, discrete_scans, candidates):
        ds = np.ascontiguousarray(discrete_scans, dtype=np.int32)
        cand = np.ascontiguousarray(candidates, dtype=np.int32).reshape(-1, 3)
        S, n, _ = ds.shape
        scores = np.empty(len(cand), np.float32)
        sums = np.empty(len(cand), np.int32)
        check(lib().csm_score_candidates2d(self._h, C.c_int32(level), ptr(ds, C.c_int32),
                                           C.c_int32(S), C.c_int32(n), ptr(cand, C.c_int32),
                                           C.c_int32(len(cand)), ptr(scores, C.c_float),
                                           ptr(sums, C.c_int32)))
        return scores, sums

    def discretize(self, point_cloud, initial_pose_estimate=(0.0, 0.0, 0.0), full_submap=False):
        xyz = _f32(point_cloud)
        ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
        S = C.c_int32(0)
        args = (self._h, ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
                C.c_int32(int(full_submap)), C.c_double(self.options.linear_search_window),
                C.c_double(self.options.angular_search_window), C.byref(S))
        check(lib().csm_discretize2d(*args, None, None))
        ds = np.empty((S.value, len(xyz), 2), np.int32)
        bounds = np.empty((S.value, 4), np.int32)
        check(lib().csm_discretize2d(*args, ptr(ds, C.c_int32), ptr(bounds, C.c_int32)))
        return ds, bounds

    TOP_FORMS = ("auto", "small", "gather", "tile", "dense")

    def score_top(self, point_cloud, initial_pose_estimate=(0.0, 0.0, 0.0), full_submap=False,
                  form="auto"):
        """csm_score_top2d: the lowest-resolution sums of the match's candidates.
        -> (sums, lattices, kernel): sums[scan] is the scan's nxc * nyc sums in slot order
        (slot = i * nyc + j), lattices is num_scans x (min_x, max_x, min_y, max_y, nxc, nyc),
        kernel = (form that ran, K of k_score_top_tile<K> or 0)."""
        xyz = _f32(point_cloud)
        ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
        S, cap = C.c_int32(0), C.c_int32(0)
        args = (self._h, ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
                C.c_int32(int(full_submap)), C.c_double(self.options.linear_search_window),
                C.c_double(self.options.angular_search_window),
                C.c_int32(self.TOP_FORMS.index(form)), C.byref(S), C.byref(cap))
        check(lib().csm_score_top2d(*args, None, None, None))
        sums = np.zeros((S.value, cap.value), np.int32)
        lattices = np.zeros((S.value, 6), np.int32)
        kernel = np.zeros(2, np.int32)
        check(lib().csm_score_top2d(*args, ptr(sums, C.c_int32), ptr(lattices, C.c_int32),
                                    ptr(kernel, C.c_int32)))
        return ([sums[k, :nxc * nyc] for k, (_, _, _, _, nxc, nyc) in enumerate(lattices)],
                lattices, (self.TOP_FORMS[kernel[0]], int(kernel[1])))

    def branch_step(self, point_cloud, initial_pose_estimate, full_submap, min_score, level,
                    parents, bound, form, unroll=8):
        """csm_branch_step2d: one branch step over `parents` (NODE2D_DTYPE records) at
        `level` with the job's bound set to `bound`; form "warp" or "lattice".
        -> (children in queue order, final bound, (candidates scored, parents expanded))."""
        xyz = _f32(point_cloud)
        ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
        par = np.ascontiguousarray(parents, dtype=NODE2D_DTYPE)
        out = np.zeros(max(1, 4 * len(par)), NODE2D_DTYPE)
        count, final = C.c_int32(0), C.c_float(0.0)
        ctr = np.zeros(2, np.int64)
        check(lib().csm_branch_step2d(
            self._h, ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
            C.c_int32(int(full_submap)), C.c_double(self.options.linear_search_window),
            C.c_double(self.options.angular_search_window), C.c_float(min_score),
            C.c_int32(level), par.ctypes.data_as(C.c_void_p), C.c_int32(len(par)),
            C.c_float(bound), C.c_int32(("warp", "lattice").index(form)), C.c_int32(unroll),
            out.ctypes.data_as(C.c_void_p), C.byref(count), C.byref(final),
            ptr(ctr, C.c_int64)))
        return out[:count.value].copy(), np.float32(final.value), (int(ctr[0]), int(ctr[1]))

    def dives(self, point_cloud, initial_pose_estimate, full_submap, min_score, dive_ratio):
        """csm_dives2d: the match's greedy dives and top-queue filter.
        -> (job_best, (bound after the dives, bound after the filter),
            (candidates the dives scored, dives run), top queue in queue order)."""
        xyz = _f32(point_cloud)
        ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
        job_best, count = C.c_int32(0), C.c_int32(0)
        bounds = np.zeros(2, np.float32)
        ctr = np.zeros(2, np.int64)
        out = np.zeros(4096, NODE2D_DTYPE)
        while True:
            check(lib().csm_dives2d(
                self._h, ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
                C.c_int32(int(full_submap)), C.c_double(self.options.linear_search_window),
                C.c_double(self.options.angular_search_window), C.c_float(min_score),
                C.c_float(dive_ratio), C.byref(job_best), ptr(bounds, C.c_float),
                ptr(ctr, C.c_int64), out.ctypes.data_as(C.c_void_p), C.c_int32(len(out)),
                C.byref(count)))
            if count.value <= len(out):
                break
            out = np.zeros(count.value, NODE2D_DTYPE)
        return (int(job_best.value), (bounds[0], bounds[1]), (int(ctr[0]), int(ctr[1])),
                out[:count.value].copy())


class SweepLimits2D(C.Structure):
    """csm_sweep_limits2d: limits of the batched 2D branch-and-bound sweep."""
    _fields_ = [("chunk", C.c_int32), ("leaf_cap", C.c_int32), ("inline_best", C.c_int32),
                ("lattice_min", C.c_int32), ("unroll", C.c_int32), ("dive_ratio", C.c_float),
                ("max_points", C.c_int64)]

    @classmethod
    def default(cls):
        out = cls()
        lib().csm_sweep_limits2d_default(C.byref(out))
        return out


def load_pbstream_matchers2d(path, options, device=0):
    """csm_pbstream_load_stacks2d: one FastCorrelativeScanMatcher2D per 2D submap of a
    .pbstream file, in file order.  -> (matchers, [(trajectory_id, submap_index), ...])"""
    n = C.c_int32(0)
    check(lib().csm_pbstream_load_stacks2d(path.encode(), C.c_int32(options.branch_and_bound_depth),
                                           C.c_int32(device), C.c_int32(0), None, None,
                                           C.byref(n)))
    count = n.value
    handles = (C.c_void_p * max(1, count))()
    ids = np.zeros((max(1, count), 2), np.int32)
    check(lib().csm_pbstream_load_stacks2d(path.encode(), C.c_int32(options.branch_and_bound_depth),
                                           C.c_int32(device), C.c_int32(count), handles,
                                           ptr(ids, C.c_int32), C.byref(n)))
    matchers = [FastCorrelativeScanMatcher2D._adopt(handles[k], options, device)
                for k in range(count)]
    return matchers, [(int(a), int(b)) for a, b in ids[:count]]


def match_batch(matchers, clouds, jobs, linear_search_window, angular_search_window,
                limits=None):
    """Batched FastCorrelativeScanMatcher2D searches (csm_match2d_batch_limits).

    matchers: list of FastCorrelativeScanMatcher2D; clouds: list of DeviceCloud;
    jobs: numpy array of JOB2D_DTYPE; limits: None (the defaults), a SweepLimits2D, or a
    dict of SweepLimits2D fields that override the defaults.  Returns
    (results[RESULT2D_DTYPE], stats dict); stats["sweep_trace"] is (collects, leaf
    compactions, most leaves held at a collect, optimal leaves).
    """
    jobs = np.ascontiguousarray(jobs, dtype=JOB2D_DTYPE)
    hs = (C.c_void_p * len(matchers))(*[m._h for m in matchers])
    cs = (C.c_void_p * len(clouds))(*[c._h for c in clouds])
    results = np.zeros(len(jobs), RESULT2D_DTYPE)
    stats = CsmStats()
    if isinstance(limits, dict):
        lim = SweepLimits2D.default()
        for k, v in limits.items():
            setattr(lim, k, v)
        limits = lim
    trace = np.zeros(4, np.int32)
    check(lib().csm_match2d_batch_limits(
        hs, C.c_int32(len(matchers)), cs, C.c_int32(len(clouds)),
        jobs.ctypes.data_as(C.c_void_p), C.c_int32(len(jobs)), C.c_double(linear_search_window),
        C.c_double(angular_search_window), C.byref(limits) if limits is not None else None,
        results.ctypes.data_as(C.c_void_p), C.byref(stats), ptr(trace, C.c_int32)))
    out = stats.as_dict()
    out["sweep_trace"] = tuple(int(v) for v in trace)
    return results, out


class RealTimeCorrelativeScanMatcher2D:
    """real_time_correlative_scan_matcher_2d.h:53-85."""

    def __init__(self, options, device=0):
        self.options = options
        self.device = device
        self.last_stats = None

    def Match(self, initial_pose_estimate, point_cloud, grid):
        """-> (score, pose_estimate), real_time_correlative_scan_matcher_2d.cc:117-149."""
        xyz = _f32(point_cloud)
        cells = np.ascontiguousarray(grid.cells, dtype=np.uint16)
        ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
        pose = np.zeros(3, np.float64)
        score = C.c_double(0.0)
        stats = CsmStats()
        o = self.options
        check(lib().csm_rt_match2d(
            ptr(cells, C.c_uint16), C.c_int32(cells.shape[1]), C.c_int32(cells.shape[0]),
            C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
            ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
            C.c_double(o.linear_search_window), C.c_double(o.angular_search_window),
            C.c_double(o.translation_delta_cost_weight),
            C.c_double(o.rotation_delta_cost_weight), C.c_int32(self.device), C.byref(score),
            ptr(pose, C.c_double), C.byref(stats)))
        self.last_stats = stats.as_dict()
        return score.value, pose


@dataclass
class TSDF2DSpec:
    """Flat record of a TSDF2D grid (mapping/internal/2d/tsdf_2d.h): tsd and weight
    cells (uint16 [num_y, num_x]) plus the TSDValueConverter parameters."""
    tsd_cells: np.ndarray
    weight_cells: np.ndarray
    resolution: float
    max_x: float
    max_y: float
    truncation_distance: float
    max_weight: float


def _rt_match_tsdf(self, initial_pose_estimate, point_cloud, grid):
    xyz = _f32(point_cloud)
    tsd = np.ascontiguousarray(grid.tsd_cells, dtype=np.uint16)
    wgt = np.ascontiguousarray(grid.weight_cells, dtype=np.uint16)
    ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
    pose = np.zeros(3, np.float64)
    score = C.c_double(0.0)
    stats = CsmStats()
    o = self.options
    check(lib().csm_rt_match2d_tsdf(
        ptr(tsd, C.c_uint16), ptr(wgt, C.c_uint16), C.c_int32(tsd.shape[1]),
        C.c_int32(tsd.shape[0]), C.c_double(grid.resolution), C.c_double(grid.max_x),
        C.c_double(grid.max_y), C.c_float(grid.truncation_distance), C.c_float(grid.max_weight),
        ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
        C.c_double(o.linear_search_window), C.c_double(o.angular_search_window),
        C.c_double(o.translation_delta_cost_weight), C.c_double(o.rotation_delta_cost_weight),
        C.c_int32(self.device), C.byref(score), ptr(pose, C.c_double), C.byref(stats)))
    self.last_stats = stats.as_dict()
    return score.value, pose


RealTimeCorrelativeScanMatcher2D.MatchTSDF = _rt_match_tsdf


class CsmRtJob2D(C.Structure):
    _fields_ = [("xyz", C.POINTER(C.c_float)), ("num_points", C.c_int32), ("reserved", C.c_int32),
                ("initial_pose", C.c_double * 3)]


class CsmRtResult2D(C.Structure):
    _fields_ = [("score", C.c_double), ("pose_estimate", C.c_double * 3),
                ("best_scan_index", C.c_int32), ("best_x_offset", C.c_int32),
                ("best_y_offset", C.c_int32), ("num_scans", C.c_int32),
                ("candidates_scored", C.c_int64)]


class CsmRtGrid2DInfo(C.Structure):
    _fields_ = [("num_x_cells", C.c_int32), ("num_y_cells", C.c_int32),
                ("resolution", C.c_double), ("max_x", C.c_double), ("max_y", C.c_double),
                ("known_min_x", C.c_int32), ("known_min_y", C.c_int32),
                ("known_max_x", C.c_int32), ("known_max_y", C.c_int32),
                ("known_empty", C.c_int32), ("is_tsdf", C.c_int32)]


@dataclass
class GridState:
    """A ProbabilityGrid read back from the device: correspondence-cost cells[y, x], MapLimits
    and the known-cells box (min_x, min_y, max_x, max_y), None when empty.  For a TSDF2D,
    cells are its tsd cells and weight_cells its weight cells.  Usable wherever a
    grid record is taken (FastCorrelativeScanMatcher2D, RealTimeGrid2D)."""
    cells: np.ndarray
    resolution: float
    max_x: float
    max_y: float
    known_cells_box: object = None
    min_cost: float = float(np.float32(1.0) - (np.float32(1.0) - np.float32(0.1)))
    max_cost: float = float(np.float32(1.0) - np.float32(0.1))
    weight_cells: object = None   # a TSDF2D's weight cells[y, x] (cells are its tsd cells)


def _serialize(fn, handle, capacity):
    """bytes of fn(handle, buf, capacity, &size), a *_to_proto entry point, given a capacity
    that holds the message."""
    buf = np.zeros(max(capacity, 1), np.uint8)
    size = C.c_int64()
    check(fn(handle, ptr(buf, C.c_uint8), C.c_int64(buf.size), C.byref(size)))
    return buf[:size.value].tobytes()


def _texture(fn, handle, pose):
    """bytes of fn(handle, pose, buf, capacity, &size), a *_to_texture entry point: every call
    does the whole work, so a first try with a buffer that holds most textures, and a second
    with the exact size only when it did not."""
    p = np.ascontiguousarray(pose, np.float64).reshape(7)
    size = C.c_int64()
    buf = np.zeros(1 << 20, np.uint8)
    st = fn(handle, ptr(p, C.c_double), ptr(buf, C.c_uint8), C.c_int64(buf.size), C.byref(size))
    if st == 3 and size.value > buf.size:   # CSM_E_CAPACITY
        buf = np.zeros(size.value, np.uint8)
        st = fn(handle, ptr(p, C.c_double), ptr(buf, C.c_uint8), C.c_int64(buf.size),
                C.byref(size))
    check(st)
    return buf[:size.value].tobytes()


class RealTimeGrid2D:
    """A ProbabilityGrid or TSDF2D resident on the device (csm_rt_grid2d): what
    LocalTrajectoryBuilder2D's active submap grid is to the real-time matcher
    (local_trajectory_builder_2d.cc:77-82).  `grid` is a probability-grid record (.cells) or
    a TSDF2DSpec-like record (.tsd_cells, .weight_cells, .truncation_distance, .max_weight);
    the grid type then selects the real-time score and the refinement's cost function.
    update() re-uploads the cells after a scan insertion (same cell limits): update(cells)
    for a ProbabilityGrid, update(tsd_cells, weight_cells) for a TSDF2D."""

    def __init__(self, grid, device=0):
        self.device = device
        self._h = C.c_void_p()
        self.is_tsdf = hasattr(grid, "tsd_cells")
        if self.is_tsdf:
            tsd = np.ascontiguousarray(grid.tsd_cells, dtype=np.uint16)
            wgt = np.ascontiguousarray(grid.weight_cells, dtype=np.uint16)
            if wgt.shape != tsd.shape:
                raise ValueError("tsd and weight cells differ in shape")
            self.shape = tsd.shape
            check(lib().csm_rt_grid2d_create_tsdf(
                ptr(tsd, C.c_uint16), ptr(wgt, C.c_uint16), C.c_int32(tsd.shape[1]),
                C.c_int32(tsd.shape[0]), C.c_double(grid.resolution), C.c_double(grid.max_x),
                C.c_double(grid.max_y), C.c_float(grid.truncation_distance),
                C.c_float(grid.max_weight), C.c_int32(device), C.byref(self._h)))
            return
        cells = np.ascontiguousarray(grid.cells, dtype=np.uint16)
        self.shape = cells.shape
        check(lib().csm_rt_grid2d_create(
            ptr(cells, C.c_uint16), C.c_int32(cells.shape[1]), C.c_int32(cells.shape[0]),
            C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
            C.c_int32(device), C.byref(self._h)))

    @classmethod
    def empty(cls, resolution, max_x, max_y, num_x=100, num_y=100, device=0):
        """An all-unknown ProbabilityGrid of the given limits (csm_rt_grid2d_create_empty), to
        be filled by ProbabilityGridRangeDataInserter2D.Insert.  ActiveSubmaps2D::CreateGrid
        makes a 100 x 100 grid with max = origin + 50 * resolution on both axes."""
        self = cls.__new__(cls)
        self.device, self.is_tsdf = device, False
        self._h = C.c_void_p()
        check(lib().csm_rt_grid2d_create_empty(
            C.c_double(resolution), C.c_double(max_x), C.c_double(max_y), C.c_int32(num_x),
            C.c_int32(num_y), C.c_int32(device), C.byref(self._h)))
        self.shape = (num_y, num_x)
        return self

    @classmethod
    def empty_tsdf(cls, resolution, max_x, max_y, truncation_distance, max_weight, num_x=100,
                   num_y=100, device=0):
        """An all-unknown TSDF2D of the given limits and converter
        (csm_rt_grid2d_create_empty_tsdf), to be filled by TSDFRangeDataInserter2D.Insert:
        ActiveSubmaps2D::CreateGrid for GridType::TSDF."""
        self = cls.__new__(cls)
        self.device, self.is_tsdf = device, True
        self._h = C.c_void_p()
        check(lib().csm_rt_grid2d_create_empty_tsdf(
            C.c_double(resolution), C.c_double(max_x), C.c_double(max_y), C.c_int32(num_x),
            C.c_int32(num_y), C.c_float(truncation_distance), C.c_float(max_weight),
            C.c_int32(device), C.byref(self._h)))
        self.shape = (num_y, num_x)
        return self

    def _info(self, cells=None):
        info = CsmRtGrid2DInfo()
        check(lib().csm_rt_grid2d_read(self._h, C.byref(info),
                                       None if cells is None else ptr(cells, C.c_uint16),
                                       C.c_int64(0 if cells is None else cells.size)))
        self.shape = (info.num_y_cells, info.num_x_cells)
        return info

    def read(self):
        """The grid as it is on the device: a GridState with cells[y, x], the limits and the
        known-cells box (csm_rt_grid2d_read)."""
        info = self._info()
        cells = np.zeros((info.num_y_cells, info.num_x_cells), np.uint16)
        info = self._info(cells)
        box = None if info.known_empty else (info.known_min_x, info.known_min_y,
                                             info.known_max_x, info.known_max_y)
        weights = None
        if info.is_tsdf:
            weights = np.zeros_like(cells)
            check(lib().csm_rt_grid2d_read_weights(self._h, ptr(weights, C.c_uint16),
                                                   C.c_int64(weights.size)))
        return GridState(cells, info.resolution, info.max_x, info.max_y, box,
                         weight_cells=weights)

    def to_proto(self):
        """The serialised proto::Grid2D that ProbabilityGrid::ToProto or TSDF2D::ToProto gives
        for this grid (csm_rt_grid2d_to_proto), as bytes."""
        info = self._info()
        cells = info.num_x_cells * info.num_y_cells
        # at most 3 bytes per cell (values below 2^15) in each packed array, and 128 for the rest
        return _serialize(lib().csm_rt_grid2d_to_proto, self._h,
                          128 + 3 * cells * (2 if info.is_tsdf else 1))

    def to_texture(self, local_pose):
        """The serialised proto::SubmapQuery::Response::SubmapTexture that
        ProbabilityGrid::DrawToSubmapTexture or TSDF2D::DrawToSubmapTexture draws for this grid
        with the submap's local pose (tx, ty, tz, qw, qx, qy, qz), as Submap2D::ToResponseProto
        adds it (csm_rt_grid2d_to_texture), as bytes."""
        return _texture(lib().csm_rt_grid2d_to_texture, self._h, local_pose)

    def draw(self):
        """io::DrawProbabilityGrid of this ProbabilityGrid (csm_rt_grid2d_draw): (pixels,
        offset), pixels a (height, width) uint32 array of cairo ARGB32 grey words over the
        cropped limits and offset their first cell (x, y).  An empty grid gives one pixel of
        128 at offset (0, 0)."""
        w, h = C.c_int32(), C.c_int32()
        offset = np.zeros(2, np.int32)
        check(lib().csm_rt_grid2d_draw(self._h, None, C.c_int64(0), C.byref(w), C.byref(h),
                                       ptr(offset, C.c_int32), None))
        pixels = np.empty((h.value, w.value), np.uint32)
        check(lib().csm_rt_grid2d_draw(self._h, ptr(pixels, C.c_uint32), C.c_int64(pixels.size),
                                       C.byref(w), C.byref(h), ptr(offset, C.c_int32), None))
        return pixels, (int(offset[0]), int(offset[1]))

    def ComputeCroppedGrid(self):
        """ProbabilityGrid::ComputeCroppedGrid from device to device: a new RealTimeGrid2D over
        the known-cells box (csm_rt_grid2d_crop)."""
        out = RealTimeGrid2D.__new__(RealTimeGrid2D)
        out.device, out.is_tsdf = self.device, False
        out._h = C.c_void_p()
        check(lib().csm_rt_grid2d_crop(self._h, C.byref(out._h)))
        out._info()
        return out

    def update(self, cells, weight_cells=None):
        cells = np.ascontiguousarray(cells, dtype=np.uint16)
        if cells.shape != self.shape:
            raise ValueError("cell limits changed: create a new RealTimeGrid2D")
        if self.is_tsdf:
            if weight_cells is None:
                raise ValueError("a TSDF2D update needs its weight cells")
            wgt = np.ascontiguousarray(weight_cells, dtype=np.uint16)
            if wgt.shape != self.shape:
                raise ValueError("cell limits changed: create a new RealTimeGrid2D")
            check(lib().csm_rt_grid2d_update_tsdf(self._h, ptr(cells, C.c_uint16),
                                                  ptr(wgt, C.c_uint16)))
            return
        if weight_cells is not None:
            raise ValueError("a ProbabilityGrid has no weight cells")
        check(lib().csm_rt_grid2d_update(self._h, ptr(cells, C.c_uint16)))

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_rt_grid2d_destroy(self._h)
            self._h = None

    __del__ = close


# ===========================================================================
# ProbabilityGridRangeDataInserter2D (mapping/2d/probability_grid_range_data_inserter_2d.h)
# ===========================================================================
class CsmRangeInserterOptions2D(C.Structure):
    _fields_ = [("hit_probability", C.c_double), ("miss_probability", C.c_double),
                ("insert_free_space", C.c_int32), ("reserved", C.c_int32)]


@dataclass
class ProbabilityGridRangeDataInserterOptions2D:
    """proto ProbabilityGridRangeDataInserterOptions2D; defaults are
    configuration_files/trajectory_builder_2d.lua's submaps.range_data_inserter."""
    hit_probability: float = 0.55
    miss_probability: float = 0.49
    insert_free_space: bool = True

    def _c(self):
        return CsmRangeInserterOptions2D(self.hit_probability, self.miss_probability,
                                         1 if self.insert_free_space else 0, 0)


class ProbabilityGridRangeDataInserter2D:
    """Insert(origin, returns, grid, misses=None) writes one scan into a ProbabilityGrid
    RealTimeGrid2D in place, as the reference's Insert(range_data, grid) writes a
    ProbabilityGrid: origin (2 or 3), returns and misses (n x 3) are in the grid's frame.  The
    grid grows as the reference's does, and its `shape` follows."""

    def __init__(self, options=None, device=0):
        self.options = options or ProbabilityGridRangeDataInserterOptions2D()
        self.last_stats = None
        self._h = C.c_void_p()
        o = self.options._c()
        check(lib().csm_range_inserter2d_create(C.byref(o), C.c_int32(device),
                                                C.byref(self._h)))

    def Insert(self, origin, returns, grid, misses=None):
        org = np.zeros(3, np.float32)
        o = np.asarray(origin, np.float32).reshape(-1)
        org[:len(o)] = o[:3]
        ret = _f32(np.zeros((0, 3)) if returns is None else returns)
        mis = _f32(np.zeros((0, 3)) if misses is None else misses)
        stats = CsmStats()
        check(lib().csm_range_inserter2d_insert(
            self._h, ptr(org, C.c_float), ptr(ret, C.c_float), C.c_int32(len(ret)),
            ptr(mis, C.c_float), C.c_int32(len(mis)), grid._h, C.byref(stats)))
        self.last_stats = stats.as_dict()
        grid._info()

    def insert_submaps(self, grids, origin, returns, misses=None):
        """Insert(range_data, grid) into every ProbabilityGrid RealTimeGrid2D of `grids`, in
        one call (csm_range_inserter2d_insert_submaps), as ActiveSubmaps2D::InsertRangeData
        inserts each scan into its active submaps: each grid ends as len(grids) Insert calls
        in order would leave it, and a refused call leaves every grid unchanged."""
        org = np.zeros(3, np.float32)
        o = np.asarray(origin, np.float32).reshape(-1)
        org[:len(o)] = o[:3]
        ret = _f32(np.zeros((0, 3)) if returns is None else returns)
        mis = _f32(np.zeros((0, 3)) if misses is None else misses)
        handles = (C.c_void_p * len(grids))(*[g._h for g in grids])
        stats = CsmStats()
        check(lib().csm_range_inserter2d_insert_submaps(
            self._h, ptr(org, C.c_float), ptr(ret, C.c_float), C.c_int32(len(ret)),
            ptr(mis, C.c_float), C.c_int32(len(mis)), handles, C.c_int32(len(grids)),
            C.byref(stats)))
        self.last_stats = stats.as_dict()
        for g in grids:
            g._info()

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_range_inserter2d_destroy(self._h)
            self._h = None

    __del__ = close


# ===========================================================================
# Submap2D and ActiveSubmaps2D (mapping/2d/submap_2d.h) over device grids
# ===========================================================================
@dataclass
class SubmapsOptions2D:
    """proto SubmapsOptions2D (mapping/proto/submaps_options_2d.proto) with its GridOptions2D
    and RangeDataInserterOptions; defaults are configuration_files/trajectory_builder_2d.lua's
    submaps.  `resolution` is the float grid option."""
    num_range_data: int = 90
    grid_type: str = "PROBABILITY_GRID"
    resolution: float = 0.05
    range_data_inserter_type: str = "PROBABILITY_GRID_INSERTER_2D"
    probability_grid_range_data_inserter_options: ProbabilityGridRangeDataInserterOptions2D = \
        field(default_factory=ProbabilityGridRangeDataInserterOptions2D)


def create_grid_limits(origin, resolution):
    """The MapLimits of ActiveSubmaps2D::CreateGrid (submap_2d.cc:192-204):
    (resolution, max_x, max_y, 100, 100).  The float resolution option and the float origin
    enter double arithmetic: max = origin.cast<double>() + 0.5 * 100 * resolution."""
    r = float(np.float32(resolution))
    o = np.asarray(origin, np.float32).reshape(-1)
    return (r, float(o[0]) + 0.5 * 100 * r, float(o[1]) + 0.5 * 100 * r, 100, 100)


class DeviceSubmap2D:
    """A ProbabilityGrid Submap2D whose grid lives on the device: .grid (a RealTimeGrid2D, the
    cropped grid once finished), .local_pose (x, y, 0, 1, 0, 0, 0) from the float origin,
    .num_range_data and .insertion_finished: what pose_graph.OverlappingSubmapsTrimmer2D reads.
    """

    def __init__(self, origin, resolution, device=0):
        o = np.asarray(origin, np.float32).reshape(-1)
        self.local_pose = (float(o[0]), float(o[1]), 0.0, 1.0, 0.0, 0.0, 0.0)
        res, max_x, max_y, nx, ny = create_grid_limits(o[:2], resolution)
        self.grid = RealTimeGrid2D.empty(res, max_x, max_y, nx, ny, device)
        self.num_range_data = 0
        self.insertion_finished = False

    def Finish(self):
        """Submap2D::Finish (submap_2d.cc:146-151): the grid becomes its crop; the uncropped
        handle is closed."""
        assert not self.insertion_finished
        cropped = self.grid.ComputeCroppedGrid()
        self.grid.close()
        self.grid = cropped
        self.insertion_finished = True

    def constraint_builder_submap(self):
        """The constraint_builder.Submap2D view ConstraintBuilder2D reads of a finished submap:
        the cropped grid and ComputeSubmapPose's (x, y, 0)."""
        from .constraint_builder import Submap2D
        if not self.insertion_finished:
            raise ValueError("DeviceSubmap2D: only a finished submap closes loops")
        return Submap2D(self.grid, (self.local_pose[0], self.local_pose[1], 0.0))


class ActiveSubmaps2D:
    """ActiveSubmaps2D (submap_2d.cc:153-236) over device grids: InsertRangeData writes each
    scan into the (at most two) active submaps with one csm_range_inserter2d_insert_submaps
    call.  ProbabilityGrid submaps only.  Evicted submaps are dropped from the list but stay
    alive while the caller holds them."""

    def __init__(self, options, device=0):
        if options.num_range_data <= 0:
            raise ValueError("num_range_data must be positive")
        if (options.grid_type != "PROBABILITY_GRID" or
                options.range_data_inserter_type != "PROBABILITY_GRID_INSERTER_2D"):
            raise ValueError("ActiveSubmaps2D on the device takes ProbabilityGrid submaps only")
        self.options = options
        self.device = device
        self.range_data_inserter = ProbabilityGridRangeDataInserter2D(
            options.probability_grid_range_data_inserter_options, device)
        self._submaps = []

    def submaps(self):
        return list(self._submaps)

    def InsertRangeData(self, origin, returns, misses=None):
        """origin (2 or 3), returns and misses (n x 3) in the local frame.  Returns the active
        submaps."""
        return self.insert_with(origin, lambda grids: self.range_data_inserter.insert_submaps(
            grids, origin, returns, misses))

    def insert_with(self, origin, insert):
        """InsertRangeData's lifecycle around insert(grids), which writes the scan whose local
        origin is `origin` into the active submaps' grids (local_slam.LocalTrajectoryBuilder2D
        inserts range data that stays on the device)."""
        n = self.options.num_range_data
        if not self._submaps or self._submaps[-1].num_range_data == n:
            self._add_submap(np.asarray(origin, np.float32).reshape(-1)[:2])
        for s in self._submaps:
            assert not s.insertion_finished
        insert([s.grid for s in self._submaps])
        for s in self._submaps:
            s.num_range_data += 1
        if self._submaps[0].num_range_data == 2 * n:
            self._submaps[0].Finish()
        return self.submaps()

    def _add_submap(self, origin):
        if len(self._submaps) >= 2:
            assert self._submaps[0].insertion_finished
            del self._submaps[0]
        self._submaps.append(DeviceSubmap2D(origin, self.options.resolution, self.device))


# ===========================================================================
# TSDFRangeDataInserter2D (mapping/internal/2d/tsdf_range_data_inserter_2d.h)
# ===========================================================================
class CsmTsdfInserterOptions2D(C.Structure):
    _fields_ = [("truncation_distance", C.c_double), ("maximum_weight", C.c_double),
                ("update_free_space", C.c_int32), ("num_normal_samples", C.c_int32),
                ("sample_radius", C.c_double),
                ("project_sdf_distance_to_scan_normal", C.c_int32),
                ("update_weight_range_exponent", C.c_int32),
                ("update_weight_angle_scan_normal_to_ray_kernel_bandwidth", C.c_double),
                ("update_weight_distance_cell_to_hit_kernel_bandwidth", C.c_double)]


@dataclass
class TSDFRangeDataInserterOptions2D:
    """proto TSDFRangeDataInserterOptions2D with NormalEstimationOptions2D flattened in; defaults
    are configuration_files/trajectory_builder_2d.lua's submaps.tsdf_range_data_inserter."""
    truncation_distance: float = 0.3
    maximum_weight: float = 10.0
    update_free_space: bool = False
    num_normal_samples: int = 4
    sample_radius: float = 0.5
    project_sdf_distance_to_scan_normal: bool = True
    update_weight_range_exponent: int = 0
    update_weight_angle_scan_normal_to_ray_kernel_bandwidth: float = 0.5
    update_weight_distance_cell_to_hit_kernel_bandwidth: float = 0.5

    def _c(self):
        return CsmTsdfInserterOptions2D(
            self.truncation_distance, self.maximum_weight, 1 if self.update_free_space else 0,
            self.num_normal_samples, self.sample_radius,
            1 if self.project_sdf_distance_to_scan_normal else 0,
            self.update_weight_range_exponent,
            self.update_weight_angle_scan_normal_to_ray_kernel_bandwidth,
            self.update_weight_distance_cell_to_hit_kernel_bandwidth)


class TSDFRangeDataInserter2D:
    """Insert(origin, returns, grid) writes one scan into a TSDF2D RealTimeGrid2D in place, as
    the reference's Insert(range_data, grid) writes a TSDF2D: origin (2 or 3) and returns (n x 3)
    are in the grid's frame.  The grid grows as the reference's does, and its `shape` follows."""

    def __init__(self, options=None, device=0):
        self.options = options or TSDFRangeDataInserterOptions2D()
        self.last_stats = None
        self._h = C.c_void_p()
        o = self.options._c()
        check(lib().csm_tsdf_inserter2d_create(C.byref(o), C.c_int32(device), C.byref(self._h)))

    def Insert(self, origin, returns, grid):
        org = np.zeros(3, np.float32)
        o = np.asarray(origin, np.float32).reshape(-1)
        org[:len(o)] = o[:3]
        ret = _f32(np.zeros((0, 3)) if returns is None else returns)
        stats = CsmStats()
        check(lib().csm_tsdf_inserter2d_insert(
            self._h, ptr(org, C.c_float), ptr(ret, C.c_float), C.c_int32(len(ret)), grid._h,
            C.byref(stats)))
        self.last_stats = stats.as_dict()
        grid._info()

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_tsdf_inserter2d_destroy(self._h)
            self._h = None

    __del__ = close


def _fast_from_device_grid(cls, grid, options):
    """FastCorrelativeScanMatcher2D over a ProbabilityGrid RealTimeGrid2D (typically a
    ComputeCroppedGrid result): the stack is built from the device cells
    (csm_stack2d_create_from_rt_grid2d)."""
    self = cls.__new__(cls)
    self.options, self.device, self.last_stats = options, grid.device, None
    self._h = C.c_void_p()
    check(lib().csm_stack2d_create_from_rt_grid2d(
        grid._h, C.c_int32(options.branch_and_bound_depth), C.byref(self._h)))
    return self


FastCorrelativeScanMatcher2D.from_device_grid = classmethod(_fast_from_device_grid)


def _rt_match_batch(self, initial_pose_estimates, point_clouds, rt_grid):
    """Many RealTimeCorrelativeScanMatcher2D::Match calls against one device-resident
    grid in one launch (csm_rt_match2d_batch).  Returns (scores[float64], poses[n, 3],
    stats dict); entry j equals Match(initial_pose_estimates[j], point_clouds[j], grid)."""
    n = len(point_clouds)
    clouds = [_f32(c) for c in point_clouds]
    jobs = (CsmRtJob2D * n)()
    for j in range(n):
        jobs[j].xyz = ptr(clouds[j], C.c_float)
        jobs[j].num_points = len(clouds[j])
        for k in range(3):
            jobs[j].initial_pose[k] = float(initial_pose_estimates[j][k])
    res = (CsmRtResult2D * n)()
    stats = CsmStats()
    o = self.options
    check(lib().csm_rt_match2d_batch(
        rt_grid._h, jobs, C.c_int32(n), C.c_double(o.linear_search_window),
        C.c_double(o.angular_search_window), C.c_double(o.translation_delta_cost_weight),
        C.c_double(o.rotation_delta_cost_weight), res, C.byref(stats)))
    self.last_stats = stats.as_dict()
    scores = np.array([r.score for r in res], np.float64)
    poses = np.array([[r.pose_estimate[0], r.pose_estimate[1], r.pose_estimate[2]] for r in res])
    self.last_results = res
    return scores, poses, self.last_stats


def _rt_scores_batch(self, initial_pose_estimates, point_clouds, rt_grid):
    """Test hook csm_rt_scores2d: MatchBatch run exactly, plus every candidate's weighted score.
    Returns (results, scores): results as MatchBatch's last_results, scores[j] job j's float32
    scores in generation order (scan, x offset, y offset)."""
    n = len(point_clouds)
    clouds = [_f32(c) for c in point_clouds]
    jobs = (CsmRtJob2D * n)()
    for j in range(n):
        jobs[j].xyz = ptr(clouds[j], C.c_float)
        jobs[j].num_points = len(clouds[j])
        for k in range(3):
            jobs[j].initial_pose[k] = float(initial_pose_estimates[j][k])
    res = (CsmRtResult2D * n)()
    o = self.options
    args = (rt_grid._h, jobs, C.c_int32(n), C.c_double(o.linear_search_window),
            C.c_double(o.angular_search_window), C.c_double(o.translation_delta_cost_weight),
            C.c_double(o.rotation_delta_cost_weight), res)
    check(lib().csm_rt_scores2d(*args, None))
    counts = [r.candidates_scored for r in res]
    flat = np.empty(sum(counts), np.float32)
    check(lib().csm_rt_scores2d(*args, ptr(flat, C.c_float)))
    return res, np.split(flat, np.cumsum(counts)[:-1])


def _rt_score_candidates(self, grid, discrete_scans, num_angular_perturbations,
                         angular_perturbation_step_size, candidates):
    """RealTimeCorrelativeScanMatcher2D::ScoreCandidates (public in the reference,
    real_time_correlative_scan_matcher_2d.h:75): candidates = [[scan, x_off, y_off], ...]."""
    cells = np.ascontiguousarray(grid.cells, dtype=np.uint16)
    ds = np.ascontiguousarray(discrete_scans, dtype=np.int32)
    cand = np.ascontiguousarray(candidates, dtype=np.int32).reshape(-1, 3)
    S, n, _ = ds.shape
    scores = np.empty(len(cand), np.float32)
    o = self.options
    check(lib().csm_rt_score_candidates2d(
        ptr(cells, C.c_uint16), C.c_int32(cells.shape[1]), C.c_int32(cells.shape[0]),
        C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
        ptr(ds, C.c_int32), C.c_int32(S), C.c_int32(n), C.c_int32(num_angular_perturbations),
        C.c_double(angular_perturbation_step_size), ptr(cand, C.c_int32), C.c_int32(len(cand)),
        C.c_double(o.translation_delta_cost_weight), C.c_double(o.rotation_delta_cost_weight),
        C.c_int32(self.device), ptr(scores, C.c_float)))
    return scores


RealTimeCorrelativeScanMatcher2D.MatchBatch = _rt_match_batch
RealTimeCorrelativeScanMatcher2D.ScoresBatch = _rt_scores_batch
RealTimeCorrelativeScanMatcher2D.ScoreCandidates = _rt_score_candidates


class MultiGpuContext:
    """csm_ctx: this process's place in a one-process-per-GPU job and its NCCL
    communicator (created inside the library).  Rank 0 calls MultiGpuContext.unique_id()
    and the 128 bytes are handed to every rank by the application (bench.py uses a
    torch.distributed object broadcast; a file or socket works as well)."""

    ID_BYTES = 128

    @staticmethod
    def unique_id():
        buf = (C.c_uint8 * MultiGpuContext.ID_BYTES)()
        check(lib().csm_comm_unique_id(buf))
        return bytes(buf)

    def __init__(self, world_size=1, rank=0, device=0, unique_id=None):
        self.world_size, self.rank, self.device = world_size, rank, device
        self._h = C.c_void_p()
        idbuf = None
        if world_size > 1:
            if unique_id is None or len(unique_id) != self.ID_BYTES:
                raise ValueError("unique_id (128 bytes from rank 0) is required for world_size > 1")
            idbuf = (C.c_uint8 * self.ID_BYTES).from_buffer_copy(unique_id)
        check(lib().csm_ctx_create(C.c_int32(world_size), C.c_int32(rank), C.c_int32(device),
                                   idbuf, C.byref(self._h)))

    def allgather(self, payload):
        """bytes -> list of world_size byte strings (one ncclAllGather)."""
        n = len(payload)
        send = (C.c_uint8 * max(1, n)).from_buffer_copy(payload if n else b"\0")
        recv = (C.c_uint8 * max(1, n * self.world_size))()
        check(lib().csm_ctx_allgather(self._h, send, C.c_int64(n), recv))
        raw = bytes(recv)
        return [raw[r * n:(r + 1) * n] for r in range(self.world_size)]

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_ctx_destroy(self._h)
            self._h = None

    __del__ = close


def match_batch_sharded(ctx, matchers, clouds, jobs, linear_search_window, angular_search_window,
                        submap_owner=None):
    """csm_cb_batch2d_run: the whole ConstraintBuilder2D queue on all GPUs of `ctx`.
    `matchers[s]` may be None on ranks that do not own submap s (owner = submap_owner[s],
    default s % world_size).  Every rank gets the results of ALL jobs, in job order."""
    jobs = np.ascontiguousarray(jobs, dtype=JOB2D_DTYPE)
    hs = (C.c_void_p * len(matchers))(*[(m._h if m is not None else None) for m in matchers])
    cs = (C.c_void_p * len(clouds))(*[(c._h if c is not None else None) for c in clouds])
    results = np.zeros(len(jobs), RESULT2D_DTYPE)
    stats = CsmStats()
    owner = None
    if submap_owner is not None:
        owner_arr = np.ascontiguousarray(submap_owner, dtype=np.int32)
        owner = ptr(owner_arr, C.c_int32)
    check(lib().csm_cb_batch2d_run(ctx._h, hs, C.c_int32(len(matchers)), cs,
                                   C.c_int32(len(clouds)), jobs.ctypes.data_as(C.c_void_p),
                                   C.c_int32(len(jobs)), owner, C.c_double(linear_search_window),
                                   C.c_double(angular_search_window),
                                   results.ctypes.data_as(C.c_void_p), C.byref(stats)))
    return results, stats.as_dict()


def kernel_launch_count():
    return int(lib().csm_kernel_launch_count())


def device_count():
    n = C.c_int32(0)
    check(lib().csm_device_count(C.byref(n)))
    return n.value


__all__ = ["FastCorrelativeScanMatcherOptions2D", "RealTimeCorrelativeScanMatcherOptions",
           "FastCorrelativeScanMatcher2D", "RealTimeCorrelativeScanMatcher2D", "DeviceCloud",
           "match_batch", "load_pbstream_matchers2d", "match_batch_sharded", "MultiGpuContext", "RealTimeGrid2D",
           "kernel_launch_count", "device_count", "JOB2D_DTYPE", "NODE2D_DTYPE",
           "RESULT2D_DTYPE", "_lib"]


# ===========================================================================
# 3D: FastCorrelativeScanMatcher3D (fast_correlative_scan_matcher_3d.h:66-101)
# ===========================================================================
class CsmOptions3D(C.Structure):
    _fields_ = [("branch_and_bound_depth", C.c_int32), ("full_resolution_depth", C.c_int32),
                ("min_rotational_score", C.c_double), ("min_low_resolution_score", C.c_double),
                ("linear_xy_search_window", C.c_double), ("linear_z_search_window", C.c_double),
                ("angular_search_window", C.c_double)]


class CsmNode3D(C.Structure):
    _fields_ = [("high_resolution_point_cloud", C.POINTER(C.c_float)), ("num_high", C.c_int32),
                ("low_resolution_point_cloud", C.POINTER(C.c_float)), ("num_low", C.c_int32),
                ("rotational_scan_matcher_histogram", C.POINTER(C.c_float)),
                ("histogram_size", C.c_int32), ("gravity_alignment", C.c_double * 4)]


# csm_bnb_node3d / csm_bnb_leaf3d: a 3D branch-and-bound frontier node and a recorded leaf
BNB_NODE3D_DTYPE = np.dtype([("scan", "<i4"), ("x", "<i4"), ("y", "<i4"), ("z", "<i4"),
                             ("score", "<f4")])
BNB_LEAF3D_DTYPE = np.dtype([("scan", "<i4"), ("x", "<i4"), ("y", "<i4"), ("z", "<i4"),
                             ("score", "<f4"), ("low", "<f4")])


class CsmResult3D(C.Structure):
    _fields_ = [("found", C.c_int32), ("score", C.c_float), ("pose_estimate", C.c_double * 7),
                ("rotational_score", C.c_float), ("low_resolution_score", C.c_float),
                ("best_scan_index", C.c_int32), ("best_offset", C.c_int32 * 3),
                ("leaves_tied", C.c_int32), ("reserved", C.c_int32)]


@dataclass
class FastCorrelativeScanMatcherOptions3D:
    """proto/scan_matching/fast_correlative_scan_matcher_options_3d.proto; defaults from
    configuration_files/pose_graph.lua:40-48."""
    branch_and_bound_depth: int = 8
    full_resolution_depth: int = 3
    min_rotational_score: float = 0.77
    min_low_resolution_score: float = 0.55
    linear_xy_search_window: float = 5.0
    linear_z_search_window: float = 1.0
    angular_search_window: float = 0.2617993877991494  # math.radians(15.)


@dataclass
class TrajectoryNodeData3D:
    """mapping/trajectory_node.h:45-63 — the fields the 3D matcher reads."""
    high_resolution_point_cloud: np.ndarray
    low_resolution_point_cloud: np.ndarray
    rotational_scan_matcher_histogram: np.ndarray
    gravity_alignment: tuple = (1.0, 0.0, 0.0, 0.0)


class _NodeHolder:
    def __init__(self, node):
        self.hi = _f32(node.high_resolution_point_cloud)
        lo = np.ascontiguousarray(node.low_resolution_point_cloud, np.float32).reshape(-1, 3)
        self.lo = lo
        self.hist = np.ascontiguousarray(node.rotational_scan_matcher_histogram,
                                         np.float32).reshape(-1)
        self.c = CsmNode3D()
        self.c.high_resolution_point_cloud = ptr(self.hi, C.c_float)
        self.c.num_high = len(self.hi)
        self.c.low_resolution_point_cloud = ptr(self.lo, C.c_float)
        self.c.num_low = len(self.lo)
        self.c.rotational_scan_matcher_histogram = ptr(self.hist, C.c_float)
        self.c.histogram_size = len(self.hist)
        self.c.gravity_alignment = (C.c_double * 4)(*[float(v) for v in node.gravity_alignment])


class FastCorrelativeScanMatcher3D:
    """FastCorrelativeScanMatcher3D(hybrid_grid, low_resolution_hybrid_grid,
    rotational_scan_matcher_histogram, options).  Grids are records with
    .resolution, .indices (n x 3 int32), .values (n uint16)."""

    def __init__(self, hybrid_grid, low_resolution_hybrid_grid,
                 rotational_scan_matcher_histogram, options, device=0, grid_size_in_voxels=0):
        self.options = options
        hist = np.ascontiguousarray(rotational_scan_matcher_histogram, np.float32).reshape(-1)
        hi_idx = np.ascontiguousarray(hybrid_grid.indices, np.int32).reshape(-1, 3)
        hi_val = np.ascontiguousarray(hybrid_grid.values, np.uint16).reshape(-1)
        lo_idx = np.ascontiguousarray(low_resolution_hybrid_grid.indices, np.int32).reshape(-1, 3)
        lo_val = np.ascontiguousarray(low_resolution_hybrid_grid.values, np.uint16).reshape(-1)
        o = CsmOptions3D(options.branch_and_bound_depth, options.full_resolution_depth,
                         options.min_rotational_score, options.min_low_resolution_score,
                         options.linear_xy_search_window, options.linear_z_search_window,
                         options.angular_search_window)
        self._h = C.c_void_p()
        check(lib().csm_matcher3d_create(
            ptr(hi_idx, C.c_int32), ptr(hi_val, C.c_uint16), C.c_int64(len(hi_val)),
            C.c_float(hybrid_grid.resolution), C.c_int32(grid_size_in_voxels),
            ptr(lo_idx, C.c_int32), ptr(lo_val, C.c_uint16), C.c_int64(len(lo_val)),
            C.c_float(low_resolution_hybrid_grid.resolution), ptr(hist, C.c_float),
            C.c_int32(len(hist)), C.byref(o), C.c_int32(device), C.byref(self._h)))
        self.last_stats = None

    @classmethod
    def from_proto(cls, serialized_hybrid_grid, serialized_low_resolution_hybrid_grid,
                   rotational_scan_matcher_histogram, options, device=0):
        """From two serialized cartographer.mapping.proto.HybridGrid messages
        (csm_matcher3d_create_from_proto)."""
        self = cls.__new__(cls)
        self.options, self.last_stats = options, None
        hist = np.ascontiguousarray(rotational_scan_matcher_histogram, np.float32).reshape(-1)
        o = CsmOptions3D(options.branch_and_bound_depth, options.full_resolution_depth,
                         options.min_rotational_score, options.min_low_resolution_score,
                         options.linear_xy_search_window, options.linear_z_search_window,
                         options.angular_search_window)
        hi, lo = serialized_hybrid_grid, serialized_low_resolution_hybrid_grid
        bh = (C.c_uint8 * len(hi)).from_buffer_copy(hi)
        bl = (C.c_uint8 * len(lo)).from_buffer_copy(lo)
        self._h = C.c_void_p()
        check(lib().csm_matcher3d_create_from_proto(bh, C.c_int64(len(hi)), bl, C.c_int64(len(lo)),
                                                    ptr(hist, C.c_float), C.c_int32(len(hist)),
                                                    C.byref(o), C.c_int32(device),
                                                    C.byref(self._h)))
        return self

    @classmethod
    def from_device_grids(cls, hybrid_grid, low_resolution_hybrid_grid,
                          rotational_scan_matcher_histogram, options, grid_size_in_voxels=0):
        """From two DeviceHybridGrids (typically filled by RangeDataInserter3D), device to
        device (csm_matcher3d_create_from_grid3d): the matcher the constructor builds from the
        grids' non-zero voxels, on the grids' device.  It owns its copies, so later inserts
        into the grids do not change it."""
        self = cls.__new__(cls)
        self.options, self.last_stats = options, None
        hist = np.ascontiguousarray(rotational_scan_matcher_histogram, np.float32).reshape(-1)
        o = CsmOptions3D(options.branch_and_bound_depth, options.full_resolution_depth,
                         options.min_rotational_score, options.min_low_resolution_score,
                         options.linear_xy_search_window, options.linear_z_search_window,
                         options.angular_search_window)
        self._h = C.c_void_p()
        check(lib().csm_matcher3d_create_from_grid3d(
            hybrid_grid._h, C.c_int32(grid_size_in_voxels), low_resolution_hybrid_grid._h,
            ptr(hist, C.c_float), C.c_int32(len(hist)), C.byref(o), C.byref(self._h)))
        return self

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_matcher3d_destroy(self._h)
            self._h = None

    __del__ = close

    def _match(self, full, node_pose, submap_pose, constant_data, min_score):
        res, self.last_stats = self.match_raw(full, node_pose, submap_pose, constant_data,
                                              min_score)
        return res

    def match_raw(self, full, node_pose, submap_pose, constant_data, min_score):
        """Thread-safe form (no state on self): -> (Result dict or None, stats dict).
        Like the reference's const Match*, it may be called from several threads at once;
        concurrent calls run on separate CUDA streams inside the library."""
        holder = _NodeHolder(constant_data)
        npose = np.ascontiguousarray(node_pose, np.float64)
        spose = np.ascontiguousarray(submap_pose, np.float64)
        res = CsmResult3D()
        stats = CsmStats()
        check(lib().csm_match3d(self._h, C.byref(holder.c), ptr(npose, C.c_double),
                                ptr(spose, C.c_double), C.c_int32(int(full)),
                                C.c_float(min_score), C.byref(res), C.byref(stats)))
        return _result3d_dict(res), stats.as_dict()

    def Match(self, global_node_pose, global_submap_pose, constant_data, min_score):
        """-> Result dict or None (nullptr), fast_correlative_scan_matcher_3d.cc:127-144.
        Poses are [tx, ty, tz, qw, qx, qy, qz]."""
        return self._match(False, global_node_pose, global_submap_pose, constant_data, min_score)

    def MatchFullSubmap(self, global_node_rotation, global_submap_rotation, constant_data,
                        min_score):
        """fast_correlative_scan_matcher_3d.cc:146-170; rotations are [qw, qx, qy, qz]."""
        return self._match(True, [0, 0, 0] + list(global_node_rotation),
                           [0, 0, 0] + list(global_submap_rotation), constant_data, min_score)

    # -- test hooks ------------------------------------------------------------------
    def precomputation_grid(self, depth, lo=None, dims=None):
        blo, bdims = np.zeros(3, np.int32), np.zeros(3, np.int32)
        check(lib().csm_matcher3d_read_level(self._h, C.c_int32(depth), ptr(blo, C.c_int32),
                                             ptr(bdims, C.c_int32), None))
        if lo is None:
            lo, dims = blo, bdims
        lo = np.ascontiguousarray(lo, np.int32)
        dims = np.ascontiguousarray(dims, np.int32)
        out = np.zeros((dims[2], dims[1], dims[0]), np.uint8)
        if out.size:
            check(lib().csm_matcher3d_read_level(self._h, C.c_int32(depth), ptr(lo, C.c_int32),
                                                 ptr(dims, C.c_int32), ptr(out, C.c_uint8)))
        return lo, out

    def discretize(self, full, node_pose, submap_pose, constant_data):
        holder = _NodeHolder(constant_data)
        npose = np.ascontiguousarray(node_pose, np.float64)
        spose = np.ascontiguousarray(submap_pose, np.float64)
        S = C.c_int32(0)
        args = (self._h, C.byref(holder.c), ptr(npose, C.c_double), ptr(spose, C.c_double),
                C.c_int32(int(full)), C.byref(S))
        check(lib().csm_discretize3d(*args, None, None, None))
        cells = np.zeros((S.value, len(holder.hi), 3), np.int32)
        poses = np.zeros((S.value, 7), np.float32)
        rot = np.zeros(S.value, np.float32)
        if S.value:
            check(lib().csm_discretize3d(*args, ptr(cells, C.c_int32), ptr(poses, C.c_float),
                                         ptr(rot, C.c_float)))
        return cells, poses, rot

    def _probe_args(self, full, node_pose, submap_pose, holder):
        npose = np.ascontiguousarray(node_pose, np.float64)
        spose = np.ascontiguousarray(submap_pose, np.float64)
        return (self._h, C.byref(holder.c), ptr(npose, C.c_double), ptr(spose, C.c_double),
                C.c_int32(int(full)))

    def score_candidates(self, full, node_pose, submap_pose, constant_data, candidates):
        """csm_score_candidates3d: `candidates` is n x {scan, x, y, z, depth}.
        -> (sums int32, scores float32) in the given order."""
        holder = _NodeHolder(constant_data)
        cand = np.ascontiguousarray(candidates, np.int32).reshape(-1, 5)
        sums = np.zeros(len(cand), np.int32)
        scores = np.zeros(len(cand), np.float32)
        check(lib().csm_score_candidates3d(
            *self._probe_args(full, node_pose, submap_pose, holder), ptr(cand, C.c_int32),
            C.c_int32(len(cand)), ptr(sums, C.c_int32), ptr(scores, C.c_float)))
        return sums, scores

    def score_top(self, full, node_pose, submap_pose, constant_data, min_score):
        """csm_score_top3d: the match up to and including its dives.  -> dict with
        angle (angle index per kept scan), rot (rotational scores), nxc, nzc,
        sums (num_scans x nzc x nxc x nxc: [scan, z, y, x]), top_best, bound and
        counters (candidates scored by the dives, gate evaluations)."""
        holder = _NodeHolder(constant_data)
        args = self._probe_args(full, node_pose, submap_pose, holder) + (C.c_float(min_score),)
        S = C.c_int32(0)
        lat = np.zeros(2, np.int32)
        check(lib().csm_score_top3d(*args, C.byref(S), ptr(lat, C.c_int32), None, None, None,
                                    None, None, None))
        S, nxc, nzc = S.value, int(lat[0]), int(lat[1])
        angle = np.zeros(S, np.int32)
        rot = np.zeros(S, np.float32)
        sums = np.zeros((S, nzc, nxc, nxc), np.int32)
        best, bound = C.c_int32(0), C.c_float(0)
        ctr = np.zeros(2, np.int64)
        S2 = C.c_int32(0)
        check(lib().csm_score_top3d(*args, C.byref(S2), ptr(lat, C.c_int32), ptr(angle, C.c_int32),
                                    ptr(rot, C.c_float), ptr(sums, C.c_int32), C.byref(best),
                                    C.byref(bound), ptr(ctr, C.c_int64)))
        assert S2.value == S
        return dict(angle=angle, rot=rot, nxc=nxc, nzc=nzc, sums=sums, top_best=best.value,
                    bound=np.float32(bound.value), counters=(int(ctr[0]), int(ctr[1])))

    def branch_step(self, full, node_pose, submap_pose, constant_data, min_score, level,
                    parents, bound):
        """csm_branch_step3d over `parents` (BNB_NODE3D_DTYPE records) of `level` with the
        bound set to `bound`.  -> (children in queue order (level >= 2) or leaves
        (BNB_LEAF3D_DTYPE, level 1), final bound, (candidates scored, parents expanded,
        gate evaluations))."""
        holder = _NodeHolder(constant_data)
        par = np.ascontiguousarray(parents, dtype=BNB_NODE3D_DTYPE)
        out = np.zeros(max(1, 8 * len(par)), BNB_NODE3D_DTYPE if level >= 2 else BNB_LEAF3D_DTYPE)
        count, final = C.c_int32(0), C.c_float(0.0)
        ctr = np.zeros(3, np.int64)
        optr = out.ctypes.data_as(C.c_void_p)
        check(lib().csm_branch_step3d(
            *self._probe_args(full, node_pose, submap_pose, holder), C.c_float(min_score),
            C.c_int32(level), par.ctypes.data_as(C.c_void_p), C.c_int32(len(par)),
            C.c_float(bound), optr if level >= 2 else None, None if level >= 2 else optr,
            C.byref(count), C.byref(final), ptr(ctr, C.c_int64)))
        return out[:count.value].copy(), np.float32(final.value), tuple(int(c) for c in ctr)

    def top_queue(self, full, node_pose, submap_pose, constant_data, min_score, dive_ratio):
        """csm_top_queue3d: the match through its dives (at `dive_ratio`) and its top-queue
        filter.  -> (bound the level loop starts from, top queue as BNB_NODE3D_DTYPE records).
        The queue is filled by atomic appends: its order is not deterministic."""
        holder = _NodeHolder(constant_data)
        args = self._probe_args(full, node_pose, submap_pose, holder) + (
            C.c_float(min_score), C.c_float(dive_ratio))
        bound, count = C.c_float(0.0), C.c_int32(0)
        out = np.zeros(1024, BNB_NODE3D_DTYPE)
        while True:
            check(lib().csm_top_queue3d(*args, C.byref(bound), out.ctypes.data_as(C.c_void_p),
                                        C.c_int32(len(out)), C.byref(count)))
            if count.value <= len(out):
                break
            out = np.zeros(count.value, BNB_NODE3D_DTYPE)
        return np.float32(bound.value), out[:count.value].copy()


class SweepLimits3D(C.Structure):
    """csm_sweep_limits3d: limits of the 3D branch-and-bound sweep."""
    _fields_ = [("chunk", C.c_int32), ("leaf_cap", C.c_int32), ("inline_best", C.c_int32),
                ("dive_ratio", C.c_float)]

    @classmethod
    def default(cls):
        out = cls()
        lib().csm_sweep_limits3d_default(C.byref(out))
        return out


class CsmJob3D(C.Structure):
    _fields_ = [("matcher_index", C.c_int32), ("node_index", C.c_int32),
                ("full_submap", C.c_int32), ("min_score", C.c_float),
                ("global_node_pose", C.c_double * 7), ("global_submap_pose", C.c_double * 7)]


def _result3d_dict(res):
    if not res.found:
        return None
    return dict(score=np.float32(res.score), pose_estimate=np.array(res.pose_estimate[:]),
                rotational_score=np.float32(res.rotational_score),
                low_resolution_score=np.float32(res.low_resolution_score),
                best_scan_index=res.best_scan_index, best_offset=tuple(res.best_offset[:]),
                leaves_tied=res.leaves_tied)


def match_batch3d(matchers, nodes, jobs, max_concurrency=0, ctx=None, submap_owner=None,
                  limits=None):
    """csm_match3d_batch: a queue of ConstraintBuilder3D searches in one call.
    jobs: iterable of (matcher_index, node_index, full_submap, global_node_pose[7],
    global_submap_pose[7], min_score).  -> ([Result dict or None per job], stats dict).
    With `ctx` (MultiGpuContext) the queue is sharded over the GPUs (csm_cb_batch3d_run:
    matcher m runs on rank submap_owner[m], default m % world_size; matchers[m] may be None
    elsewhere) and every rank gets all results after one ncclAllGather.
    limits: None (the defaults), a SweepLimits3D, or a dict of SweepLimits3D fields that
    override the defaults (csm_match3d_batch_limits; not with `ctx`); then
    stats["sweep_trace"] is (collects summed over the jobs, most leaves recorded by one
    match, optimal leaves summed)."""
    if limits is not None and ctx is not None:
        raise ValueError("sweep limits apply to the unsharded batch only")
    jobs = list(jobs)
    holders = [_NodeHolder(n) for n in nodes]
    c_nodes = (CsmNode3D * max(1, len(holders)))(*[h.c for h in holders])
    c_matchers = (C.c_void_p * max(1, len(matchers)))(
        *[(m._h if m is not None else None) for m in matchers])
    c_jobs = (CsmJob3D * max(1, len(jobs)))()
    for k, (mi, ni, full, npose, spose, min_score) in enumerate(jobs):
        c_jobs[k].matcher_index = int(mi)
        c_jobs[k].node_index = int(ni)
        c_jobs[k].full_submap = int(bool(full))
        c_jobs[k].min_score = float(min_score)
        c_jobs[k].global_node_pose = (C.c_double * 7)(*[float(v) for v in npose])
        c_jobs[k].global_submap_pose = (C.c_double * 7)(*[float(v) for v in spose])
    c_res = (CsmResult3D * max(1, len(jobs)))()
    stats = CsmStats()
    trace = None
    if limits is not None:
        if isinstance(limits, dict):
            lim = SweepLimits3D.default()
            for k, v in limits.items():
                setattr(lim, k, v)
            limits = lim
        trace = np.zeros(3, np.int32)
        check(lib().csm_match3d_batch_limits(
            c_matchers, C.c_int32(len(matchers)), c_nodes, C.c_int32(len(holders)), c_jobs,
            C.c_int32(len(jobs)), C.c_int32(int(max_concurrency)), C.byref(limits), c_res,
            C.byref(stats), ptr(trace, C.c_int32)))
    elif ctx is None:
        check(lib().csm_match3d_batch(c_matchers, C.c_int32(len(matchers)), c_nodes,
                                      C.c_int32(len(holders)), c_jobs, C.c_int32(len(jobs)),
                                      C.c_int32(int(max_concurrency)), c_res, C.byref(stats)))
    else:
        owner = None
        if submap_owner is not None:
            owner_arr = np.ascontiguousarray(submap_owner, dtype=np.int32)
            owner = ptr(owner_arr, C.c_int32)
        check(lib().csm_cb_batch3d_run(ctx._h, c_matchers, C.c_int32(len(matchers)), c_nodes,
                                       C.c_int32(len(holders)), c_jobs, C.c_int32(len(jobs)),
                                       owner, C.c_int32(int(max_concurrency)), c_res,
                                       C.byref(stats)))
    out = stats.as_dict()
    if trace is not None:
        out["sweep_trace"] = tuple(int(v) for v in trace)
    return [_result3d_dict(c_res[k]) for k in range(len(jobs))], out


def rotational_match(submap_histogram, histogram, initial_angle, angles, device=0):
    """RotationalScanMatcher::Match (rotational_scan_matcher.cc:178-189) on the device."""
    a = np.ascontiguousarray(submap_histogram, np.float32).reshape(-1)
    b = np.ascontiguousarray(histogram, np.float32).reshape(-1)
    ang = np.ascontiguousarray(angles, np.float32).reshape(-1)
    out = np.zeros(len(ang), np.float32)
    check(lib().csm_rotational_match3d(ptr(a, C.c_float), ptr(b, C.c_float), C.c_int32(len(a)),
                                       C.c_float(initial_angle), ptr(ang, C.c_float),
                                       C.c_int32(len(ang)), C.c_int32(device),
                                       ptr(out, C.c_float)))
    return out


# ===========================================================================
# RealTimeCorrelativeScanMatcher3D (real_time_correlative_scan_matcher_3d.h:41-67)
# ===========================================================================
class DeviceHybridGrid:
    """A HybridGrid resident on the device (csm_grid3d); `hybrid_grid` is any record with
    resolution, indices (n x 3 int32) and values (n uint16) — proto::HybridGrid's flat form."""

    def __init__(self, hybrid_grid, device=0):
        idx = np.ascontiguousarray(hybrid_grid.indices, dtype=np.int32).reshape(-1, 3)
        val = np.ascontiguousarray(hybrid_grid.values, dtype=np.uint16).reshape(-1)
        self.resolution = float(hybrid_grid.resolution)
        self._h = C.c_void_p()
        check(lib().csm_grid3d_create(ptr(idx, C.c_int32), ptr(val, C.c_uint16),
                                      C.c_int64(len(val)), C.c_float(self.resolution),
                                      C.c_int32(device), C.byref(self._h)))

    @classmethod
    def empty(cls, resolution, device=0):
        """The grid of a fresh submap: no voxels, filled by RangeDataInserter3D.Insert."""
        return cls(_EmptyGrid(resolution, np.zeros((0, 3), np.int32), np.zeros(0, np.uint16)),
                   device)

    def read(self):
        """(lo, values): the dense box, values[z, y, x] of voxel lo + (x, y, z)."""
        lo, dims = np.zeros(3, np.int32), np.zeros(3, np.int32)
        check(lib().csm_grid3d_read(self._h, ptr(lo, C.c_int32), ptr(dims, C.c_int32), None))
        out = np.zeros(tuple(dims[::-1]), np.uint16)
        check(lib().csm_grid3d_read(self._h, ptr(lo, C.c_int32), ptr(dims, C.c_int32),
                                    ptr(out, C.c_uint16)))
        return lo, out

    def voxels(self):
        """(indices, values): the non-zero voxels in HybridGrid's iteration order, the order
        HybridGrid::ToProto writes them (csm_grid3d_voxels) — n x 3 int32 and n uint16."""
        n = C.c_int64()
        check(lib().csm_grid3d_voxels(self._h, None, None, C.c_int64(0), C.byref(n)))
        idx = np.zeros((n.value, 3), np.int32)
        val = np.zeros(n.value, np.uint16)
        if n.value:
            check(lib().csm_grid3d_voxels(self._h, ptr(idx, C.c_int32), ptr(val, C.c_uint16),
                                          C.c_int64(n.value), C.byref(n)))
        return idx, val

    def to_proto(self):
        """The serialised proto::HybridGrid that HybridGrid::ToProto gives for this grid
        (csm_grid3d_to_proto), as bytes."""
        n = C.c_int64()
        check(lib().csm_grid3d_voxels(self._h, None, None, C.c_int64(0), C.byref(n)))
        # resolution, four packed-field headers, at most 5 bytes per index and 3 per value
        return _serialize(lib().csm_grid3d_to_proto, self._h, 5 + 4 * 11 + 18 * n.value)

    def to_texture(self, global_submap_pose):
        """The serialised proto::SubmapQuery::Response::SubmapTexture that AddToTextureProto
        draws for this grid under the global submap pose (tx, ty, tz, qw, qx, qy, qz):
        Submap3D::ToResponseProto adds the high-resolution grid's texture, then the
        low-resolution grid's (csm_grid3d_to_texture), as bytes."""
        return _texture(lib().csm_grid3d_to_texture, self._h, global_submap_pose)

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_grid3d_destroy(self._h)
            self._h = None

    __del__ = close


@dataclass
class _EmptyGrid:
    resolution: float
    indices: np.ndarray
    values: np.ndarray


@dataclass
class IntensityGridSpec:
    """An IntensityHybridGrid (mapping/3d/hybrid_grid.h:547-570) in the flat form
    HybridGridBase<AverageIntensityData>::Iterator gives: indices (n x 3 int32), sums (n
    float32) and counts (n int32) of each voxel's AverageIntensityData."""
    resolution: float
    indices: np.ndarray
    sums: np.ndarray
    counts: np.ndarray


class DeviceIntensityGrid:
    """An IntensityHybridGrid resident on the device (csm_intensity_grid3d): GetIntensity of
    every voxel of an IntensityGridSpec, 0 outside them."""

    def __init__(self, intensity_grid, device=0):
        idx = np.ascontiguousarray(intensity_grid.indices, dtype=np.int32).reshape(-1, 3)
        sums = np.ascontiguousarray(intensity_grid.sums, dtype=np.float32).reshape(-1)
        counts = np.ascontiguousarray(intensity_grid.counts, dtype=np.int32).reshape(-1)
        if not len(idx) == len(sums) == len(counts):
            raise ValueError("indices, sums and counts differ in length")
        self.resolution = float(intensity_grid.resolution)
        self._h = C.c_void_p()
        check(lib().csm_intensity_grid3d_create(
            ptr(idx, C.c_int32), ptr(sums, C.c_float), ptr(counts, C.c_int32),
            C.c_int64(len(counts)), C.c_float(self.resolution), C.c_int32(device),
            C.byref(self._h)))

    @classmethod
    def empty(cls, resolution, device=0):
        """The intensity grid of a fresh submap: no voxels."""
        return cls(IntensityGridSpec(resolution, np.zeros((0, 3), np.int32),
                                     np.zeros(0, np.float32), np.zeros(0, np.int32)), device)

    def read(self):
        """(lo, mean, sum, count): the dense box, each indexed [z, y, x] from voxel lo;
        mean is GetIntensity, sum / count each voxel's AverageIntensityData."""
        lo, dims = np.zeros(3, np.int32), np.zeros(3, np.int32)
        check(lib().csm_intensity_grid3d_read(self._h, ptr(lo, C.c_int32), ptr(dims, C.c_int32),
                                              None, None, None))
        shape = tuple(dims[::-1])
        mean, sums = np.zeros(shape, np.float32), np.zeros(shape, np.float32)
        counts = np.zeros(shape, np.int32)
        check(lib().csm_intensity_grid3d_read(
            self._h, ptr(lo, C.c_int32), ptr(dims, C.c_int32), ptr(mean, C.c_float),
            ptr(sums, C.c_float), ptr(counts, C.c_int32)))
        return lo, mean, sums, counts

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_intensity_grid3d_destroy(self._h)
            self._h = None

    __del__ = close


# ===========================================================================
# RangeDataInserter3D (mapping/3d/range_data_inserter_3d.h)
# ===========================================================================
class CsmRangeInserterOptions3D(C.Structure):
    _fields_ = [("hit_probability", C.c_double), ("miss_probability", C.c_double),
                ("num_free_space_voxels", C.c_int32), ("intensity_threshold", C.c_float)]


@dataclass
class RangeDataInserterOptions3D:
    """proto RangeDataInserterOptions3D (mapping/proto/range_data_inserter_options_3d.proto);
    defaults are configuration_files/trajectory_builder_3d.lua's submaps.range_data_inserter."""
    hit_probability: float = 0.55
    miss_probability: float = 0.49
    num_free_space_voxels: int = 2
    intensity_threshold: float = 40.0

    def _c(self):
        return CsmRangeInserterOptions3D(self.hit_probability, self.miss_probability,
                                         self.num_free_space_voxels, self.intensity_threshold)


class RangeDataInserter3D:
    """Insert(origin, returns, intensities, grid, intensity_grid=None) writes one scan into a
    DeviceHybridGrid and, with intensities, a DeviceIntensityGrid, as the reference's
    RangeDataInserter3D::Insert writes a HybridGrid / IntensityHybridGrid.  origin (3) and
    returns (n x 3) are in the grid's frame; intensities (n) may be None."""

    def __init__(self, options, device=0):
        self.options = options
        self.last_stats = None
        self._h = C.c_void_p()
        o = options._c()
        check(lib().csm_range_inserter3d_create(C.byref(o), C.c_int32(device),
                                                C.byref(self._h)))

    def Insert(self, origin, returns, intensities, grid, intensity_grid=None):
        org = np.ascontiguousarray(origin, dtype=np.float32).reshape(3)
        xyz = _f32(returns)
        inten = None
        if intensities is not None:
            inten = np.ascontiguousarray(intensities, dtype=np.float32).reshape(-1)
            if len(inten) != len(xyz):
                raise ValueError("intensities and returns differ in length")
        stats = CsmStats()
        check(lib().csm_range_inserter3d_insert(
            self._h, ptr(org, C.c_float), ptr(xyz, C.c_float),
            None if inten is None else ptr(inten, C.c_float), C.c_int32(len(xyz)), grid._h,
            None if intensity_grid is None else intensity_grid._h, C.byref(stats)))
        self.last_stats = stats.as_dict()

    def insert_submaps(self, submaps, origin, returns, intensities, high_resolution_max_range):
        """Submap3D::InsertData's inserts (submap_3d.cc:271-287) into several submaps in one
        call (csm_range_inserter3d_insert_submaps).  `submaps`: (local_pose, high_resolution,
        low_resolution, intensity) tuples, local_pose (tx, ty, tz, qw, qx, qy, qz), the grids
        DeviceHybridGrids and intensity a DeviceIntensityGrid or None.  origin (3), returns
        (n x 3) and intensities (n, or None) are in the local frame."""
        entries = (CsmSubmapInsert3D * len(submaps))()
        for e, (pose, high, low, intensity) in zip(entries, submaps):
            e.local_pose[:] = [float(v) for v in pose]
            e.high_resolution = high._h
            e.low_resolution = low._h
            e.intensity = None if intensity is None else intensity._h
        org = np.ascontiguousarray(origin, dtype=np.float32).reshape(3)
        xyz = _f32(returns)
        inten = None
        if intensities is not None:
            inten = np.ascontiguousarray(intensities, dtype=np.float32).reshape(-1)
            if len(inten) != len(xyz):
                raise ValueError("intensities and returns differ in length")
        stats = CsmStats()
        check(lib().csm_range_inserter3d_insert_submaps(
            self._h, entries, C.c_int32(len(submaps)), ptr(org, C.c_float), ptr(xyz, C.c_float),
            None if inten is None else ptr(inten, C.c_float), C.c_int32(len(xyz)),
            C.c_float(high_resolution_max_range), C.byref(stats)))
        self.last_stats = stats.as_dict()

    def close(self):
        if getattr(self, "_h", None):
            lib().csm_range_inserter3d_destroy(self._h)
            self._h = None

    __del__ = close


class CsmSubmapInsert3D(C.Structure):
    _fields_ = [("local_pose", C.c_double * 7), ("high_resolution", C.c_void_p),
                ("low_resolution", C.c_void_p), ("intensity", C.c_void_p)]


# ===========================================================================
# Submap3D and ActiveSubmaps3D (mapping/3d/submap_3d.h) over device grids
# ===========================================================================
@dataclass
class SubmapsOptions3D:
    """proto SubmapsOptions3D (mapping/proto/submaps_options_3d.proto); defaults are
    configuration_files/trajectory_builder_3d.lua's submaps."""
    high_resolution: float = 0.10
    high_resolution_max_range: float = 20.0
    low_resolution: float = 0.45
    num_range_data: int = 160
    range_data_inserter_options: RangeDataInserterOptions3D = field(
        default_factory=RangeDataInserterOptions3D)


def yaw_in_submap_from_gravity(local_pose, local_from_gravity_aligned):
    """transform::GetYaw(local_pose.inverse().rotation() * local_from_gravity_aligned) in
    double (submap_3d.cc:289-290), as the float InsertData passes on.  Quaternions are
    (w, x, y, z); the product and the rotation of UnitX in Eigen's scalar order."""
    pw, px, py, pz = (float(local_pose[3]), -float(local_pose[4]), -float(local_pose[5]),
                      -float(local_pose[6]))
    qw, qx, qy, qz = (float(v) for v in local_from_gravity_aligned)
    w = pw * qw - px * qx - py * qy - pz * qz
    x = pw * qx + px * qw + py * qz - pz * qy
    y = pw * qy + py * qw + pz * qx - px * qz
    z = pw * qz + pz * qw + px * qy - py * qx
    # q * UnitX (_transformVector): uv = q.vec x v, uv += uv, v + w uv + q.vec x uv, with
    # every product of the zeros of UnitX kept (they decide the sign of a zero y)
    v = (1.0, 0.0, 0.0)
    uv = [y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0]]
    uv = [u + u for u in uv]
    cross = (y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0])
    dx = v[0] + w * uv[0] + cross[0]
    dy = v[1] + w * uv[1] + cross[1]
    return np.float32(math.atan2(dy, dx))


def rotate_histogram(histogram, angle):
    """RotationalScanMatcher::RotateHistogram (rotational_scan_matcher.cc:141-162) in float."""
    h = np.ascontiguousarray(histogram, np.float32).reshape(-1)
    size = len(h)
    if size == 0:
        return h.copy()
    rotate_by_buckets = np.float32(float(-np.float32(angle) * np.float32(size)) / math.pi)
    v = np.float32(rotate_by_buckets - np.float32(0.5))
    full = int(math.floor(abs(float(v)) + 0.5) * (1 if v >= 0 else -1))   # std::lround
    fraction = np.float32(rotate_by_buckets - np.float32(full))
    full %= size
    r0 = np.roll(h, -full)
    r1 = np.roll(h, -(full + 1))
    return (fraction * r1 + (np.float32(1) - fraction) * r0).astype(np.float32)


class DeviceSubmap3D:
    """A Submap3D whose grids live on the device: local_pose (tx, ty, tz, qw, qx, qy, qz),
    the high- and low-resolution DeviceHybridGrids, the high-resolution DeviceIntensityGrid
    (None once forgotten), num_range_data, insertion_finished and the float32 rotational scan
    matcher histogram, accumulated on the host."""

    def __init__(self, options, local_pose, histogram_size, device=0):
        self.local_pose = tuple(float(v) for v in local_pose)
        self.high_resolution_hybrid_grid = DeviceHybridGrid.empty(options.high_resolution,
                                                                  device)
        self.low_resolution_hybrid_grid = DeviceHybridGrid.empty(options.low_resolution, device)
        self.high_resolution_intensity_hybrid_grid = DeviceIntensityGrid.empty(
            options.high_resolution, device)
        self.rotational_scan_matcher_histogram = np.zeros(histogram_size, np.float32)
        self.num_range_data = 0
        self.insertion_finished = False

    def Finish(self):
        assert not self.insertion_finished
        self.insertion_finished = True

    def ForgetIntensityHybridGrid(self):
        if self.high_resolution_intensity_hybrid_grid is not None:
            self.high_resolution_intensity_hybrid_grid.close()
        self.high_resolution_intensity_hybrid_grid = None

    def constraint_builder_submap(self):
        """The constraint_builder.Submap3D view ConstraintBuilder3D reads."""
        from .constraint_builder import Submap3D
        return Submap3D(self.high_resolution_hybrid_grid, self.low_resolution_hybrid_grid,
                        self.rotational_scan_matcher_histogram)


class ActiveSubmaps3D:
    """ActiveSubmaps3D (submap_3d.cc:296-351) over device grids: InsertData writes each scan
    into the (at most two) active submaps with one csm_range_inserter3d_insert_submaps call.
    Evicted submaps are dropped from the list but stay alive while the caller holds them."""

    def __init__(self, options, device=0):
        self.options = options
        self.device = device
        self.range_data_inserter = RangeDataInserter3D(options.range_data_inserter_options,
                                                       device)
        self._submaps = []

    def submaps(self):
        return list(self._submaps)

    def InsertData(self, origin, returns, intensities, local_from_gravity_aligned,
                   rotational_scan_matcher_histogram_in_gravity):
        """origin (3), returns (n x 3), intensities (n or None) in the local frame;
        local_from_gravity_aligned (w, x, y, z).  Returns the active submaps."""
        hist = np.ascontiguousarray(rotational_scan_matcher_histogram_in_gravity,
                                    np.float32).reshape(-1)
        if (not self._submaps or
                self._submaps[-1].num_range_data == self.options.num_range_data):
            org = np.asarray(origin, np.float32).reshape(3)
            self._add_submap([float(org[0]), float(org[1]), float(org[2])] +
                             [float(v) for v in local_from_gravity_aligned], len(hist))
        self.range_data_inserter.insert_submaps(
            [(s.local_pose, s.high_resolution_hybrid_grid, s.low_resolution_hybrid_grid,
              s.high_resolution_intensity_hybrid_grid) for s in self._submaps],
            origin, returns, intensities, self.options.high_resolution_max_range)
        for s in self._submaps:
            assert not s.insertion_finished
            s.num_range_data += 1
            yaw = yaw_in_submap_from_gravity(s.local_pose, local_from_gravity_aligned)
            s.rotational_scan_matcher_histogram = (s.rotational_scan_matcher_histogram +
                                                   rotate_histogram(hist, yaw))
        if self._submaps[0].num_range_data == 2 * self.options.num_range_data:
            self._submaps[0].Finish()
        return self.submaps()

    def _add_submap(self, local_pose, histogram_size):
        if len(self._submaps) >= 2:
            assert self._submaps[0].insertion_finished
            self._submaps[0].ForgetIntensityHybridGrid()
            del self._submaps[0]
        self._submaps.append(DeviceSubmap3D(self.options, local_pose, histogram_size,
                                            self.device))


class RealTimeCorrelativeScanMatcher3D:
    """Match(initial_pose_estimate, point_cloud, hybrid_grid) -> (score, pose_estimate);
    poses are {tx, ty, tz, qw, qx, qy, qz}.  `hybrid_grid` is a DeviceHybridGrid."""

    def __init__(self, options):
        self.options = options
        self.last_stats = None

    def Match(self, initial_pose_estimate, point_cloud, hybrid_grid):
        xyz = _f32(point_cloud)
        ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
        pose = np.zeros(7, np.float64)
        score = C.c_float(0.0)
        stats = CsmStats()
        o = self.options
        check(lib().csm_rt_match3d(
            hybrid_grid._h, ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
            C.c_double(o.linear_search_window), C.c_double(o.angular_search_window),
            C.c_double(o.translation_delta_cost_weight),
            C.c_double(o.rotation_delta_cost_weight), C.byref(score), ptr(pose, C.c_double),
            C.byref(stats)))
        self.last_stats = stats.as_dict()
        return np.float32(score.value), pose

    def Scores(self, initial_pose_estimate, point_cloud, hybrid_grid):
        """Test hook csm_rt_scores3d: every candidate's weighted score of Match, float32 in
        generation order (translations z, y, x, then rotations rz, ry, rx)."""
        xyz = _f32(point_cloud)
        ip = np.ascontiguousarray(initial_pose_estimate, dtype=np.float64)
        o = self.options
        count = C.c_int64(0)
        args = (hybrid_grid._h, ptr(xyz, C.c_float), C.c_int32(len(xyz)), ptr(ip, C.c_double),
                C.c_double(o.linear_search_window), C.c_double(o.angular_search_window),
                C.c_double(o.translation_delta_cost_weight),
                C.c_double(o.rotation_delta_cost_weight))
        check(lib().csm_rt_scores3d(*args, None, C.byref(count)))
        scores = np.empty(count.value, np.float32)
        check(lib().csm_rt_scores3d(*args, ptr(scores, C.c_float), C.byref(count)))
        return scores


# ===========================================================================
# CeresScanMatcher2D (mapping/internal/2d/scan_matching/ceres_scan_matcher_2d.{h,cc})
# ===========================================================================
class CsmCeresOptions2D(C.Structure):
    _fields_ = [("occupied_space_weight", C.c_double), ("translation_weight", C.c_double),
                ("rotation_weight", C.c_double), ("use_nonmonotonic_steps", C.c_int32),
                ("max_num_iterations", C.c_int32)]


class CsmCeresJob2D(C.Structure):
    _fields_ = [("grid", C.c_void_p), ("xyz", C.POINTER(C.c_float)), ("num_points", C.c_int32),
                ("reserved", C.c_int32), ("target_translation", C.c_double * 2),
                ("initial_pose", C.c_double * 3)]


class CsmCeresResult2D(C.Structure):
    _fields_ = [("pose_estimate", C.c_double * 3), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("iterations", C.c_int32),
                ("num_successful_steps", C.c_int32), ("termination", C.c_int32),
                ("reserved", C.c_int32)]


CERES_TERMINATION = ("NO_CONVERGENCE", "FUNCTION_TOLERANCE", "GRADIENT_TOLERANCE",
                     "PARAMETER_TOLERANCE", "MIN_TRUST_REGION_RADIUS", "INVALID_STEPS",
                     "EVALUATION_FAILED")


@dataclass
class CeresScanMatcherOptions2D:
    """proto/scan_matching/ceres_scan_matcher_options_2d.proto +
    common/proto/ceres_solver_options.proto; defaults = the constraint builder's
    (configuration_files/pose_graph.lua:30-39).  num_threads has no meaning here."""
    occupied_space_weight: float = 20.0
    translation_weight: float = 10.0
    rotation_weight: float = 1.0
    use_nonmonotonic_steps: bool = True
    max_num_iterations: int = 10

    def _c(self):
        return CsmCeresOptions2D(self.occupied_space_weight, self.translation_weight,
                                 self.rotation_weight, int(self.use_nonmonotonic_steps),
                                 int(self.max_num_iterations))


class CeresScanMatcher2D:
    """ceres_scan_matcher_2d.h:42-64.  `grid` arguments are RealTimeGrid2D handles (the
    submap's ProbabilityGrid or TSDF2D resident on the device; the grid type selects the cost
    function, as GetGridType() does).  Match returns (pose_estimate, summary) where the
    reference fills *pose_estimate and a ceres::Solver::Summary."""

    def __init__(self, options=None):
        self.options = options if options is not None else CeresScanMatcherOptions2D()

    def Match(self, target_translation, initial_pose_estimate, point_cloud, grid):
        poses, summaries = self.MatchBatch([target_translation], [initial_pose_estimate],
                                           [point_cloud], [grid])
        return poses[0], summaries[0]

    def MatchBatch(self, target_translations, initial_pose_estimates, point_clouds, grids):
        """Many Match calls in one launch (csm_ceres_match2d_batch); grids[j] may differ per
        job (one per submap) but must live on one device."""
        n = len(point_clouds)
        clouds = [_f32(c) for c in point_clouds]
        jobs = (CsmCeresJob2D * n)()
        for j in range(n):
            jobs[j].grid = grids[j]._h
            jobs[j].xyz = ptr(clouds[j], C.c_float)
            jobs[j].num_points = len(clouds[j])
            jobs[j].target_translation[0] = float(target_translations[j][0])
            jobs[j].target_translation[1] = float(target_translations[j][1])
            for k in range(3):
                jobs[j].initial_pose[k] = float(initial_pose_estimates[j][k])
        res = (CsmCeresResult2D * n)()
        stats = CsmStats()
        opt = self.options._c()
        check(lib().csm_ceres_match2d_batch(jobs, C.c_int32(n), C.byref(opt), res,
                                            C.byref(stats)))
        self.last_stats = stats.as_dict()
        poses = np.array([[r.pose_estimate[0], r.pose_estimate[1], r.pose_estimate[2]]
                          for r in res], np.float64)
        summaries = [dict(initial_cost=r.initial_cost, final_cost=r.final_cost,
                          iterations=r.iterations, num_successful_steps=r.num_successful_steps,
                          termination=CERES_TERMINATION[r.termination]) for r in res]
        return poses, summaries

    def Evaluate(self, grid, point_cloud, pose, target_translation, target_angle, jacobian=True):
        """Residuals (n + 3) and Jacobian ((n + 3) x 3) of the three residual blocks at
        `pose` (csm_ceres_evaluate2d; what Problem::Evaluate would give)."""
        xyz = _f32(point_cloud)
        n = len(xyz)
        res = np.zeros(n + 3, np.float64)
        jac = np.zeros((n + 3, 3), np.float64) if jacobian else None
        p = np.ascontiguousarray(pose, np.float64)
        t = np.ascontiguousarray(target_translation, np.float64)
        opt = self.options._c()
        check(lib().csm_ceres_evaluate2d(
            grid._h, ptr(xyz, C.c_float), C.c_int32(n), C.byref(opt), ptr(t, C.c_double),
            C.c_double(target_angle), ptr(p, C.c_double), ptr(res, C.c_double),
            ptr(jac, C.c_double) if jacobian else None))
        return res, jac

    def EvaluateChecked(self, grid, point_cloud, pose, target_translation, target_angle,
                        jacobian=True):
        """As Evaluate, for either grid type, plus whether the cost function succeeded
        (csm_ceres_evaluate2d_checked; False on a TSDF2D where summed_weight == 0)."""
        xyz = _f32(point_cloud)
        n = len(xyz)
        res = np.zeros(n + 3, np.float64)
        jac = np.zeros((n + 3, 3), np.float64) if jacobian else None
        p = np.ascontiguousarray(pose, np.float64)
        t = np.ascontiguousarray(target_translation, np.float64)
        opt = self.options._c()
        valid = C.c_int32(0)
        check(lib().csm_ceres_evaluate2d_checked(
            grid._h, ptr(xyz, C.c_float), C.c_int32(n), C.byref(opt), ptr(t, C.c_double),
            C.c_double(target_angle), ptr(p, C.c_double), ptr(res, C.c_double),
            ptr(jac, C.c_double) if jacobian else None, C.byref(valid)))
        return res, jac, bool(valid.value)


# ===========================================================================
# CeresScanMatcher3D (mapping/internal/3d/scan_matching/ceres_scan_matcher_3d.{h,cc})
# ===========================================================================
class CsmCeresOptions3D(C.Structure):
    _fields_ = [("occupied_space_weight", C.c_double * 2), ("translation_weight", C.c_double),
                ("rotation_weight", C.c_double), ("only_optimize_yaw", C.c_int32),
                ("use_nonmonotonic_steps", C.c_int32), ("max_num_iterations", C.c_int32),
                ("reserved", C.c_int32)]


class CsmCeresJob3D(C.Structure):
    _fields_ = [("grid", C.c_void_p * 2), ("xyz", C.POINTER(C.c_float) * 2),
                ("num_points", C.c_int32 * 2), ("num_clouds", C.c_int32),
                ("reserved", C.c_int32), ("target_translation", C.c_double * 3),
                ("initial_pose", C.c_double * 7)]


class CsmCeresResult3D(C.Structure):
    _fields_ = [("pose_estimate", C.c_double * 7), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("iterations", C.c_int32),
                ("num_successful_steps", C.c_int32), ("termination", C.c_int32),
                ("reserved", C.c_int32)]


class CsmCeresIntensityJob3D(C.Structure):
    _fields_ = [("intensity_grid", C.c_void_p * 2), ("intensities", C.POINTER(C.c_float) * 2)]


class CsmCeresIntensityOptions3D(C.Structure):
    _fields_ = [("weight", C.c_double * 2), ("huber_scale", C.c_double * 2),
                ("intensity_threshold", C.c_float * 2)]


@dataclass
class IntensityCostFunctionOptions:
    """proto IntensityCostFunctionOptions (ceres_scan_matcher_options_3d.proto:21-26); each
    must be positive for a cloud that carries an intensity grid."""
    weight: float = 0.0
    huber_scale: float = 0.0
    intensity_threshold: float = 0.0


@dataclass
class CeresScanMatcherOptions3D:
    """proto/scan_matching/ceres_scan_matcher_options_3d.proto; defaults = the constraint
    builder's (configuration_files/pose_graph.lua:49-60).  only_optimize_yaw = true is not
    supported.  intensity_cost_function_options_0 / _1 apply to clouds given with an
    intensity grid."""
    occupied_space_weight_0: float = 5.0
    occupied_space_weight_1: float = 30.0
    translation_weight: float = 10.0
    rotation_weight: float = 1.0
    only_optimize_yaw: bool = False
    use_nonmonotonic_steps: bool = False
    max_num_iterations: int = 10
    intensity_cost_function_options_0: IntensityCostFunctionOptions = field(
        default_factory=IntensityCostFunctionOptions)
    intensity_cost_function_options_1: IntensityCostFunctionOptions = field(
        default_factory=IntensityCostFunctionOptions)

    def _c_intensity(self):
        o = CsmCeresIntensityOptions3D()
        for b, io in enumerate((self.intensity_cost_function_options_0,
                                self.intensity_cost_function_options_1)):
            o.weight[b] = io.weight
            o.huber_scale[b] = io.huber_scale
            o.intensity_threshold[b] = io.intensity_threshold
        return o

    def _c(self):
        o = CsmCeresOptions3D()
        o.occupied_space_weight[0] = self.occupied_space_weight_0
        o.occupied_space_weight[1] = self.occupied_space_weight_1
        o.translation_weight = self.translation_weight
        o.rotation_weight = self.rotation_weight
        o.only_optimize_yaw = int(self.only_optimize_yaw)
        o.use_nonmonotonic_steps = int(self.use_nonmonotonic_steps)
        o.max_num_iterations = int(self.max_num_iterations)
        return o


class CeresScanMatcher3D:
    """ceres_scan_matcher_3d.h:44-66.  `point_clouds_and_hybrid_grids` is a list of one or
    two entries, high resolution first, as PointCloudAndHybridGridsPointers: either
    (point_cloud, DeviceHybridGrid) or (point_cloud, DeviceHybridGrid, DeviceIntensityGrid,
    intensities), where intensities are the cloud's per-point PointCloud::intensities() and
    the intensity grid may be None.  Poses are {tx, ty, tz, qw, qx, qy, qz}."""

    def __init__(self, options=None):
        self.options = options if options is not None else CeresScanMatcherOptions3D()

    def _job(self, job, target_translation, initial_pose_estimate, pairs, keep, ijob=None):
        job.num_clouds = len(pairs)
        for b, entry in enumerate(pairs):
            cloud, grid = entry[0], entry[1]
            xyz = _f32(cloud)
            keep.append(xyz)
            job.grid[b] = grid._h
            job.xyz[b] = ptr(xyz, C.c_float)
            job.num_points[b] = len(xyz)
            if len(entry) > 2 and entry[2] is not None:
                values = np.ascontiguousarray(entry[3], dtype=np.float32).reshape(-1)
                if len(values) != len(xyz):
                    raise ValueError("one intensity per point")
                ijob.intensity_grid[b] = entry[2]._h
                ijob.intensities[b] = ptr(values, C.c_float)
                keep.append(values)
        for k in range(3):
            job.target_translation[k] = float(target_translation[k])
        for k in range(7):
            job.initial_pose[k] = float(initial_pose_estimate[k])

    @staticmethod
    def _has_intensity(pairs):
        return any(len(e) > 2 and e[2] is not None for e in pairs)

    def Match(self, target_translation, initial_pose_estimate, point_clouds_and_hybrid_grids):
        poses, summaries = self.MatchBatch([target_translation], [initial_pose_estimate],
                                           [point_clouds_and_hybrid_grids])
        return poses[0], summaries[0]

    def MatchBatch(self, target_translations, initial_pose_estimates, pairs_per_job):
        """Many Match calls in one launch (csm_ceres_match3d_batch, or
        csm_ceres_match3d_intensity_batch where a job carries an intensity grid)."""
        n = len(pairs_per_job)
        jobs = (CsmCeresJob3D * n)()
        ijobs = (CsmCeresIntensityJob3D * n)()
        keep = []
        for j in range(n):
            self._job(jobs[j], target_translations[j], initial_pose_estimates[j],
                      pairs_per_job[j], keep, ijobs[j])
        res = (CsmCeresResult3D * n)()
        stats = CsmStats()
        opt = self.options._c()
        if any(self._has_intensity(p) for p in pairs_per_job):
            iopt = self.options._c_intensity()
            check(lib().csm_ceres_match3d_intensity_batch(
                jobs, ijobs, C.c_int32(n), C.byref(opt), C.byref(iopt), res, C.byref(stats)))
        else:
            check(lib().csm_ceres_match3d_batch(jobs, C.c_int32(n), C.byref(opt), res,
                                                C.byref(stats)))
        self.last_stats = stats.as_dict()
        poses = np.array([[r.pose_estimate[k] for k in range(7)] for r in res], np.float64)
        summaries = [dict(initial_cost=r.initial_cost, final_cost=r.final_cost,
                          iterations=r.iterations, num_successful_steps=r.num_successful_steps,
                          termination=CERES_TERMINATION[r.termination]) for r in res]
        return poses, summaries

    def Evaluate(self, pairs, pose, target_translation, target_rotation, jacobian=True):
        """All residuals (per cloud its occupied-space residuals, then its intensity residuals
        where it has an intensity grid; then 3 translation and 3 rotation) and the (rows x 6)
        tangent-space Jacobian at `pose`, uncorrected by the Huber loss
        (csm_ceres_evaluate3d / csm_ceres_evaluate3d_intensity)."""
        job = CsmCeresJob3D()
        ijob = CsmCeresIntensityJob3D()
        keep = []
        self._job(job, target_translation, [0.0, 0.0, 0.0] + list(target_rotation), pairs, keep,
                  ijob)
        rows = sum(len(e[0]) * (2 if len(e) > 2 and e[2] is not None else 1) for e in pairs) + 6
        res = np.zeros(rows, np.float64)
        jac = np.zeros((rows, 6), np.float64) if jacobian else None
        p = np.ascontiguousarray(pose, np.float64)
        opt = self.options._c()
        jp = ptr(jac, C.c_double) if jacobian else None
        if self._has_intensity(pairs):
            iopt = self.options._c_intensity()
            check(lib().csm_ceres_evaluate3d_intensity(C.byref(job), C.byref(ijob), C.byref(opt),
                                                       C.byref(iopt), ptr(p, C.c_double),
                                                       ptr(res, C.c_double), jp))
        else:
            check(lib().csm_ceres_evaluate3d(C.byref(job), C.byref(opt), ptr(p, C.c_double),
                                             ptr(res, C.c_double), jp))
        return res, jac
