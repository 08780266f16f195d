"""OverlappingSubmapsTrimmer2D (mapping/internal/2d/overlapping_submaps_trimmer_2d.h), Cartographer's
lifelong-mapping trimmer, over submaps whose grids live on the device (RealTimeGrid2D).

The coverage pass — every known cell of every finished submap moved into the global frame, the
freshest submaps kept per global cell, and the covered cells counted per submap — runs on the
device (csm_trim_overlapping_submaps2d).  The host keeps what the reference's Trim does around it:
the early return, ComputeSubmapFreshness, the first submap's limits, the uint16 conversions and
the TrimSubmap calls in SubmapId order."""
import ctypes as C
import math

import numpy as np

from ._lib import check, lib

INTRA_SUBMAP = "INTRA_SUBMAP"
INTER_SUBMAP = "INTER_SUBMAP"


class CsmCoverageSubmap2D(C.Structure):
    _fields_ = [("grid", C.c_void_p), ("translation", C.c_double * 3),
                ("rotation", C.c_double * 4), ("freshness", C.c_int64)]


class CsmCoverageStats2D(C.Structure):
    _fields_ = [("entries", C.c_int64), ("coverage_cells", C.c_int64),
                ("device_tie_cells", C.c_int64), ("host_sorted_cells", C.c_int64),
                ("host_syncs", C.c_int32), ("reserved", C.c_int32)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


def trim_overlapping_submaps2d(submaps, first_limits, fresh_submaps_count,
                               min_covered_cells_count):
    """The coverage pass of OverlappingSubmapsTrimmer2D::Trim on the device.

    submaps: (grid, pose, freshness) per finished submap with a freshness, in SubmapId order:
    a RealTimeGrid2D, global_frame_from_local_frame as (tx, ty, tz, qw, qx, qy, qz) and the
    common::Time ticks of its latest intra-submap node.  first_limits: (max_x, max_y,
    resolution) of the first submap's grid.  Returns (trim flags, covered entries per submap
    before the uint16 wrap, stats)."""
    n = len(submaps)
    recs = (CsmCoverageSubmap2D * max(n, 1))()
    for i, (grid, pose, freshness) in enumerate(submaps):
        p = [float(v) for v in np.asarray(pose, np.float64).reshape(7)]
        recs[i].grid = grid._h
        recs[i].translation[:] = p[:3]
        recs[i].rotation[:] = p[3:]
        recs[i].freshness = int(freshness)
    trim = np.zeros(max(n, 1), np.uint8)
    counts = np.zeros(max(n, 1), np.uint32)
    stats = CsmCoverageStats2D()
    max_x, max_y, resolution = first_limits
    check(lib().csm_trim_overlapping_submaps2d(
        recs, C.c_int32(n), C.c_double(max_x), C.c_double(max_y), C.c_double(resolution),
        C.c_uint16(_uint16(fresh_submaps_count)), C.c_uint16(_uint16(min_covered_cells_count)),
        trim.ctypes.data_as(C.POINTER(C.c_uint8)), counts.ctypes.data_as(C.POINTER(C.c_uint32)),
        C.byref(stats)))
    return trim[:n].astype(bool), counts[:n], stats.as_dict()


def _uint16(v):
    v = int(v)
    if not 0 <= v <= 0xFFFF:
        raise ValueError("%d is not a uint16" % v)
    return v


def double_to_uint16(x):
    """The C++ conversion of a double to uint16 (truncation toward zero), defined only when the
    truncated value is in [0, 65535]; anything else raises ValueError."""
    x = float(x)
    if not (x > -1.0 and x < 65536.0):
        raise ValueError("%r is outside the range a double converts to uint16 in" % x)
    return int(x)


# ---- Rigid3d arithmetic in Eigen's scalar order: poses are (tx, ty, tz, qw, qx, qy, qz) -------
def _rotate(q, v):
    w, a, b, c = q
    uv = [b * v[2] - c * v[1], c * v[0] - a * v[2], a * v[1] - b * v[0]]
    uv = [u + u for u in uv]
    x = [b * uv[2] - c * uv[1], c * uv[0] - a * uv[2], a * uv[1] - b * uv[0]]
    return [v[k] + w * uv[k] + x[k] for k in range(3)]


def _quat_product(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return [aw * bw - ax * bx - ay * by - az * bz,
            aw * bx + ax * bw + ay * bz - az * by,
            aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx]


def rigid3_inverse(p):
    q = [p[3], -p[4], -p[5], -p[6]]
    t = _rotate(q, p[:3])
    return [-t[0], -t[1], -t[2]] + q


def rigid3_multiply(lhs, rhs):
    t = _rotate(lhs[3:], rhs[:3])
    t = [t[k] + lhs[k] for k in range(3)]
    q = _quat_product(lhs[3:], rhs[3:])
    norm = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    return t + [v / norm for v in q]


def global_frame_from_local_frame(global_pose, local_pose):
    """global_pose * local_pose.inverse() (overlapping_submaps_trimmer_2d.cc:78-81)."""
    g = [float(v) for v in np.asarray(global_pose, np.float64).reshape(7)]
    loc = [float(v) for v in np.asarray(local_pose, np.float64).reshape(7)]
    return rigid3_multiply(g, rigid3_inverse(loc))


def compute_submap_freshness(submap_data, trajectory_nodes, constraints):
    """ComputeSubmapFreshness (overlapping_submaps_trimmer_2d.cc:105-143): per submap the time of
    its largest NodeId over INTRA_SUBMAP constraints, if the submap and that node exist."""
    latest = {}
    for c in constraints:
        if c.tag != INTRA_SUBMAP:
            continue
        if c.submap_id not in latest or latest[c.submap_id] < c.node_id:
            latest[c.submap_id] = c.node_id
    freshness = {}
    for submap_id, node_id in sorted(latest.items()):
        if submap_id not in submap_data or node_id not in trajectory_nodes:
            continue
        freshness[submap_id] = int(trajectory_nodes[node_id].time)
    return freshness


def _grid_limits(grid):
    """(max_x, max_y, resolution) of a RealTimeGrid2D (csm_rt_grid2d_limits: no stream
    synchronisation)."""
    res, mx, my = C.c_double(), C.c_double(), C.c_double()
    check(lib().csm_rt_grid2d_limits(grid._h, C.byref(res), C.byref(mx), C.byref(my), None, None))
    return mx.value, my.value, res.value


class OverlappingSubmapsTrimmer2D:
    """OverlappingSubmapsTrimmer2D(fresh_submaps_count, min_covered_area,
    min_added_submaps_count) with Trim(pose_graph) and IsFinished().

    pose_graph is duck-typed as the reference's Trimmable: GetOptimizedSubmapData() maps
    SubmapId (any ordered key, e.g. (trajectory_id, submap_index)) to an entry with .pose
    (global, 7 values) and .submap (.grid a RealTimeGrid2D: the cropped grid of a finished
    submap, the active grid of an unfinished one, whose limits are read when it comes first;
    .local_pose, .insertion_finished);
    GetTrajectoryNodes() maps NodeId to a node with .time (common::Time ticks);
    GetConstraints() lists constraints with .submap_id, .node_id and .tag (INTRA_SUBMAP or
    INTER_SUBMAP); TrimSubmap(submap_id) trims."""

    def __init__(self, fresh_submaps_count, min_covered_area, min_added_submaps_count):
        self.fresh_submaps_count = _uint16(fresh_submaps_count)
        self.min_covered_area = float(min_covered_area)
        self.min_added_submaps_count = _uint16(min_added_submaps_count)
        self.current_submap_count = 0   # uint16
        self.last_stats = None

    def IsFinished(self):
        return False

    def Trim(self, pose_graph):
        submap_data = pose_graph.GetOptimizedSubmapData()
        ids = sorted(submap_data)
        # submap_data.size() - current_submap_count_ in size_t
        if (len(ids) - self.current_submap_count) % (1 << 64) <= self.min_added_submaps_count:
            return
        freshness = compute_submap_freshness(submap_data, pose_graph.GetTrajectoryNodes(),
                                             pose_graph.GetConstraints())
        participating = [i for i in ids
                         if i in freshness and submap_data[i].submap.insertion_finished]
        to_remove = []
        self.last_stats = None
        if participating:
            first = self._limits(submap_data[ids[0]].submap.grid)
            min_cells = double_to_uint16(self.min_covered_area / (first[2] * first[2]))
            records = []
            for i in participating:
                d = submap_data[i]
                records.append((d.submap.grid,
                                global_frame_from_local_frame(d.pose, d.submap.local_pose),
                                freshness[i]))
            trim, _, self.last_stats = self._coverage(records, first, self.fresh_submaps_count,
                                                      min_cells)
            to_remove = [i for i, t in zip(participating, trim) if t]
        self.current_submap_count = (len(ids) - len(to_remove)) & 0xFFFF
        for i in to_remove:
            pose_graph.TrimSubmap(i)

    # The two steps that read grids: a grid's (max_x, max_y, resolution), and the coverage pass.
    def _limits(self, grid):
        return _grid_limits(grid)

    def _coverage(self, records, first_limits, fresh_submaps_count, min_covered_cells_count):
        return trim_overlapping_submaps2d(records, first_limits, fresh_submaps_count,
                                          min_covered_cells_count)
