"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes front-end for oracle/_build/liboracle.so (the CPU restatement of the
reference path, see oracle_common.h).  Imported only by tests/, by
__graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference leg.
The product package cartographer_b200 never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_DIR, "_build", "liboracle.so")


def build(force=False):
    srcs = [os.path.join(_DIR, f) for f in os.listdir(_DIR) if f.endswith((".cc", ".h"))]
    if force or not os.path.exists(_SO) or any(
            os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
        subprocess.check_call(["make", "-C", _DIR, "-s"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        _lib = C.CDLL(_SO)
        _lib.orc_constant.restype = C.c_float
        _lib.orc_probability_to_value.restype = C.c_uint16
        _lib.orc_probability_to_value.argtypes = [C.c_float]
        _lib.orc_correspondence_cost_to_value.restype = C.c_uint16
        _lib.orc_correspondence_cost_to_value.argtypes = [C.c_float]
        _lib.orc_frontend2d_create.restype = C.c_void_p
        _lib.orc_frontend2d_step.restype = C.c_double
        _lib.orc_fast2d_create.restype = C.c_void_p
        _lib.orc_rt2d_match.restype = C.c_double
        _lib.orc_rt2d_match_tsdf.restype = C.c_double
        _lib.orc_fast2d_batch.restype = C.c_double
        _lib.orc_fast3d_create.restype = C.c_void_p
        _lib.orc_hybrid_create.restype = C.c_void_p
        _lib.orc_hybrid_get_probability.restype = C.c_float
        _lib.orc_rt3d_match.restype = C.c_float
        _lib.orc_rt2d_scores.restype = C.c_int64
        _lib.orc_rt2d_scores_tsdf.restype = C.c_int64
        _lib.orc_rt3d_scores.restype = C.c_int64
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _u16(a):
    return np.ascontiguousarray(a, dtype=np.uint16)


def constant(which):
    return float(lib().orc_constant(C.c_int(which)))


def value_to_cost_table(min_cost, max_cost):
    out = np.empty(65536, np.float32)
    lib().orc_value_to_cost_table(C.c_float(min_cost), C.c_float(max_cost), _p(out, C.c_float))
    return out


def probability_to_value(p):
    return int(lib().orc_probability_to_value(C.c_float(p)))


def correspondence_cost_to_value(c):
    return int(lib().orc_correspondence_cost_to_value(C.c_float(c)))


def get_cell_index(res, max_x, max_y, px, py):
    out = np.zeros(2, np.int32)
    lib().orc_get_cell_index(C.c_double(res), C.c_double(max_x), C.c_double(max_y),
                             C.c_float(px), C.c_float(py), _p(out, C.c_int32))
    return int(out[0]), int(out[1])


def search_params(lin, ang, xyz, res):
    xyz = _f32(xyz)
    na, ns, nl = C.c_int32(), C.c_int32(), C.c_int32()
    step = C.c_double()
    lib().orc_search_params(C.c_double(lin), C.c_double(ang), _p(xyz, C.c_float),
                            C.c_int(len(xyz)), C.c_double(res), C.byref(na), C.byref(step),
                            C.byref(ns), C.byref(nl))
    return dict(num_angular_perturbations=na.value, angular_perturbation_step_size=step.value,
                num_scans=ns.value, num_linear_perturbations=nl.value)


def candidate(num_lin, num_ang, step, res, scan, xo, yo):
    out = np.zeros(3, np.float64)
    lib().orc_candidate(C.c_int(num_lin), C.c_int(num_ang), C.c_double(step), C.c_double(res),
                        C.c_int(scan), C.c_int(xo), C.c_int(yo), _p(out, C.c_double))
    return out


def generate_rotated_scans(xyz, num_ang, step):
    xyz = _f32(xyz)
    out = np.empty((2 * num_ang + 1, len(xyz), 3), np.float32)
    lib().orc_generate_rotated_scans(_p(xyz, C.c_float), C.c_int(len(xyz)), C.c_int(num_ang),
                                     C.c_double(step), _p(out, C.c_float))
    return out


def discretize_scans(res, max_x, max_y, nx, ny, scans_xyz, tx=0.0, ty=0.0):
    scans_xyz = _f32(scans_xyz)
    S, n, _ = scans_xyz.shape
    out = np.empty((S, n, 2), np.int32)
    lib().orc_discretize_scans(C.c_double(res), C.c_double(max_x), C.c_double(max_y),
                               C.c_int(nx), C.c_int(ny), _p(scans_xyz, C.c_float), C.c_int(S),
                               C.c_int(n), C.c_float(tx), C.c_float(ty), _p(out, C.c_int32))
    return out


def frontend2d(grid, xyz, init_pose=(0, 0, 0), full=False, lin=0.0, ang=0.0, rt_mode=False,
               want_rotated=False):
    """Rotated + discretised scans and post-ShrinkToFit bounds, as Match builds them."""
    xyz = _f32(xyz)
    ip = np.ascontiguousarray(init_pose, dtype=np.float64)
    h = C.c_void_p(lib().orc_frontend2d_create(
        C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
        C.c_int(grid.num_x), C.c_int(grid.num_y), _p(xyz, C.c_float), C.c_int(len(xyz)),
        _p(ip, C.c_double), C.c_int(int(full)), C.c_double(lin), C.c_double(ang),
        C.c_int(int(rt_mode))))
    try:
        S = lib().orc_frontend2d_num_scans(h)
        step = lib().orc_frontend2d_step(h)
        ds = np.empty((S, len(xyz), 2), np.int32)
        bounds = np.empty((S, 4), np.int32)
        rot = np.empty((S, len(xyz), 3), np.float32) if want_rotated else None
        lib().orc_frontend2d_get(h, _p(ds, C.c_int32), _p(bounds, C.c_int32),
                                 _p(rot, C.c_float) if want_rotated else None)
    finally:
        lib().orc_frontend2d_destroy(h)
    return dict(num_scans=S, step=step, discrete_scans=ds, bounds=bounds, rotated=rot)


def precompute_grid2d(cells, min_cost, max_cost, width):
    cells = _u16(cells)
    ny, nx = cells.shape
    out = np.empty((ny + width - 1, nx + width - 1), np.uint8)
    lib().orc_precompute_grid2d(_p(cells, C.c_uint16), C.c_int(nx), C.c_int(ny),
                                C.c_float(min_cost), C.c_float(max_cost), C.c_int(width),
                                _p(out, C.c_uint8))
    return out


class Grid2D:
    """Plain record of a ProbabilityGrid: cells[y, x] uint16 (num_x * y + x)."""

    def __init__(self, cells, resolution, max_x, max_y, min_cost=None, max_cost=None):
        self.cells = _u16(cells)
        self.num_y, self.num_x = self.cells.shape
        self.resolution = float(resolution)
        self.max_x = float(max_x)
        self.max_y = float(max_y)
        self.min_cost = constant(2) if min_cost is None else float(min_cost)
        self.max_cost = constant(3) if max_cost is None else float(max_cost)


STAT_KEYS = ("candidates_scored", "lowest_resolution_candidates", "nodes_expanded", "num_scans",
             "best_scan_index", "best_x_offset", "best_y_offset")


class FastCorrelativeScanMatcher2D:
    def __init__(self, grid, linear_search_window, angular_search_window, branch_and_bound_depth):
        self.grid = grid
        self.depth = branch_and_bound_depth
        self._h = C.c_void_p(lib().orc_fast2d_create(
            _p(grid.cells, C.c_uint16), C.c_int(grid.num_x), C.c_int(grid.num_y),
            C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
            C.c_float(grid.min_cost), C.c_float(grid.max_cost), C.c_double(linear_search_window),
            C.c_double(angular_search_window), C.c_int(branch_and_bound_depth)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_fast2d_destroy(self._h)
            self._h = None

    def _match(self, xyz, init_pose, full, min_score):
        xyz = _f32(xyz)
        ip = np.ascontiguousarray(init_pose, dtype=np.float64)
        score = C.c_float(0)
        pose = np.zeros(3, np.float64)
        stats = np.zeros(8, np.int64)
        found = lib().orc_fast2d_match(self._h, _p(xyz, C.c_float), C.c_int(len(xyz)),
                                       _p(ip, C.c_double), C.c_int(int(full)),
                                       C.c_float(min_score), C.byref(score), _p(pose, C.c_double),
                                       _p(stats, C.c_int64))
        return dict(found=bool(found), score=np.float32(score.value), pose=pose,
                    **{k: int(stats[i]) for i, k in enumerate(STAT_KEYS)})

    def match(self, init_pose, xyz, min_score):
        return self._match(xyz, init_pose, False, min_score)

    def match_full_submap(self, xyz, min_score):
        return self._match(xyz, (0, 0, 0), True, min_score)

    def level(self, level):
        nx, ny = C.c_int32(), C.c_int32()
        lib().orc_fast2d_level(self._h, C.c_int(level), None, C.byref(nx), C.byref(ny))
        out = np.empty((ny.value, nx.value), np.uint8)
        lib().orc_fast2d_level(self._h, C.c_int(level), _p(out, C.c_uint8), C.byref(nx),
                               C.byref(ny))
        return out

    def score_candidates(self, level, discrete_scans, cand):
        ds = _i32(discrete_scans)
        cand = _i32(cand)
        S, n, _ = ds.shape
        scores = np.empty(len(cand), np.float32)
        sums = np.empty(len(cand), np.int32)
        lib().orc_fast2d_score_candidates(self._h, C.c_int(level), _p(ds, C.c_int32), C.c_int(S),
                                          C.c_int(n), _p(cand, C.c_int32), C.c_int(len(cand)),
                                          _p(scores, C.c_float), _p(sums, C.c_int32))
        return scores, sums


def rt2d_match(grid, xyz, init_pose, lin, ang, w_t, w_r):
    xyz = _f32(xyz)
    ip = np.ascontiguousarray(init_pose, dtype=np.float64)
    pose = np.zeros(3, np.float64)
    stats = np.zeros(8, np.int64)
    score = lib().orc_rt2d_match(_p(grid.cells, C.c_uint16), C.c_int(grid.num_x),
                                 C.c_int(grid.num_y), C.c_double(grid.resolution),
                                 C.c_double(grid.max_x), C.c_double(grid.max_y),
                                 _p(xyz, C.c_float), C.c_int(len(xyz)), _p(ip, C.c_double),
                                 C.c_double(lin), C.c_double(ang), C.c_double(w_t),
                                 C.c_double(w_r), _p(pose, C.c_double), _p(stats, C.c_int64))
    return dict(score=float(score), pose=pose,
                **{k: int(stats[i]) for i, k in enumerate(STAT_KEYS)})


def tsdf_values(truncation, max_weight, tsd, weight):
    out = np.zeros(2, np.uint16)
    lib().orc_tsdf_values(C.c_float(truncation), C.c_float(max_weight), C.c_float(tsd),
                          C.c_float(weight), _p(out, C.c_uint16))
    return int(out[0]), int(out[1])


def rt2d_match_tsdf(tsd_cells, weight_cells, resolution, max_x, max_y, truncation, max_weight,
                    xyz, init_pose, lin, ang, w_t, w_r):
    tsd, wgt = _u16(tsd_cells), _u16(weight_cells)
    ny, nx = tsd.shape
    xyz = _f32(xyz)
    ip = np.ascontiguousarray(init_pose, dtype=np.float64)
    pose = np.zeros(3, np.float64)
    stats = np.zeros(8, np.int64)
    score = lib().orc_rt2d_match_tsdf(
        _p(tsd, C.c_uint16), _p(wgt, C.c_uint16), C.c_int(nx), C.c_int(ny), C.c_double(resolution),
        C.c_double(max_x), C.c_double(max_y), C.c_float(truncation), C.c_float(max_weight),
        _p(xyz, C.c_float), C.c_int(len(xyz)), _p(ip, C.c_double), C.c_double(lin),
        C.c_double(ang), C.c_double(w_t), C.c_double(w_r), _p(pose, C.c_double),
        _p(stats, C.c_int64))
    return dict(score=float(score), pose=pose,
                **{k: int(stats[i]) for i, k in enumerate(STAT_KEYS)})


def _sized(call):
    """call(scores_ptr, cap) -> count: count first, then the scores (float32)."""
    n = call(None, C.c_int64(0))
    out = np.empty(n, np.float32)
    call(_p(out, C.c_float), C.c_int64(n))
    return out


def rt2d_scores(grid, xyz, init_pose, lin, ang, w_t, w_r):
    """Every candidate's score of rt2d_match's Match, in generation order (scan, x offset,
    y offset), as std::max_element sees them."""
    xyz = _f32(xyz)
    ip = np.ascontiguousarray(init_pose, dtype=np.float64)
    return _sized(lambda out, cap: lib().orc_rt2d_scores(
        _p(grid.cells, C.c_uint16), C.c_int(grid.num_x), C.c_int(grid.num_y),
        C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
        _p(xyz, C.c_float), C.c_int(len(xyz)), _p(ip, C.c_double), C.c_double(lin),
        C.c_double(ang), C.c_double(w_t), C.c_double(w_r), out, cap))


def rt2d_scores_tsdf(tsd_cells, weight_cells, resolution, max_x, max_y, truncation, max_weight,
                     xyz, init_pose, lin, ang, w_t, w_r):
    """As rt2d_scores, for rt2d_match_tsdf's Match."""
    tsd, wgt = _u16(tsd_cells), _u16(weight_cells)
    ny, nx = tsd.shape
    xyz = _f32(xyz)
    ip = np.ascontiguousarray(init_pose, dtype=np.float64)
    return _sized(lambda out, cap: lib().orc_rt2d_scores_tsdf(
        _p(tsd, C.c_uint16), _p(wgt, C.c_uint16), C.c_int(nx), C.c_int(ny), C.c_double(resolution),
        C.c_double(max_x), C.c_double(max_y), C.c_float(truncation), C.c_float(max_weight),
        _p(xyz, C.c_float), C.c_int(len(xyz)), _p(ip, C.c_double), C.c_double(lin),
        C.c_double(ang), C.c_double(w_t), C.c_double(w_r), out, cap))


def rt2d_score_candidates(grid, discrete_scans, num_lin, num_ang, step, w_t, w_r, cand):
    ds = _i32(discrete_scans)
    cand = _i32(cand)
    S, n, _ = ds.shape
    assert S == 2 * num_ang + 1
    scores = np.empty(len(cand), np.float32)
    lib().orc_rt2d_score_candidates(_p(grid.cells, C.c_uint16), C.c_int(grid.num_x),
                                    C.c_int(grid.num_y), C.c_double(grid.resolution),
                                    C.c_double(grid.max_x), C.c_double(grid.max_y),
                                    _p(ds, C.c_int32), C.c_int(n), C.c_int(num_lin),
                                    C.c_int(num_ang), C.c_double(step), C.c_double(w_t),
                                    C.c_double(w_r), _p(cand, C.c_int32), C.c_int(len(cand)),
                                    _p(scores, C.c_float))
    return scores


def fast2d_batch(matchers, job_matcher, job_cloud, job_init_pose, clouds, full, min_score,
                 threads):
    """CPU-baseline batch runner; returns (seconds, found, scores, poses, cand_scored)."""
    J = len(job_matcher)
    hs = (C.c_void_p * len(matchers))(*[m._h for m in matchers])
    clouds = [_f32(c) for c in clouds]
    cptr = (C.POINTER(C.c_float) * len(clouds))(*[_p(c, C.c_float) for c in clouds])
    cn = _i32([len(c) for c in clouds])
    jm, jc = _i32(job_matcher), _i32(job_cloud)
    jp = np.ascontiguousarray(job_init_pose, dtype=np.float64).reshape(J, 3)
    found = np.zeros(J, np.int32)
    scores = np.zeros(J, np.float32)
    poses = np.zeros((J, 3), np.float64)
    cs = np.zeros(J, np.int64)
    secs = lib().orc_fast2d_batch(hs, _p(jm, C.c_int32), _p(jc, C.c_int32), _p(jp, C.c_double),
                                  C.c_int(J), cptr, _p(cn, C.c_int32), C.c_int(int(full)),
                                  C.c_float(min_score), C.c_int(threads), _p(found, C.c_int32),
                                  _p(scores, C.c_float), _p(poses, C.c_double),
                                  _p(cs, C.c_int64))
    return secs, found, scores, poses, cs


# ===========================================================================
# 3D
# ===========================================================================
STAT3_KEYS = ("candidates_scored", "lowest_resolution_candidates", "nodes_expanded",
              "low_resolution_evaluations", "num_scans", "num_angles", "best_scan_index",
              "best_x", "best_y", "best_z")


def hybrid_get_cell_index(resolution, p):
    p = _f32(p)
    out = np.zeros(3, np.int32)
    lib().orc_hybrid_get_cell_index(C.c_float(resolution), _p(p, C.c_float), _p(out, C.c_int32))
    return tuple(int(v) for v in out)


class HybridGrid:
    """Sparse voxel grid given as (indices n x 3 int32, values n uint16) — the flat
    form of proto::HybridGrid (mapping/proto/hybrid_grid.proto:19-28)."""

    def __init__(self, resolution, indices, values):
        self.resolution = float(np.float32(resolution))
        self.indices = _i32(indices).reshape(-1, 3)
        self.values = _u16(values).reshape(-1)
        lib().orc_hybrid_get_probability.restype = C.c_float
        self._h = C.c_void_p(lib().orc_hybrid_create(
            C.c_float(resolution), _p(self.indices, C.c_int32), _p(self.values, C.c_uint16),
            C.c_int64(len(self.values))))

    def grid_size(self):
        return int(lib().orc_hybrid_grid_size(self._h))

    def get_probability(self, x, y, z):
        return float(lib().orc_hybrid_get_probability(self._h, C.c_int(x), C.c_int(y), C.c_int(z)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_hybrid_destroy(self._h)
            self._h = None


class FastCorrelativeScanMatcher3D:
    def __init__(self, hi, lo, histogram, options):
        """options: dict with branch_and_bound_depth, full_resolution_depth,
        min_rotational_score, min_low_resolution_score, linear_xy_search_window,
        linear_z_search_window, angular_search_window."""
        self.hi, self.lo = hi, lo
        self.histogram = _f32(histogram).reshape(-1)
        o = options
        self._h = C.c_void_p(lib().orc_fast3d_create(
            hi._h, lo._h, _p(self.histogram, C.c_float), C.c_int(len(self.histogram)),
            C.c_int(o["branch_and_bound_depth"]), C.c_int(o["full_resolution_depth"]),
            C.c_double(o["min_rotational_score"]), C.c_double(o["min_low_resolution_score"]),
            C.c_double(o["linear_xy_search_window"]), C.c_double(o["linear_z_search_window"]),
            C.c_double(o["angular_search_window"])))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_fast3d_destroy(self._h)
            self._h = None

    def _match(self, full, node_pose, submap_pose, node, min_score):
        npose = np.ascontiguousarray(node_pose, np.float64)
        spose = np.ascontiguousarray(submap_pose, np.float64)
        grav = np.ascontiguousarray(node["gravity_alignment"], np.float64)
        hi, lo = _f32(node["high_resolution_point_cloud"]), _f32(node["low_resolution_point_cloud"])
        hist = _f32(node["rotational_scan_matcher_histogram"]).reshape(-1)
        score, rot, low = C.c_float(0), C.c_float(0), C.c_float(0)
        pose = np.zeros(7, np.float64)
        stats = np.zeros(12, np.int64)
        found = lib().orc_fast3d_match(
            self._h, C.c_int(int(full)), _p(npose, C.c_double), _p(spose, C.c_double),
            _p(grav, C.c_double), _p(hi, C.c_float), C.c_int(len(hi)), _p(lo, C.c_float),
            C.c_int(len(lo)), _p(hist, C.c_float), C.c_int(len(hist)), C.c_float(min_score),
            C.byref(score), _p(pose, C.c_double), C.byref(rot), C.byref(low), _p(stats, C.c_int64))
        return dict(found=bool(found), score=np.float32(score.value), pose=pose,
                    rotational_score=np.float32(rot.value),
                    low_resolution_score=np.float32(low.value),
                    **{k: int(stats[i]) for i, k in enumerate(STAT3_KEYS)})

    def match(self, node_pose, submap_pose, node, min_score):
        return self._match(False, node_pose, submap_pose, node, min_score)

    def match_full_submap(self, node_rotation, submap_rotation, node, min_score):
        return self._match(True, [0, 0, 0] + list(node_rotation), [0, 0, 0] + list(submap_rotation),
                           node, min_score)

    def level(self, depth):
        lo, dims = np.zeros(3, np.int32), np.zeros(3, np.int32)
        lib().orc_fast3d_level(self._h, C.c_int(depth), _p(lo, C.c_int32), _p(dims, C.c_int32),
                               None)
        out = np.zeros((dims[2], dims[1], dims[0]), np.uint8)
        if out.size:
            lib().orc_fast3d_level(self._h, C.c_int(depth), _p(lo, C.c_int32),
                                   _p(dims, C.c_int32), _p(out, C.c_uint8))
        return lo, out

    def level_box(self, depth, lo, dims):
        lo, dims = _i32(lo), _i32(dims)
        out = np.zeros((dims[2], dims[1], dims[0]), np.uint8)
        lib().orc_fast3d_level(self._h, C.c_int(depth), _p(lo, C.c_int32), _p(dims, C.c_int32),
                               _p(out, C.c_uint8))
        return out

    def discrete_scans(self, full, node_pose, submap_pose, node):
        npose = np.ascontiguousarray(node_pose, np.float64)
        spose = np.ascontiguousarray(submap_pose, np.float64)
        grav = np.ascontiguousarray(node["gravity_alignment"], np.float64)
        hi = _f32(node["high_resolution_point_cloud"])
        hist = _f32(node["rotational_scan_matcher_histogram"]).reshape(-1)
        args = (self._h, C.c_int(int(full)), _p(npose, C.c_double), _p(spose, C.c_double),
                _p(grav, C.c_double), _p(hi, C.c_float), C.c_int(len(hi)), _p(hist, C.c_float),
                C.c_int(len(hist)))
        S = lib().orc_fast3d_discrete_scans(*args, None, None, None)
        cells = np.zeros((S, len(hi), 3), np.int32)
        poses = np.zeros((S, 7), np.float32)
        rot = np.zeros(S, np.float32)
        if S:
            lib().orc_fast3d_discrete_scans(*args, _p(cells, C.c_int32), _p(poses, C.c_float),
                                            _p(rot, C.c_float))
        return cells, poses, rot

    def score_candidates(self, full, node_pose, submap_pose, node, depth, candidates):
        """ScoreCandidates of `candidates` (n x {scan, x, y, z}) at `depth` on the discrete
        scans of this match, unsorted -> (sums int32, scores float32, low-resolution scores
        float32 of GetPoseFromCandidate at depth 0, else None)."""
        npose = np.ascontiguousarray(node_pose, np.float64)
        spose = np.ascontiguousarray(submap_pose, np.float64)
        grav = np.ascontiguousarray(node["gravity_alignment"], np.float64)
        hi, lo = _f32(node["high_resolution_point_cloud"]), _f32(node["low_resolution_point_cloud"])
        hist = _f32(node["rotational_scan_matcher_histogram"]).reshape(-1)
        cand = _i32(candidates).reshape(-1, 4)
        n = len(cand)
        sums = np.zeros(n, np.int32)
        scores = np.zeros(n, np.float32)
        low = np.zeros(n, np.float32)
        lib().orc_fast3d_score_candidates(
            self._h, C.c_int(int(full)), _p(npose, C.c_double), _p(spose, C.c_double),
            _p(grav, C.c_double), _p(hi, C.c_float), C.c_int(len(hi)), _p(lo, C.c_float),
            C.c_int(len(lo)), _p(hist, C.c_float), C.c_int(len(hist)), C.c_int(depth),
            _p(cand, C.c_int32), C.c_int(n), _p(sums, C.c_int32), _p(scores, C.c_float),
            _p(low, C.c_float) if depth == 0 else None)
        return sums, scores, (low if depth == 0 else None)


def rotational_match(submap_hist, hist, initial_angle, angles):
    a, b = _f32(submap_hist).reshape(-1), _f32(hist).reshape(-1)
    ang = _f32(angles).reshape(-1)
    out = np.zeros(len(ang), np.float32)
    lib().orc_rotational_match(_p(a, C.c_float), _p(b, C.c_float), C.c_int(len(a)),
                               C.c_float(initial_angle), _p(ang, C.c_float), C.c_int(len(ang)),
                               _p(out, C.c_float))
    return out


def rt3d_match(hybrid_grid, xyz, initial_pose, lin, ang, w_t, w_r):
    """RealTimeCorrelativeScanMatcher3D::Match; initial_pose / pose = {t xyz, q wxyz}."""
    xyz = _f32(xyz)
    ip = np.ascontiguousarray(initial_pose, dtype=np.float64)
    pose = np.zeros(7, np.float64)
    stats = np.zeros(2, np.int64)
    score = lib().orc_rt3d_match(hybrid_grid._h, _p(xyz, C.c_float), C.c_int(len(xyz)),
                                 _p(ip, C.c_double), C.c_double(lin), C.c_double(ang),
                                 C.c_double(w_t), C.c_double(w_r), _p(pose, C.c_double),
                                 _p(stats, C.c_int64))
    return dict(score=np.float32(score), pose=pose, candidates_scored=int(stats[0]),
                best_index=int(stats[1]))


def rt3d_scores(hybrid_grid, xyz, initial_pose, lin, ang, w_t, w_r):
    """Every candidate's score of rt3d_match's Match, in generation order (translations z, y,
    x, then rotations rz, ry, rx), as its `score > best_score` loop sees them."""
    xyz = _f32(xyz)
    ip = np.ascontiguousarray(initial_pose, dtype=np.float64)
    return _sized(lambda out, cap: lib().orc_rt3d_scores(
        hybrid_grid._h, _p(xyz, C.c_float), C.c_int(len(xyz)), _p(ip, C.c_double),
        C.c_double(lin), C.c_double(ang), C.c_double(w_t), C.c_double(w_r), out, cap))


# ---- CeresScanMatcher2D restatement (oracle_ceres2d.h; parity unpinned against Ceres) ----
CERES_TERMINATION = ("NO_CONVERGENCE", "FUNCTION_TOLERANCE", "GRADIENT_TOLERANCE",
                     "PARAMETER_TOLERANCE", "MIN_TRUST_REGION_RADIUS", "INVALID_STEPS")


# One record per pass of the trust-region loop (oracle_ceres2d.h, CeresIterationTrace); the
# Python restatements in tests/ append the same dicts.
CERES_STEP_OUTCOME = ("ACCEPTED", "REJECTED", "INVALID", "PARAMETER_TOLERANCE",
                      "FUNCTION_TOLERANCE", "LOOP_EXIT")
CERES_TRACE_KEYS = ("outcome", "reused_diagonal", "reference_switched", "x_cost",
                    "gradient_max_norm", "radius_before", "radius_after", "candidate_cost",
                    "model_cost_change", "step_quality", "step_norm", "step_norm_threshold",
                    "cost_change", "cost_change_threshold", "evaluator_minimum_cost",
                    "evaluator_candidate_cost")


def ceres_trace_record(outcome, **values):
    """A trace record with every key; what the pass did not reach is NaN."""
    rec = dict.fromkeys(CERES_TRACE_KEYS, float("nan"))
    rec.update(outcome=outcome, reused_diagonal=False, reference_switched=False)
    rec.update(values)
    return rec


def _traced(call):
    """call(trace_ptr, cap) -> count: the records as dicts."""
    buf = np.zeros((256, len(CERES_TRACE_KEYS)), np.float64)
    count = call(_p(buf, C.c_double), C.c_int(len(buf)))
    assert count <= len(buf)
    return [dict(zip(CERES_TRACE_KEYS, (CERES_STEP_OUTCOME[int(r[0])], bool(r[1]), bool(r[2]))
                     + tuple(float(v) for v in r[3:]))) for r in buf[:count]]


def _ceres_opts(occupied_space_weight, translation_weight, rotation_weight,
                use_nonmonotonic_steps, max_num_iterations):
    return np.array([occupied_space_weight, translation_weight, rotation_weight,
                     float(bool(use_nonmonotonic_steps)), float(max_num_iterations)], np.float64)


def ceres2d_evaluate(grid, xyz, pose, target_xy, target_angle, occupied_space_weight=20.0,
                     translation_weight=10.0, rotation_weight=1.0, jacobian=True):
    """Residuals (n + 3) and Jacobian ((n + 3) x 3) of CeresScanMatcher2D's three blocks."""
    xyz = _f32(xyz)
    n = len(xyz)
    o = _ceres_opts(occupied_space_weight, translation_weight, rotation_weight, True, 1)
    p = np.ascontiguousarray(pose, np.float64)
    t = np.ascontiguousarray(target_xy, np.float64)
    res = np.zeros(n + 3, np.float64)
    jac = np.zeros((n + 3, 3), np.float64) if jacobian else None
    lib().orc_ceres2d_evaluate(_p(grid.cells, C.c_uint16), C.c_int(grid.num_x),
                               C.c_int(grid.num_y), C.c_double(grid.resolution),
                               C.c_double(grid.max_x), C.c_double(grid.max_y),
                               _p(xyz, C.c_float), C.c_int(n), _p(o, C.c_double),
                               _p(t, C.c_double), C.c_double(target_angle), _p(p, C.c_double),
                               _p(res, C.c_double), _p(jac, C.c_double) if jacobian else None)
    return res, jac


def ceres2d_match(grid, xyz, target_xy, initial_pose, occupied_space_weight=20.0,
                  translation_weight=10.0, rotation_weight=1.0, use_nonmonotonic_steps=True,
                  max_num_iterations=10, trace=False):
    """CeresScanMatcher2D::Match -> dict(pose, initial_cost, final_cost, iterations, ...);
    with trace also "trace", the per-iteration records."""
    xyz = _f32(xyz)
    o = _ceres_opts(occupied_space_weight, translation_weight, rotation_weight,
                    use_nonmonotonic_steps, max_num_iterations)
    t = np.ascontiguousarray(target_xy, np.float64)
    ip = np.ascontiguousarray(initial_pose, np.float64)
    pose = np.zeros(3, np.float64)
    sm = np.zeros(5, np.float64)
    args = (_p(grid.cells, C.c_uint16), C.c_int(grid.num_x), C.c_int(grid.num_y),
            C.c_double(grid.resolution), C.c_double(grid.max_x), C.c_double(grid.max_y),
            _p(xyz, C.c_float), C.c_int(len(xyz)), _p(o, C.c_double), _p(t, C.c_double),
            _p(ip, C.c_double), _p(pose, C.c_double), _p(sm, C.c_double))
    extra = {}
    if trace:
        extra["trace"] = _traced(lambda buf, cap: lib().orc_ceres2d_match_traced(*args, buf, cap))
    else:
        lib().orc_ceres2d_match(*args)
    return dict(pose=pose, initial_cost=float(sm[0]), final_cost=float(sm[1]),
                iterations=int(sm[2]), num_successful_steps=int(sm[3]),
                termination=CERES_TERMINATION[int(sm[4])], **extra)


# ---- CeresScanMatcher3D restatement (oracle_ceres3d.h; parity unpinned against Ceres) ----
def interpolated_probability(hybrid_grid, x, y, z, gradient=False):
    """InterpolatedGrid<HybridGrid>::GetInterpolatedValue (+ d/d(x, y, z) on dual numbers)."""
    lib().orc_interpolated_probability.restype = C.c_double
    g = np.zeros(3, np.float64)
    f = lib().orc_interpolated_probability(hybrid_grid._h, C.c_double(x), C.c_double(y),
                                           C.c_double(z), _p(g, C.c_double) if gradient else None)
    return (float(f), g) if gradient else float(f)


def _ceres3d_args(clouds_and_grids, occupied_space_weights, translation_weight, rotation_weight,
                  use_nonmonotonic_steps, max_num_iterations):
    num = len(clouds_and_grids)
    clouds = [_f32(c) for c, _ in clouds_and_grids]
    hy = (C.c_void_p * num)(*[g._h for _, g in clouds_and_grids])
    xs = (C.POINTER(C.c_float) * num)(*[_p(c, C.c_float) for c in clouds])
    ns = np.array([len(c) for c in clouds], np.int32)
    o = np.array([translation_weight, rotation_weight, float(bool(use_nonmonotonic_steps)),
                  float(max_num_iterations)] + list(occupied_space_weights)[:num], np.float64)
    return num, clouds, hy, xs, ns, o


def ceres3d_evaluate(clouds_and_grids, pose, target_translation, target_rotation,
                     occupied_space_weights=(5.0, 30.0), translation_weight=10.0,
                     rotation_weight=1.0, jacobian=True):
    """clouds_and_grids = [(xyz, HybridGrid), ...]; pose = {t xyz, q wxyz}.  Residuals
    (sum n + 6) and the tangent-space Jacobian (rows x 6)."""
    num, clouds, hy, xs, ns, o = _ceres3d_args(clouds_and_grids, occupied_space_weights,
                                               translation_weight, rotation_weight, False, 1)
    rows = int(ns.sum()) + 6
    res = np.zeros(rows, np.float64)
    jac = np.zeros((rows, 6), np.float64) if jacobian else None
    p = np.ascontiguousarray(pose, np.float64)
    tt = np.ascontiguousarray(target_translation, np.float64)
    tq = np.ascontiguousarray(target_rotation, np.float64)
    lib().orc_ceres3d_evaluate(hy, xs, _p(ns, C.c_int32), C.c_int(num), _p(o, C.c_double),
                               _p(tt, C.c_double), _p(tq, C.c_double), _p(p, C.c_double),
                               _p(res, C.c_double), _p(jac, C.c_double) if jacobian else None)
    return res, jac


def ceres3d_match(clouds_and_grids, target_translation, initial_pose,
                  occupied_space_weights=(5.0, 30.0), translation_weight=10.0,
                  rotation_weight=1.0, use_nonmonotonic_steps=False, max_num_iterations=10,
                  trace=False):
    """CeresScanMatcher3D::Match (no intensity grids, only_optimize_yaw = false); with trace
    also "trace", the per-iteration records."""
    num, clouds, hy, xs, ns, o = _ceres3d_args(clouds_and_grids, occupied_space_weights,
                                               translation_weight, rotation_weight,
                                               use_nonmonotonic_steps, max_num_iterations)
    tt = np.ascontiguousarray(target_translation, np.float64)
    ip = np.ascontiguousarray(initial_pose, np.float64)
    pose = np.zeros(7, np.float64)
    sm = np.zeros(5, np.float64)
    args = (hy, xs, _p(ns, C.c_int32), C.c_int(num), _p(o, C.c_double), _p(tt, C.c_double),
            _p(ip, C.c_double), _p(pose, C.c_double), _p(sm, C.c_double))
    extra = {}
    if trace:
        extra["trace"] = _traced(lambda buf, cap: lib().orc_ceres3d_match_traced(*args, buf, cap))
    else:
        lib().orc_ceres3d_match(*args)
    return dict(pose=pose, initial_cost=float(sm[0]), final_cost=float(sm[1]),
                iterations=int(sm[2]), num_successful_steps=int(sm[3]),
                termination=CERES_TERMINATION[int(sm[4])], **extra)
