"""3D fixtures shared by the oracle and GPU tests (CPU, numpy)."""
import math

import numpy as np

from benchmarks import synthetic

# fast_correlative_scan_matcher_3d_test.cc:42-55
AXIS_CLOUD = np.array([[4, 0, 0], [4.5, 0, 0], [5, 0, 0], [5.5, 0, 0],
                       [0, 4, 0], [0, 4.5, 0], [0, 5, 0], [0, 5.5, 0],
                       [0, 0, 4], [0, 0, 4.5], [0, 0, 5], [0, 0, 5.5]], np.float32)

# fast_correlative_scan_matcher_3d_test.cc:67-88
TEST_OPTIONS = dict(branch_and_bound_depth=6, full_resolution_depth=6, min_rotational_score=0.1,
                    min_low_resolution_score=0.15, linear_xy_search_window=0.8,
                    linear_z_search_window=0.8, angular_search_window=0.3)


def std_uniform_float(rng, a=-1.0, b=1.0):
    """std::uniform_real_distribution<float>(a, b)(std::mt19937) as libstdc++ computes
    it: one 32-bit draw, generate_canonical<float, 24> = float(draw) / 2^32 (clamped
    below 1), then * (b - a) + a in float.  numpy's RandomState(seed) is the same
    MT19937 stream as std::mt19937(seed), so the reference tests' random poses are
    reproduced exactly."""
    draw = int(rng.randint(0, 2 ** 32, dtype=np.uint32))
    ret = np.float32(draw) / np.float32(4294967296.0)
    if ret >= np.float32(1.0):
        ret = np.nextafter(np.float32(1.0), np.float32(0.0))
    return np.float32(ret * (np.float32(b) - np.float32(a)) + np.float32(a))


def random_pose(rng):
    """GetRandomPose (fast_correlative_scan_matcher_3d_test.cc:57-65) with
    std::mt19937(42): translation 0.7f * U(-1,1)^3, yaw 0.2f * U(-1,1); returned as
    [tx, ty, tz, qw, qx, qy, qz]."""
    x = np.float32(0.7) * std_uniform_float(rng)
    y = np.float32(0.7) * std_uniform_float(rng)
    z = np.float32(0.7) * std_uniform_float(rng)
    th = float(np.float32(0.2) * std_uniform_float(rng))
    return np.array([float(x), float(y), float(z), math.cos(th / 2), 0.0, 0.0,
                     math.sin(th / 2)])


def transform_points(pose7, pts):
    t, (w, x, y, z) = pose7[:3], pose7[3:]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return (np.asarray(pts, np.float64) @ R.T + t).astype(np.float32)


def range_insert_3d(resolution, origin, returns, hit=0.7, miss=0.4, free_voxels=5):
    """Stand-in for RangeDataInserter3D::Insert on an empty grid (mapping/3d/
    range_data_inserter_3d.cc:95-114, hit 0.7 / miss 0.4 / 5 free-space voxels as in
    the reference test): hit voxels get the hit probability, the `free_voxels`
    voxels in front of each hit get the miss probability unless they are hits."""
    hits = synthetic.cell_index_3d(returns, resolution)
    cells = {tuple(c): hit for c in hits}
    o = np.asarray(origin, np.float64)
    for p in np.asarray(returns, np.float64):
        d = p - o
        n = np.linalg.norm(d)
        if n < 1e-9:
            continue
        for k in range(1, free_voxels + 1):
            q = p - d / n * (k * resolution)
            c = tuple(synthetic.cell_index_3d(q[None, :].astype(np.float32), resolution)[0])
            cells.setdefault(c, miss)
    idx = np.array(list(cells.keys()), np.int32)
    vals = synthetic.probability_to_value(np.array(list(cells.values()), np.float32))
    return synthetic.HybridGridSpec(resolution, idx, vals)


def insert_cloud(oracle, resolution, pose7, cloud=AXIS_CLOUD):
    spec = range_insert_3d(resolution, pose7[:3], transform_points(pose7, cloud))
    g = oracle.HybridGrid(resolution, spec.indices, spec.values)
    g.spec = spec
    return g


def node_data(hi, low=None, hist=None, gravity=(1.0, 0.0, 0.0, 0.0)):
    return dict(gravity_alignment=gravity, high_resolution_point_cloud=hi,
                low_resolution_point_cloud=hi if low is None else low,
                rotational_scan_matcher_histogram=np.zeros(10, np.float32) if hist is None else hist)


def random_voxels(rng, n, extent, resolution, values=None, center=(0, 0, 0)):
    """n random voxels (unique) in center + [-extent, extent)^3 with random values in
    1 .. 32767, or `values` (a scalar or an array), as a HybridGridSpec."""
    idx = np.unique(rng.randint(-extent, extent, size=(n, 3)) + np.asarray(center), axis=0)
    if values is None:
        vals = rng.randint(1, 32768, size=len(idx))
    elif np.ndim(values):
        vals = np.asarray(values)[:len(idx)]
    else:
        vals = np.full(len(idx), values)
    return synthetic.HybridGridSpec(resolution, idx.astype(np.int32), vals.astype(np.uint16))


def random_cloud(rng, n, radius, center=(0.0, 0.0, 0.0)):
    """n points uniform in a cube of half-width `radius` around `center` (float32)."""
    return (rng.uniform(-radius, radius, size=(n, 3)) + np.asarray(center)).astype(np.float32)


def fast_options(depth=5, frd=3, xy=0.7, z=0.3, angular=0.05, min_rot=0.0, min_low=0.0):
    return dict(branch_and_bound_depth=depth, full_resolution_depth=frd,
                min_rotational_score=min_rot, min_low_resolution_score=min_low,
                linear_xy_search_window=xy, linear_z_search_window=z,
                angular_search_window=angular)


def search_window(options, resolution):
    """SearchParameters of Match (:127-144): (wxy, wz) = lround(window / resolution)."""
    res = np.float32(resolution)
    return (int(np.floor(options["linear_xy_search_window"] / res + 0.5)),
            int(np.floor(options["linear_z_search_window"] / res + 0.5)))


def to_score(sums, n):
    """PrecomputationGrid3D::ToProbability(sum / float(n)) (precomputation_grid_3d.h:32-35)."""
    k_min = np.float32(0.1)
    k = (np.float32(1.0) - k_min - k_min) / np.float32(255.0)
    return (k_min + (np.asarray(sums).astype(np.float32) / np.float32(n)) * k).astype(np.float32)


def make_pair(oracle, sm, hi, lo, od, hist=None):
    """The oracle's and the engine's FastCorrelativeScanMatcher3D on the same grids, the
    engine given the oracle's grid size (MatchFullSubmap's window depends on it)."""
    hist = np.zeros(10, np.float32) if hist is None else np.asarray(hist, np.float32)
    ohi = oracle.HybridGrid(hi.resolution, hi.indices, hi.values)
    olo = oracle.HybridGrid(lo.resolution, lo.indices, lo.values)
    om = oracle.FastCorrelativeScanMatcher3D(ohi, olo, hist, od)
    opts = sm.FastCorrelativeScanMatcherOptions3D(
        od["branch_and_bound_depth"], od["full_resolution_depth"], od["min_rotational_score"],
        od["min_low_resolution_score"], od["linear_xy_search_window"],
        od["linear_z_search_window"], od["angular_search_window"])
    m = sm.FastCorrelativeScanMatcher3D(hi, lo, hist, opts, grid_size_in_voxels=ohi.grid_size())
    return om, m


def engine_node(sm, d):
    return sm.TrajectoryNodeData3D(d["high_resolution_point_cloud"],
                                   d["low_resolution_point_cloud"],
                                   d["rotational_scan_matcher_histogram"], d["gravity_alignment"])


def numpy_sums(om, cells, depth, frd, wxy, wz, candidates):
    """ScoreCandidates' sums (fast_correlative_scan_matcher_3d.cc:332-355) in numpy over the
    oracle's level box: the per-depth cell indices of DiscretizeScan (:200-244), the
    candidate offset >> reduction_exponent, 0 outside the box.  cells: the full-resolution
    cells of the discrete scans (S x n x 3); candidates: m x {scan, x, y, z}."""
    cand = np.asarray(candidates, np.int64).reshape(-1, 4)
    e = max(0, depth - frd + 1)
    start = np.array([-wxy, -wxy, -wz], np.int64)
    c = np.asarray(cells, np.int64)
    if e:
        c = ((c + start) >> e) - (start >> e)
    pts = c[cand[:, 0]] + (cand[:, 1:4] >> e)[:, None, :]
    lo, box = om.level(depth)
    rel = pts - np.asarray(lo, np.int64)
    dims = np.array(box.shape[::-1], np.int64)
    inside = np.all((rel >= 0) & (rel < dims), axis=-1)
    rel = np.where(inside[..., None], rel, 0)
    v = np.where(inside, box[rel[..., 2], rel[..., 1], rel[..., 0]] if box.size else 0, 0)
    return v.astype(np.int64).sum(axis=1)


def _mat(p):
    t, (w, x, y, z) = p[:3], p[3:]
    M = np.eye(4, dtype=np.float32)
    M[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                 [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    M[:3, 3] = t
    return M


def is_nearly(a, b, eps):
    """transform/rigid_transform_test_helpers.h:42-46 (Eigen isApprox on the 4x4)."""
    A, B = _mat(np.asarray(a, np.float64)), _mat(np.asarray(b, np.float64))
    return float(((A - B) ** 2).sum()) <= eps * eps * min(float((A ** 2).sum()),
                                                         float((B ** 2).sum()))
