"""Test-side references for the 3D map-writing edge tests — TEST INFRASTRUCTURE ONLY.

* ulp_neighbours(): a float32 value and its two float32 neighbours.
* submap_frame64() / range_sides64() / cell_sides64(): the submap transform, the
  high-resolution range filter (submap_3d.cc:41-49) and GetCellIndex (hybrid_grid.h:428-433) in
  float64 from a rotation matrix, independent of rigid3f.h and its operation order.  Each side
  comes with a bound on the float32 computation's error; a point whose float64 margin is inside
  the bound is undecided (0), any other is decided (+1 / -1 for the range filter, the cell for
  GetCellIndex).
* slack_box(): the box a grown handle gets (DESIGN §9): extent / 8 voxels per side, clamped to
  the 2^14 cube.
* lane_keep(): which returns of a launch a keep pattern keeps, by lane and warp.
Checked against brute-force and exact-arithmetic versions in tests/test_map_writing3d_refs_cpu.py.
"""
import numpy as np

F = np.float32
CUBE = 8192
# float32 ulps of the largest magnitude in play that the device's transform, norm and quotient
# may be off by (a rotation and a translation, three products, two sums, a square root, a
# division, each within half an ulp, and the float32 cast of the pose): generous on purpose
F32_ERROR_ULPS = 16.0


def ulp_neighbours(x):
    """(x - 1 ulp, x, x + 1 ulp) in float32, elementwise."""
    x = np.asarray(x, F)
    return (np.nextafter(x, F(-np.inf)).astype(F), x, np.nextafter(x, F(np.inf)).astype(F))


def ulp32(x):
    """The float32 ulp of |x| (elementwise), at least that of the smallest normal."""
    a = np.maximum(np.abs(np.asarray(x, np.float64)), np.finfo(F).tiny)
    return np.spacing(a.astype(F)).astype(np.float64)


def rotation64(q):
    """The rotation matrix of the unit quaternion (w, x, y, z), in float64."""
    w, x, y, z = (float(v) for v in q)
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def submap_frame64(pose, points):
    """local_pose.inverse() * p for pose (tx, ty, tz, qw, qx, qy, qz), in float64: R^T (p - t).
    Also the magnitude each result's float32 error scales with."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    t = np.asarray(pose[:3], np.float64)
    out = (p - t) @ rotation64(pose[3:])
    scale = np.maximum(np.abs(p).max(1), np.abs(t).max())
    return out, np.maximum(scale, np.abs(out).max(1))


def range_sides64(pose, origin, points, max_range):
    """+1 kept, -1 dropped, 0 undecided: |p - o| <= max_range in the submap frame."""
    o, so = submap_frame64(pose, origin)
    p, sp = submap_frame64(pose, points)
    margin = max_range - np.linalg.norm(p - o, axis=1)
    bound = F32_ERROR_ULPS * (ulp32(np.maximum(sp, so[0])) + ulp32(max_range))
    return np.where(margin > bound, 1, np.where(margin < -bound, -1, 0))


def lround64(q):
    """std::lround of float64 values (halves away from zero)."""
    q = np.asarray(q, np.float64)
    return (np.sign(q) * np.floor(np.abs(q) + 0.5)).astype(np.int64)


def cell_sides64(points, resolution, scale=None):
    """(cells, decided): GetCellIndex of float64 points at the float32 resolution, and per point
    whether every axis's quotient is farther from a half-integer than the float32 error bound.
    `scale`: the magnitude the points' own float32 error scales with (the points themselves when
    they are float32 inputs)."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    res = float(F(resolution))
    q = p / res
    if scale is None and np.frexp(res)[0] == 0.5:   # a power of two: the quotient is exact
        return lround64(q), np.ones(len(p), bool)
    frac = np.abs(np.abs(q) - np.floor(np.abs(q)) - 0.5)
    if scale is None:   # exact float32 inputs: only the quotient's rounding, half an ulp
        bound = ulp32(q)
    else:
        s = np.asarray(scale, np.float64).reshape(-1, 1)
        bound = F32_ERROR_ULPS * (ulp32(q) + ulp32(s) / res)
    return lround64(q), np.all(frac > bound, axis=1)


def slack_box(lo, hi):
    """(box lo, dims) a handle grows to around the tight box lo .. hi (inclusive)."""
    lo, hi = np.asarray(lo, np.int64), np.asarray(hi, np.int64)
    s = (hi - lo + 1) // 8
    blo = np.maximum(-CUBE, lo - s)
    return blo, np.minimum(CUBE - 1, hi + s) - blo + 1


KEEP_PATTERNS = ("all", "none", "lane0", "lane31", "alternating", "warps_dropped")


def lane_keep(pattern, n):
    """Which of n returns a pattern keeps: lane = i % 32, warp = i // 32."""
    i = np.arange(n)
    lane, warp = i % 32, i // 32
    return {"all": np.ones(n, bool), "none": np.zeros(n, bool), "lane0": lane == 0,
            "lane31": lane == 31, "alternating": i % 2 == 0,
            "warps_dropped": warp % 3 != 1}[pattern]
