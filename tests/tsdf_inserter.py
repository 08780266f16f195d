"""Fixture builder for TSDF2D grids — TEST INFRASTRUCTURE ONLY, not product code.

Restates TSDFRangeDataInserter2D::Insert (mapping/internal/2d/tsdf_range_data_inserter_2d.cc)
with NormalEstimation2D (normal_estimation_2d.cc), the RangeDataSorter, the subpixel ray mask
of RayToPixelMask (ray_to_pixel_mask.cc) and TSDF2D's GetTSDAndWeight / SetCell, so that the
reference's cost-function tests (tsdf_match_cost_function_2d_test.cc) can be reproduced on the
grid they build.  Float arithmetic is float32 where the reference's is; the grid does not
grow (GrowAsNeeded) — a fixture whose rays leave the limits is refused.
"""
import math
from dataclasses import dataclass

import numpy as np

from tests import tsdf2d_oracle as T

F = np.float32
K_SUBPIXEL_SCALE = 1000
K_MIN_RANGE_METERS = F(1e-6)


@dataclass
class TSDFInserterOptions2D:
    """proto/tsdf_range_data_inserter_options_2d.proto"""
    truncation_distance: float = 0.3
    maximum_weight: float = 10.0
    update_free_space: bool = False
    num_normal_samples: int = 4
    sample_radius: float = 0.5
    project_sdf_distance_to_scan_normal: bool = True
    update_weight_range_exponent: int = 0
    update_weight_angle_scan_normal_to_ray_kernel_bandwidth: float = 0.5
    update_weight_distance_cell_to_hit_kernel_bandwidth: float = 0.5


def _norm(v):
    return F(math.sqrt(float(F(v[0]) * F(v[0]) + F(v[1]) * F(v[1]))))


def _sort_returns(returns, origin):
    """RangeDataSorter: by the direction from the origin, negative y first."""
    import functools

    def key_cmp(a, b):
        da = (a[:2] - origin) / _norm(a[:2] - origin)
        db = (b[:2] - origin) / _norm(b[:2] - origin)
        if (da[1] < 0) != (db[1] < 0):
            lt = da[1] < 0
            gt = db[1] < 0
        elif da[1] < 0:
            lt, gt = da[0] < db[0], db[0] < da[0]
        else:
            lt, gt = da[0] > db[0], db[0] > da[0]
        return -1 if lt else (1 if gt else 0)
    return sorted(returns, key=functools.cmp_to_key(key_cmp))


def _estimate_normal(returns, i, begin, end, origin3):
    p = returns[i]
    if end - begin < 2:
        d = origin3 - p
        return F(math.atan2(d[1], d[0]))
    mean = np.zeros(3, F)
    to_obs = origin3 - p
    for k in range(begin, end):
        if k == i:
            continue
        t = p - returns[k]
        n = np.array([-t[1], t[0], 0.0], F)
        if _norm(n) < F(1e-6):
            continue
        if float(np.dot(n, to_obs)) < 0:
            n = -n
        n = (n / _norm(n)).astype(F)
        mean = (mean + n).astype(F)
    return F(math.atan2(mean[1], mean[0]))


def estimate_normals(returns, origin3, num_normal_samples, sample_radius):
    """NormalEstimation2D::EstimateNormals over returns sorted by angle."""
    out = []
    n = len(returns)
    radius = F(sample_radius)
    for cur in range(n):
        hit = returns[cur]
        begin = cur
        while (begin > 0 and cur - begin < num_normal_samples // 2 and
               _norm(hit - returns[begin - 1]) < radius):
            begin -= 1
        end = cur
        while (end < n and end - cur < math.ceil(num_normal_samples / 2.0) + 1 and
               _norm(hit - returns[end]) < radius):
            end += 1
        out.append(_estimate_normal(returns, cur, begin, end, origin3))
    return out


def ray_to_pixel_mask(b, e, s):
    """RayToPixelMask: every pixel touched by the segment between the subpixel indices b, e."""
    if b[0] > e[0]:
        return ray_to_pixel_mask(e, b, s)
    assert b[0] >= 0 and b[1] >= 0 and e[1] >= 0
    mask = []

    def push(c):
        if not mask or mask[-1] != tuple(c):
            mask.append(tuple(c))
    if b[0] // s == e[0] // s:
        cur = [b[0] // s, min(b[1], e[1]) // s]
        mask.append(tuple(cur))
        end_y = max(b[1], e[1]) // s
        while cur[1] <= end_y:
            push(cur)
            cur[1] += 1
        return mask
    dx = e[0] - b[0]
    dy = e[1] - b[1]
    den = 2 * s * dx
    cur = [b[0] // s, b[1] // s]
    mask.append(tuple(cur))
    sub_y = (2 * (b[1] % s) + 1) * dx
    first_pixel = 2 * s - 2 * (b[0] % s) - 1
    last_pixel = 2 * (e[0] % s) + 1
    end_x = max(b[0], e[0]) // s
    sub_y += dy * first_pixel
    if dy > 0:
        while True:
            push(cur)
            while sub_y > den:
                sub_y -= den
                cur[1] += 1
                push(cur)
            cur[0] += 1
            if sub_y == den:
                sub_y -= den
                cur[1] += 1
            if cur[0] == end_x:
                break
            sub_y += dy * 2 * s
        sub_y += dy * last_pixel
        push(cur)
        while sub_y > den:
            sub_y -= den
            cur[1] += 1
            push(cur)
        return mask
    while True:
        push(cur)
        while sub_y < 0:
            sub_y += den
            cur[1] -= 1
            push(cur)
        cur[0] += 1
        if sub_y == 0:
            sub_y += den
            cur[1] -= 1
        if cur[0] == end_x:
            break
        sub_y += dy * 2 * s
    sub_y += dy * last_pixel
    push(cur)
    while sub_y < 0:
        sub_y += den
        cur[1] -= 1
        push(cur)
    return mask


def _gaussian(x, sigma):
    return F(1.0 / (math.sqrt(2.0 * math.pi) * sigma) * math.exp(-0.5 * x * x / (sigma * sigma)))


def _normalize_angle_difference(d):
    while d > math.pi:
        d -= 2.0 * math.pi
    while d < -math.pi:
        d += 2.0 * math.pi
    return F(d)


def _superscaled_index(g, p):
    """MapLimits(resolution / kSubpixelScale, max, ...)::GetCellIndex(p)"""
    r = g.resolution / K_SUBPIXEL_SCALE
    px, py = float(F(p[0])), float(F(p[1]))
    return (int(T.lround((g.max_y - py) / r - 0.5)), int(T.lround((g.max_x - px) / r - 0.5)))


def _update_cell(g, ix, iy, update_tsd, update_weight, maximum_weight):
    """TSDFRangeDataInserter2D::UpdateCell through GetTSDAndWeight / SetCell."""
    if update_weight == 0.0:
        return
    tsd = F(g.conv.min_tsd if (g.tsd_cells[iy, ix] & 0x7fff) == 0 else
            g.conv.value_to_cost(g.tsd_cells[iy, ix]))
    w = F(g.get_weight(ix, iy))
    updated_weight = F(w + update_weight)
    updated_sdf = F((tsd * w + update_tsd * update_weight) / updated_weight)
    updated_weight = min(updated_weight, F(maximum_weight))
    g.set_cell(ix, iy, updated_sdf, updated_weight)


def insert(g, origin_xy, returns_xyz, options):
    """TSDFRangeDataInserter2D::Insert of one RangeData into the TSDF2D `g` (in place),
    followed by FinishUpdate."""
    trunc = F(options.truncation_distance)
    origin = np.array(origin_xy[:2], F)
    origin3 = np.array([origin[0], origin[1], 0.0], F)
    returns = [np.asarray(p, F) for p in returns_xyz]
    # GrowAsNeeded: the fixture must already cover every ray end
    for p in returns:
        d = (p[:2] - origin) / _norm(p[:2] - origin)
        end = p[:2] + trunc * d
        assert (g.max_x - g.num_y * g.resolution < end[0] < g.max_x and
                g.max_y - g.num_x * g.resolution < end[1] < g.max_y), "the grid would grow"
    scale_angle = options.update_weight_angle_scan_normal_to_ray_kernel_bandwidth != 0.0
    normals = []
    if options.project_sdf_distance_to_scan_normal or scale_angle:
        returns = _sort_returns(returns, origin)
        normals = estimate_normals(returns, origin3, options.num_normal_samples,
                                   options.sample_radius)
    for k, p in enumerate(returns):
        hit = p[:2]
        normal = normals[k] if normals else F("nan")
        ray = (hit - origin).astype(F)
        rng = _norm(ray)
        if rng < trunc:
            continue
        ratio = F(trunc / rng)
        begin = origin if options.update_free_space else (origin + (F(1) - ratio) * ray).astype(F)
        end = (origin + (F(1) + ratio) * ray).astype(F)
        mask = ray_to_pixel_mask(_superscaled_index(g, begin), _superscaled_index(g, end),
                                 K_SUBPIXEL_SCALE)
        w_angle = F(1)
        if scale_angle:
            a = _normalize_angle_difference(float(normal) - math.atan2(-ray[1], -ray[0]))
            w_angle = _gaussian(a, options.update_weight_angle_scan_normal_to_ray_kernel_bandwidth)
        w_range = F(1)
        if options.update_weight_range_exponent != 0:
            w_range = (F(1) / F(float(rng) ** options.update_weight_range_exponent)
                       if abs(rng) > K_MIN_RANGE_METERS else F(0))
        for ix, iy in mask:
            if g.tsd_cells[iy, ix] >= T.UPDATE_MARKER:
                continue
            cx, cy = g.cell_center(ix, iy)
            center = np.array([cx, cy], F)
            update_tsd = F(rng - _norm(center - origin))
            if options.project_sdf_distance_to_scan_normal:
                v = (center - hit).astype(F)
                update_tsd = F(v[0] * F(math.cos(normal)) + v[1] * F(math.sin(normal)))
            update_tsd = F(min(max(update_tsd, -trunc), trunc))
            update_weight = F(w_range * w_angle)
            if options.update_weight_distance_cell_to_hit_kernel_bandwidth != 0.0:
                update_weight = F(update_weight * _gaussian(
                    float(update_tsd), options.update_weight_distance_cell_to_hit_kernel_bandwidth))
            _update_cell(g, ix, iy, update_tsd, update_weight, options.maximum_weight)
    g.finish_update()
    return g
