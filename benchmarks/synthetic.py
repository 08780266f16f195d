"""Seeded synthetic inputs for tests and bench.py (SURVEY.md §8d).

Pure numpy; no oracle, no CUDA.  Produces the flat records the C ABI consumes:
probability-grid cells (uint16, row-major ``num_x * y + x``), map limits, and
scan point clouds (N x 3 float32 in the sensor frame).

World 2D: a 50 m x 50 m procedural floor plan (outer walls, axis-aligned rooms
with door gaps, square pillars) rasterised at 5 cm; scans are 1081-beam / 270
degree ray casts with N(0, 1 cm) range noise, beams without a hit clamp to the
maximum range so N is always 1081.
"""
import math

import numpy as np

K_MIN_P = np.float32(0.1)
K_MAX_P = np.float32(1.0) - K_MIN_P
K_MIN_COST = np.float32(1.0) - K_MAX_P
K_MAX_COST = np.float32(1.0) - K_MIN_P


def correspondence_cost_to_value(cost):
    """mapping/probability_values.h:32-44 (BoundedFloatToValue) in float32."""
    c = np.clip(np.asarray(cost, np.float32), K_MIN_COST, K_MAX_COST)
    scaled = (c - K_MIN_COST) * (np.float32(32766.0) / (K_MAX_COST - K_MIN_COST))
    return (np.floor(scaled.astype(np.float64) + 0.5).astype(np.int64) + 1).astype(np.uint16)


def probability_to_cell_value(p):
    return correspondence_cost_to_value(np.float32(1.0) - np.asarray(p, np.float32))


class GridSpec:
    """Plain record of a ProbabilityGrid (cells[y, x]) + MapLimits."""

    def __init__(self, cells, resolution, max_x, max_y):
        self.cells = np.ascontiguousarray(cells, np.uint16)
        self.num_y, self.num_x = self.cells.shape
        self.resolution = float(resolution)
        self.max_x = float(max_x)
        self.max_y = float(max_y)
        self.min_cost = float(K_MIN_COST)
        self.max_cost = float(K_MAX_COST)


def world_to_cell(grid, wx, wy):
    """mapping/2d/map_limits.h:69-76: index.x <- world y, index.y <- world x."""
    cx = np.floor((grid.max_y - wy) / grid.resolution).astype(np.int64)
    cy = np.floor((grid.max_x - wx) / grid.resolution).astype(np.int64)
    return cx, cy


def make_floorplan(seed, size_m=50.0, resolution=0.05, rooms=8, pillars=20):
    """Boolean occupancy (cells[y, x]) of a procedural floor plan, plus limits.

    Returns (occ, max_x, max_y); world x in (max_x - size, max_x], same for y.
    """
    rng = np.random.RandomState(seed)
    n = int(round(size_m / resolution))
    occ = np.zeros((n, n), bool)
    t = 3  # wall thickness in cells
    occ[:t, :] = occ[-t:, :] = True
    occ[:, :t] = occ[:, -t:] = True
    for _ in range(rooms):
        w = rng.randint(n // 8, n // 3)
        h = rng.randint(n // 8, n // 3)
        x0 = rng.randint(t, n - w - t)
        y0 = rng.randint(t, n - h - t)
        wall = np.zeros_like(occ)
        wall[y0:y0 + t, x0:x0 + w] = True
        wall[y0 + h - t:y0 + h, x0:x0 + w] = True
        wall[y0:y0 + h, x0:x0 + t] = True
        wall[y0:y0 + h, x0 + w - t:x0 + w] = True
        # two door gaps per room
        for _d in range(2):
            side = rng.randint(4)
            g = rng.randint(20, 40)
            if side < 2:
                gx = rng.randint(x0 + t, max(x0 + t + 1, x0 + w - g - t))
                yy = y0 if side == 0 else y0 + h - t
                wall[yy:yy + t, gx:gx + g] = False
            else:
                gy = rng.randint(y0 + t, max(y0 + t + 1, y0 + h - g - t))
                xx = x0 if side == 2 else x0 + w - t
                wall[gy:gy + g, xx:xx + t] = False
        occ |= wall
    for _ in range(pillars):
        s = rng.randint(4, 12)
        x0 = rng.randint(t, n - s - t)
        y0 = rng.randint(t, n - s - t)
        occ[y0:y0 + s, x0:x0 + s] = True
    return occ, size_m / 2.0, size_m / 2.0


def occupancy_to_grid(occ, seed, resolution, max_x, max_y, unknown_fraction=0.25):
    """Wall cells p~U(0.70,0.90); free cells p~U(0.10,0.25); 25% unknown (value 0)."""
    rng = np.random.RandomState(seed + 7919)
    p = np.where(occ, rng.uniform(0.70, 0.90, occ.shape), rng.uniform(0.10, 0.25, occ.shape))
    cells = probability_to_cell_value(p.astype(np.float32))
    unknown = (rng.uniform(size=occ.shape) < unknown_fraction) & ~occ
    cells[unknown] = 0
    return GridSpec(cells, resolution, max_x, max_y)


def make_grid2d(seed, size_cells=1000, resolution=0.05):
    size_m = size_cells * resolution
    occ, max_x, max_y = make_floorplan(seed, size_m=size_m, resolution=resolution,
                                       rooms=max(2, int(8 * size_m / 50.0)),
                                       pillars=max(3, int(20 * size_m / 50.0)))
    return occupancy_to_grid(occ, seed, resolution, max_x, max_y), occ


class TSDFGridSpec:
    """Plain record of a TSDF2D (tsd_cells[y, x], weight_cells[y, x]) + MapLimits + the
    TSDValueConverter parameters; the fields of scan_matching.TSDF2DSpec."""

    def __init__(self, tsd_cells, weight_cells, resolution, max_x, max_y, truncation_distance,
                 max_weight):
        self.tsd_cells = np.ascontiguousarray(tsd_cells, np.uint16)
        self.weight_cells = np.ascontiguousarray(weight_cells, np.uint16)
        self.num_y, self.num_x = self.tsd_cells.shape
        self.resolution = float(resolution)
        self.max_x = float(max_x)
        self.max_y = float(max_y)
        self.truncation_distance = float(truncation_distance)
        self.max_weight = float(max_weight)


def make_tsdf2d(seed, size_cells=1000, resolution=0.05, truncation_distance=0.3,
                max_weight=10.0):
    """The world of make_grid2d(seed, ...) as a TSDF2D: the signed distance to its walls
    (positive in free space, negative inside walls), clamped to +-truncation_distance
    (configuration_files/trajectory_builder_2d.lua: 0.3 m, max weight 10).  Cells within the
    truncation band carry a weight that falls from max_weight at the wall to half of it at the
    band's edge; the others are unknown (value 0, weight 0).  Values as TSDValueConverter
    stores them (float32, lround).  Returns (spec, occ)."""
    _, occ = make_grid2d(seed, size_cells=size_cells, resolution=resolution)
    ny, nx = occ.shape
    reach = int(math.ceil(truncation_distance / resolution)) + 1
    # distance (in cells, between cell centres) to the nearest cell of the other kind
    dist = np.full(occ.shape, np.inf)
    pad = np.pad(occ, reach, mode="edge")
    for dy in range(-reach, reach + 1):
        for dx in range(-reach, reach + 1):
            d = math.hypot(dx, dy)
            if d == 0 or d > reach:
                continue
            other = pad[reach + dy:reach + dy + ny, reach + dx:reach + dx + nx] != occ
            dist = np.where(other & (d < dist), d, dist)
    # the surface lies half a cell from either centre
    sd = np.where(occ, -1.0, 1.0) * (dist - 0.5) * resolution
    band = np.abs(sd) < truncation_distance
    trunc = np.float32(truncation_distance)
    tsd = np.clip(sd.astype(np.float32), -trunc, trunc)
    weight = (max_weight * (1.0 - 0.5 * np.abs(sd) / truncation_distance)).astype(np.float32)
    weight = np.clip(weight, np.float32(0), np.float32(max_weight))
    tsd_resolution = np.float32(32766) / (trunc - (-trunc))
    w_resolution = np.float32(32766) / (np.float32(max_weight) - np.float32(0))

    def lround(v):   # std::lround: halves away from zero
        v = v.astype(np.float64)
        return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)
    tsd_v = lround((tsd - (-trunc)) * tsd_resolution) + 1
    w_v = lround((weight - np.float32(0)) * w_resolution) + 1
    tsd_cells = np.where(band, tsd_v, 0).astype(np.uint16)
    weight_cells = np.where(band, w_v, 0).astype(np.uint16)
    size_m = size_cells * resolution
    return TSDFGridSpec(tsd_cells, weight_cells, resolution, size_m / 2.0, size_m / 2.0,
                        truncation_distance, max_weight), occ


def crop_grid(grid, occ, x0, y0, nx, ny):
    """Sub-grid of nx x ny cells starting at cell (x0, y0); limits shifted accordingly."""
    cells = grid.cells[y0:y0 + ny, x0:x0 + nx]
    # cell (x0, y0) of the parent becomes (0, 0): max shifts by resolution * (y0, x0)
    return (GridSpec(cells, grid.resolution, grid.max_x - grid.resolution * y0,
                     grid.max_y - grid.resolution * x0), occ[y0:y0 + ny, x0:x0 + nx])


def random_free_pose(occ, grid, rng, margin_cells=20):
    ny, nx = occ.shape
    while True:
        cx = rng.randint(margin_cells, nx - margin_cells)
        cy = rng.randint(margin_cells, ny - margin_cells)
        if not occ[max(0, cy - 4):cy + 5, max(0, cx - 4):cx + 5].any():
            wx = grid.max_x - (cy + 0.5) * grid.resolution
            wy = grid.max_y - (cx + 0.5) * grid.resolution
            return np.array([wx, wy, rng.uniform(-math.pi, math.pi)])


def cast_scan(occ, grid, pose, beams=1081, fov_deg=270.0, max_range=30.0, noise=0.01, seed=0):
    """Ray-cast a planar lidar from `pose` (world x, y, yaw); returns N x 3 float32 in the
    sensor frame.  Beams with no hit clamp to max_range."""
    rng = np.random.RandomState(seed)
    ang = np.deg2rad(np.linspace(-fov_deg / 2.0, fov_deg / 2.0, beams))
    step = grid.resolution * 0.5
    steps = np.arange(1, int(max_range / step) + 1) * step                  # (T,)
    ca, sa = np.cos(ang + pose[2]), np.sin(ang + pose[2])
    ranges = np.full(beams, max_range)
    ny, nx = occ.shape
    alive = np.ones(beams, bool)
    chunk = 128
    for t0 in range(0, len(steps), chunk):
        r = steps[t0:t0 + chunk]                                             # (c,)
        wx = pose[0] + np.outer(ca, r)
        wy = pose[1] + np.outer(sa, r)
        cx, cy = world_to_cell(grid, wx, wy)
        inside = (cx >= 0) & (cx < nx) & (cy >= 0) & (cy < ny)
        hit = np.zeros_like(inside)
        hit[inside] = occ[cy[inside], cx[inside]]
        hit |= ~inside                                                       # leaving the map ends the ray
        any_hit = hit.any(axis=1) & alive
        first = hit.argmax(axis=1)
        rr = r[first]
        left_map = ~inside[np.arange(beams), first]
        ranges[any_hit] = np.where(left_map[any_hit], max_range, rr[any_hit])
        alive &= ~any_hit
        if not alive.any():
            break
    ranges = np.clip(ranges + rng.normal(0.0, noise, beams), 0.05, max_range)
    pts = np.zeros((beams, 3), np.float32)
    pts[:, 0] = (ranges * np.cos(ang)).astype(np.float32)
    pts[:, 1] = (ranges * np.sin(ang)).astype(np.float32)
    return pts


# ===========================================================================
# 3D
# ===========================================================================
def probability_to_value(p):
    """mapping/probability_values.h:91-93 (ProbabilityToValue) in float32."""
    p = np.clip(np.asarray(p, np.float32), K_MIN_P, K_MAX_P)
    scaled = (p - K_MIN_P) * (np.float32(32766.0) / (K_MAX_P - K_MIN_P))
    return (np.floor(scaled.astype(np.float64) + 0.5).astype(np.int64) + 1).astype(np.uint16)


class HybridGridSpec:
    """Flat record of a HybridGrid: voxel indices (n x 3 int32), values (n uint16)."""

    def __init__(self, resolution, indices, values):
        self.resolution = float(np.float32(resolution))
        self.indices = np.ascontiguousarray(indices, np.int32).reshape(-1, 3)
        self.values = np.ascontiguousarray(values, np.uint16).reshape(-1)


def cell_index_3d(points, resolution):
    """HybridGridBase::GetCellIndex (mapping/3d/hybrid_grid.h:428-433): lround(p / res)."""
    q = np.asarray(points, np.float32) / np.float32(resolution)
    return (np.sign(q) * np.floor(np.abs(q).astype(np.float64) + 0.5)).astype(np.int32)


def grid_from_points(points, resolution, seed=0, p_lo=0.6, p_hi=0.9):
    """Voxelise surface points into a HybridGrid record with hit probabilities."""
    idx = np.unique(cell_index_3d(points, resolution), axis=0)
    rng = np.random.RandomState(seed + 31)
    vals = probability_to_value(rng.uniform(p_lo, p_hi, len(idx)).astype(np.float32))
    return HybridGridSpec(resolution, idx, vals)


def make_building(seed, size_m=40.0, height_m=6.0, cell=0.1):
    """Boolean occupancy volume occ[z, y, x] of a two-storey box-and-pillars building
    (walls extruded from the 2D floor plan, floor slabs at z = 0, h/2, h) centred at
    the origin in x/y, z in [0, height]."""
    occ2, _, _ = make_floorplan(seed, size_m=size_m, resolution=cell,
                                rooms=max(2, int(6 * size_m / 40.0)),
                                pillars=max(3, int(12 * size_m / 40.0)))
    n = occ2.shape[0]
    nz = int(round(height_m / cell)) + 1
    occ = np.zeros((nz, n, n), bool)
    occ[:] = occ2[None, :, :]
    for zs in (0, nz // 2, nz - 1):
        occ[zs] = True
    return occ, cell, np.array([-size_m / 2.0, -size_m / 2.0, 0.0])


def building_surface_points(occ, cell, origin):
    z, y, x = np.nonzero(occ)
    return (np.stack([x, y, z], axis=1).astype(np.float32) + 0.5) * np.float32(cell) + \
        origin.astype(np.float32)


def cast_lidar_3d(occ, cell, origin, pose_xyzyaw, rings=16, azimuths=2048, vfov_deg=15.0,
                  max_range=20.0, noise=0.01, seed=0):
    """Multi-ring lidar (VLP-16 like) ray-cast in the occupancy volume.  Returns the
    hit points in the sensor frame (rays without a hit inside max_range are dropped)."""
    rng = np.random.RandomState(seed)
    el = np.deg2rad(np.linspace(-vfov_deg, vfov_deg, rings))
    az = np.linspace(-math.pi, math.pi, azimuths, endpoint=False)
    E, A = np.meshgrid(el, az, indexing="ij")
    d_s = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], axis=-1).reshape(-1, 3)
    yaw = pose_xyzyaw[3]
    c, s = math.cos(yaw), math.sin(yaw)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    d_w = d_s @ R.T
    o = np.asarray(pose_xyzyaw[:3], np.float64)
    nrays = len(d_w)
    ranges = np.full(nrays, np.inf)
    alive = np.ones(nrays, bool)
    step = cell * 0.5
    nz, ny, nx = occ.shape
    ts = np.arange(1, int(max_range / step) + 1) * step
    for t0 in range(0, len(ts), 64):
        t = ts[t0:t0 + 64]
        idx = np.nonzero(alive)[0]
        if len(idx) == 0:
            break
        p = o[None, None, :] + d_w[idx, None, :] * t[None, :, None]
        c3 = np.floor((p - origin[None, None, :]) / cell).astype(np.int64)
        inside = ((c3[..., 0] >= 0) & (c3[..., 0] < nx) & (c3[..., 1] >= 0) & (c3[..., 1] < ny) &
                  (c3[..., 2] >= 0) & (c3[..., 2] < nz))
        hit = np.zeros(inside.shape, bool)
        ci = c3[inside]
        hit[inside] = occ[ci[:, 2], ci[:, 1], ci[:, 0]]
        any_hit = hit.any(axis=1)
        first = hit.argmax(axis=1)
        ranges[idx[any_hit]] = t[first[any_hit]]
        alive[idx[any_hit]] = False
    ok = np.isfinite(ranges)
    r = ranges[ok] + rng.normal(0.0, noise, ok.sum())
    return (d_s[ok] * r[:, None]).astype(np.float32)


def voxel_downsample(points, size):
    """One point per `size` voxel (first occurrence) — stand-in for sensor::VoxelFilter."""
    key = np.floor(np.asarray(points, np.float64) / size).astype(np.int64)
    _, first = np.unique(key, axis=0, return_index=True)
    return np.ascontiguousarray(np.asarray(points, np.float32)[np.sort(first)])


def rotational_histogram(points, size=120, slice_height=0.2, jitter_deg=2.0, seed=0):
    """Stand-in for RotationalScanMatcher::ComputeHistogram (producer side, out of scope;
    rotational_scan_matcher.cc:164-176): per z-slice, points sorted by angle around the
    slice centroid, histogram of the direction of consecutive-point segments weighted
    by how orthogonal they are to the ray from the centroid."""
    pts = np.asarray(points, np.float64)
    hist = np.zeros(size, np.float32)
    sl = np.round(pts[:, 2] / slice_height).astype(np.int64)
    for s in np.unique(sl):
        p = pts[sl == s]
        if len(p) < 3:
            continue
        cen = p.mean(axis=0)
        d = p[:, :2] - cen[:2]
        keep = np.linalg.norm(d, axis=1) >= 0.2
        p, d = p[keep], d[keep]
        order = np.argsort(np.arctan2(d[:, 1], d[:, 0]), kind="stable")
        p, d = p[order], d[order]
        delta = p[1:, :2] - p[:-1, :2]
        dist = np.linalg.norm(delta, axis=1)
        direction = d[1:]
        ok = (dist >= 0.2) & (dist <= 0.9) & (np.linalg.norm(direction, axis=1) >= 0.2)
        if not ok.any():
            continue
        delta, direction, dist = delta[ok], direction[ok], dist[ok]
        ang = np.arctan2(delta[:, 1], delta[:, 0])
        if jitter_deg > 0:  # real walls are not perfectly straight: broaden the peaks a little
            ang = ang + np.random.RandomState(seed + int(s) + 977).normal(
                0.0, math.radians(jitter_deg), len(ang))
        ang = np.mod(ang, math.pi)
        val = np.maximum(0.0, 1.0 - np.abs(np.sum(delta / dist[:, None] * direction /
                                                  np.linalg.norm(direction, axis=1)[:, None], axis=1)))
        b = np.clip(np.floor(size * ang / math.pi).astype(np.int64), 0, size - 1)
        np.add.at(hist, b, val.astype(np.float32))
    return hist


def rotate_histogram(hist, angle):
    """RotationalScanMatcher::RotateHistogram (rotational_scan_matcher.cc:141-162) in
    numpy (input generation only): rotate by `angle` with fractional-bucket interpolation."""
    h = np.asarray(hist, np.float32)
    n = len(h)
    rot = -angle * n / math.pi
    full = int(np.floor(rot))
    frac = np.float32(rot - full)
    idx = np.arange(n)
    return frac * h[(idx + 1 + full) % n] + (np.float32(1.0) - frac) * h[(idx + full) % n]


def yaw_pose7(x, y, z, yaw):
    return np.array([x, y, z, math.cos(yaw / 2.0), 0.0, 0.0, math.sin(yaw / 2.0)])


def random_free_pose_3d(occ, cell, origin, rng, heights=(1.2,), margin_m=4.0):
    nz, ny, nx = occ.shape
    for _ in range(500):
        pose = np.array([rng.uniform(origin[0] + margin_m, origin[0] + nx * cell - margin_m),
                         rng.uniform(origin[1] + margin_m, origin[1] + ny * cell - margin_m),
                         rng.choice(heights), rng.uniform(-math.pi, math.pi)])
        c = np.floor((pose[:3] - origin) / cell).astype(int)
        if not occ[max(0, c[2] - 3):c[2] + 4, c[1] - 4:c[1] + 5, c[0] - 4:c[0] + 5].any():
            return pose
    raise RuntimeError("no free pose found")


def make_submap3d(seed, size_m=40.0, rings=16, azimuths=2048, max_range=20.0, map_scans=10,
                  hist_size=120, hi_res=0.10, lo_res=0.45):
    """A 3D submap the way Cartographer builds one: `map_scans` lidar scans from
    random free poses are inserted (hit voxels, p ~ U(0.6, 0.9)) into a high- and a
    low-resolution hybrid grid, and their rotated histograms are accumulated
    (mapping/3d/submap_3d.cc:289-293).  Returns (hi, lo, submap_histogram, world) where
    world = (occ, cell, origin) for casting further node scans."""
    occ, cell, origin = make_building(seed, size_m=size_m, height_m=6.0, cell=0.1)
    rng = np.random.RandomState(seed + 101)
    pts, hist, map_poses = [], np.zeros(hist_size, np.float32), []
    for k in range(map_scans):
        pose = random_free_pose_3d(occ, cell, origin, rng, heights=(1.2, 4.2))
        map_poses.append(pose)
        cloud = cast_lidar_3d(occ, cell, origin, pose, rings=rings, azimuths=azimuths,
                              max_range=max_range, seed=seed * 1000 + k)
        c, s = math.cos(pose[3]), math.sin(pose[3])
        world = cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T + pose[:3]
        pts.append(world.astype(np.float32))
        hist += rotate_histogram(rotational_histogram(cloud, hist_size), pose[3])
    pts = np.concatenate(pts)
    return (grid_from_points(pts, hi_res, seed), grid_from_points(pts, lo_res, seed + 1), hist,
            (occ, cell, origin, map_poses))


def make_node3d(world, rng, rings=16, azimuths=2048, max_range=20.0, seed=0, hist_size=120,
                lo_res=0.45, jitter=0.7):
    """A node to match against a submap: one lidar scan taken near one of the poses
    the submap was built from (a revisit, as in loop closure).  `jitter` (m) is how far
    from that pose: smaller = more of the scan falls on mapped surfaces."""
    occ, cell, origin, map_poses = world
    for _ in range(200):
        base = map_poses[rng.randint(len(map_poses))]
        pose = base + np.array([rng.uniform(-jitter, jitter), rng.uniform(-jitter, jitter), 0.0,
                                rng.uniform(-0.4, 0.4)])
        c = np.floor((pose[:3] - origin) / cell).astype(int)
        if not occ[max(0, c[2] - 2):c[2] + 3, c[1] - 2:c[1] + 3, c[0] - 2:c[0] + 3].any():
            break
    cloud = cast_lidar_3d(occ, cell, origin, pose, rings=rings, azimuths=azimuths,
                          max_range=max_range, seed=seed)
    return dict(pose=yaw_pose7(*pose), cloud=cloud, low=voxel_downsample(cloud, lo_res),
                hist=rotational_histogram(cloud, hist_size))


def surface_intensity(world, points_world, seed=0, bright_fraction=0.01):
    """Per-point intensities of world-frame points on the building's surfaces: each 0.5 m
    block of the occupancy volume has one seeded reflectivity in [10, 90), each return adds
    N(0, 2) noise, and `bright_fraction` of them are retroreflections at 200.  Draws from its
    own RNG streams, so no other generator's output depends on it."""
    occ, cell, origin = world[0], world[1], world[2]
    block = max(1, int(round(0.5 / cell)))
    shape = tuple(-(-s // block) for s in occ.shape)
    table = np.random.RandomState(seed + 60013).uniform(10.0, 90.0, shape).astype(np.float32)
    c = np.floor((np.asarray(points_world, np.float64) - origin) / cell).astype(np.int64) // block
    for a, s in zip((0, 1, 2), (shape[2], shape[1], shape[0])):
        c[:, a] = np.clip(c[:, a], 0, s - 1)
    rng = np.random.RandomState(seed + 60017)
    v = table[c[:, 2], c[:, 1], c[:, 0]] + rng.normal(0.0, 2.0, len(c)).astype(np.float32)
    v[rng.uniform(size=len(c)) < bright_fraction] = 200.0
    return np.maximum(v, 0.0).astype(np.float32)


def make_intensity_grid3d(hybrid_grid, world, seed=0):
    """An IntensityHybridGrid over the voxels of `hybrid_grid` (the submap's high-resolution
    grid): each voxel averages 1-3 returns of its surface's intensity (surface_intensity
    without retroreflections), as AverageIntensityData {sum, count}."""
    from cartographer_b200.scan_matching import IntensityGridSpec
    idx = hybrid_grid.indices
    centres = idx.astype(np.float64) * hybrid_grid.resolution
    counts = np.random.RandomState(seed + 60019).randint(1, 4, len(idx)).astype(np.int32)
    mean = surface_intensity(world, centres, seed, bright_fraction=0.0)
    sums = (mean * counts).astype(np.float32)
    return IntensityGridSpec(hybrid_grid.resolution, idx, sums, counts)


def node_intensities(world, node, seed=0):
    """PointCloud::intensities() of a make_node3d scan: surface_intensity at its world points."""
    p = node["pose"]
    yaw = 2.0 * math.atan2(p[6], p[3])
    c, s = math.cos(yaw), math.sin(yaw)
    w = node["cloud"].astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T + p[:3]
    return surface_intensity(world, w, seed)
