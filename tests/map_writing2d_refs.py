"""Test-side references for the 2D map-writing edge tests — TEST INFRASTRUCTURE ONLY.

Written in exact or float64 arithmetic from the reference's definitions, sharing no code with
tests/insert2d_oracle.cc, tests/insert_tsdf2d_oracle.cc or tests/tsdf_inserter.py:

* cell_index_exact(): MapLimits::GetCellIndex of a float32 point at double limits, from the exact
  quotient (fractions.Fraction), with a flag that says whether the double computation can only
  round to that cell.
* geometric_mask(): the pixels a superscaled ray covers, from the segment itself rather than an
  integer walk; count_bound() is the |dx| + |dy| + 1 slot count of one ray.
* grow_limits() / expected_probability_grid(): ProbabilityGridRangeDataInserter2D::Insert as
  sets of cells (hit cells, mask cells, the rest), with the known-cells box.
* tsdf_expected(): TSDFRangeDataInserter2D::Insert without normals (no projection, no angle
  weight: the rays keep their input order) in float64, each cell's winner and its quantised
  values, with a flag wherever float32 could land on the other side of a rounding boundary.
* slot_reservation() / exact_slot_total(): the host's per-handle slot range and the device's
  exact per-handle total.
* keep patterns by lane, partial warp and last block, and a grid maker whose pitch * ny is a
  chosen number.
Checked against brute force and the restatements in tests/test_map_writing2d_refs_cpu.py.
"""
import math
from fractions import Fraction

import numpy as np

F = np.float32
SUBPIXEL = 1000
MAX_CELLS = 30000
VALUE_COUNT = 32768
# double ulps the GetCellIndex quotient may be off by: a subtraction, a division and the - 0.5,
# each within half an ulp of a value no larger than the quotient's magnitude; generous on purpose
F64_ERROR_ULPS = 8.0
# float32 ulps of the range that a TSDF update may be off by (the range, the cell centre's
# distance and their difference; the weighted average's product, sum and division)
F32_ERROR_ULPS = 16.0


# ---------------------------------------------------------------------------------------------
# GetCellIndex
# ---------------------------------------------------------------------------------------------
def _round_half_away(q):
    """llround of an exact Fraction."""
    f = math.floor(abs(q) + Fraction(1, 2))
    return f if q >= 0 else -f


def _axis_exact(lim, p, res):
    """(index, decided) of llround((lim - p) / res - 0.5) for doubles lim, res and float32 p."""
    d = Fraction(float(lim)) - Fraction(float(F(p)))
    q = d / Fraction(float(res)) - Fraction(1, 2)
    frac = abs(q) - math.floor(abs(q))
    dist = abs(frac - Fraction(1, 2))
    bound = F64_ERROR_ULPS * 2.0 ** -52 * (abs(float(d)) / float(res) + 1.0)
    return _round_half_away(q), float(dist) > bound


def cell_index_double(resolution, max_x, max_y, px, py):
    """GetCellIndex as the double operations round it, for the undecided points: Python floats
    are IEEE doubles, and each operation here is one rounded operation."""
    def axis(lim, p):
        q = (float(lim) - float(F(p))) / float(resolution) - 0.5
        return int(math.floor(abs(q) + 0.5)) * (1 if q >= 0 else -1)
    return axis(max_y, py), axis(max_x, px)


def cell_index_exact(resolution, max_x, max_y, px, py):
    """(ix, iy, decided): GetCellIndex (map_limits.h:69-76), ix from y and iy from x.  Pass the
    superscaled resolution as the double the caller computes (resolution / 1000)."""
    ix, dx = _axis_exact(max_y, py, resolution)
    iy, dy = _axis_exact(max_x, px, resolution)
    return ix, iy, dx and dy


# ---------------------------------------------------------------------------------------------
# Ray masks
# ---------------------------------------------------------------------------------------------
def count_bound(b, e, s=SUBPIXEL):
    """|dx| + |dy| + 1 in pixels: the slots one ray is given."""
    return abs(e[0] // s - b[0] // s) + abs(e[1] // s - b[1] // s) + 1


def geometric_mask(b, e, s=SUBPIXEL):
    """The set of pixels (X, Y) whose open square (X s, (X + 1) s) x (Y s, (Y + 1) s) the
    segment from (b + 1/2) to (e + 1/2) meets, in subpixel units; b, e non-negative.  The ends
    lie on no border (k + 1/2), so their pixels are among them."""
    assert min(b[0], b[1], e[0], e[1]) >= 0
    if b[0] > e[0]:
        b, e = e, b
    # doubled coordinates: the ends are odd integers, the borders multiples of 2 s
    bx, by = 2 * b[0] + 1, 2 * b[1] + 1
    dx, dy = 2 * (e[0] - b[0]), 2 * (e[1] - b[1])
    S = 2 * s
    out = set()
    for X in range(bx // S, (bx + dx) // S + 1):
        if dx == 0:
            lo, hi = Fraction(0), Fraction(1)
        else:   # t where x is strictly inside the column, within [0, 1]
            lo = max(Fraction(X * S - bx, dx), Fraction(0))
            hi = min(Fraction((X + 1) * S - bx, dx), Fraction(1))
            if not lo < hi:
                continue
        y0, y1 = by + lo * dy, by + hi * dy
        c, d = min(y0, y1), max(y0, y1)
        if c == d:   # a horizontal ray: y = by, never on a border
            out.add((X, by // S))
            continue
        for Y in range(math.floor(c / S), math.ceil(d / S)):
            out.add((X, Y))
    return out


# ---------------------------------------------------------------------------------------------
# ProbabilityGrid
# ---------------------------------------------------------------------------------------------
def grow_limits(limits, points):
    """Grid2D::GrowLimits (grid_2d.cc:125-164) for each float32 point in turn, on the limits
    (res, max_x, max_y, nx, ny) alone: (limits, (ox, oy)) with the old cells' offset, or None
    where the grid would reach MAX_CELLS."""
    res, max_x, max_y, nx, ny = limits
    ox = oy = 0
    for px, py in points:
        while True:
            ix, iy, _ = cell_index_exact(res, max_x, max_y, px, py)
            if 0 <= ix < nx and 0 <= iy < ny:
                break
            if 2 * nx >= MAX_CELLS or 2 * ny >= MAX_CELLS:
                return None
            xo, yo = nx // 2, ny // 2
            max_x, max_y = max_x + res * yo, max_y + res * xo
            nx, ny, ox, oy = 2 * nx, 2 * ny, ox + xo, oy + yo
    return (res, max_x, max_y, nx, ny), (ox, oy)


def grow_as_needed(limits, origin, returns, misses=(), padding=F(1e-6)):
    """ProbabilityGridRangeDataInserter2D's GrowAsNeeded (:35-50): the float32 bounding box of
    origin, returns and misses, padded by 1e-6 in float32, its two corners grown in turn."""
    pts = np.concatenate([np.asarray(origin, F).reshape(1, -1)[:, :2],
                          np.asarray(returns, F).reshape(-1, 3)[:, :2],
                          np.asarray(misses, F).reshape(-1, 3)[:, :2]])
    lo, hi = pts.min(0), pts.max(0)
    return grow_limits(limits, [(F(lo[0] - padding), F(lo[1] - padding)),
                                (F(hi[0] + padding), F(hi[1] + padding))])


def nonzero_box(cells):
    """(min x, min y, max x, max y) of the non-zero cells, None when all are zero."""
    ys, xs = np.nonzero(cells)
    if len(xs) == 0:
        return None
    return (int(xs.min()), int(ys.min()), int(xs.max()), int(ys.max()))


def _extend(box, xs, ys):
    if len(xs) == 0:
        return box
    lo = (min(xs), min(ys))
    hi = (max(xs), max(ys))
    if box is None:
        return (lo[0], lo[1], hi[0], hi[1])
    return (min(box[0], lo[0]), min(box[1], lo[1]), max(box[2], hi[0]), max(box[3], hi[1]))


def superscaled_ends(limits, origin, points):
    """The superscaled (res / 1000) index of the origin and of each point, and whether every one
    is decided by the exact quotient (an undecided one is the double computation's)."""
    res, max_x, max_y, nx, ny = limits
    sres = res / SUBPIXEL
    def index(p):
        ix, iy, ok = cell_index_exact(sres, max_x, max_y, p[0], p[1])
        return ((ix, iy) if ok else cell_index_double(sres, max_x, max_y, p[0], p[1])), ok
    o, decided = index(origin)
    ends = []
    for p in points:
        e, ok = index(p)
        ends.append(e)
        decided = decided and ok
    return o, ends, decided


def expected_probability_grid(limits, cells, box, origin, returns, misses, tables,
                              free_space=True):
    """One Insert as sets: (limits, cells, known box, decided) after it, or None where the grid
    would grow past the guard.  `cells` [ny, nx] and `box` are the grid before; `tables` (hit,
    miss) come from Inserter.tables().  `decided` is False where some superscaled index sits
    within the double error bound of a tie (the origin on a cell corner, as CreateGrid puts
    it): the double computation then picks that index, and the result is no longer independent
    of it."""
    returns = np.asarray(returns, F).reshape(-1, 3)
    misses = np.zeros((0, 3), F) if misses is None else np.asarray(misses, F).reshape(-1, 3)
    grown = grow_as_needed(limits, origin, returns, misses if free_space else ())
    if grown is None:
        return None
    (res, max_x, max_y, nx, ny), (ox, oy) = grown
    new = np.zeros((ny, nx), np.uint16)
    old_ny, old_nx = cells.shape
    new[oy:oy + old_ny, ox:ox + old_nx] = cells
    if box is not None:
        box = (box[0] + ox, box[1] + oy, box[2] + ox, box[3] + oy)
    L = (res, max_x, max_y, nx, ny)
    pts = np.concatenate([returns, misses]) if free_space else returns
    o, ends, decided = superscaled_ends(L, origin, pts)
    S = SUBPIXEL
    for e in ends:
        assert 0 <= e[0] < nx * S and 0 <= e[1] < ny * S
    hit = {(e[0] // S, e[1] // S) for e in ends[:len(returns)]}
    miss = set()
    if free_space:
        for e in ends:
            miss |= geometric_mask(o, e)
        miss -= hit
    hit_table, miss_table = tables
    for cell_set, table in ((hit, hit_table), (miss, miss_table)):
        if cell_set:
            xs, ys = (np.array(v) for v in zip(*cell_set))
            new[ys, xs] = table[new[ys, xs]] & 0x7fff
    touched = hit | miss
    if free_space and len(pts):
        touched = touched | {(o[0] // S, o[1] // S)}
    if touched:
        xs, ys = zip(*touched)
        box = _extend(box, xs, ys)
    return L, new, box, decided


# ---------------------------------------------------------------------------------------------
# Slots
# ---------------------------------------------------------------------------------------------
def l1_sum(origin, points):
    """Σ |p - o|_1 as the host sums it: each float32 coordinate in double, in input order."""
    o = [float(F(origin[0])), float(F(origin[1]))]
    s = 0.0
    for p in np.asarray(points, F).reshape(-1, 3):
        s += abs(float(p[0]) - o[0]) + abs(float(p[1]) - o[1])
    return s


def slot_reservation(l1, resolution, num_rays):
    """The slots a handle reserves (DESIGN §9): floor(Σ L1 / res (1 + 1e-9)) + 3 rays + 1,
    capped at 2^31 - 1."""
    bound = l1 / resolution * (1.0 + 1e-9) + 3.0 * num_rays + 1.0
    return 2 ** 31 - 1 if bound >= float(2 ** 31 - 1) else int(bound)


def exact_slot_total(origin_cell, end_cells, s=SUBPIXEL):
    """The handle's exact total: Σ count_bound over its rays."""
    return sum(count_bound(origin_cell, e, s) for e in end_cells)


# ---------------------------------------------------------------------------------------------
# TSDF
# ---------------------------------------------------------------------------------------------
def _ulp32(x):
    return float(np.spacing(F(max(abs(x), float(np.finfo(F).tiny)))))


def tsdf_value64(v, lo, hi):
    """RoundToInt((clamp(v) - lo) * resolution) + 1 in float64 with the float32 resolution,
    and the distance of the product from the nearest rounding boundary (x.5)."""
    resolution = float(F(F(VALUE_COUNT - 2) / F(F(hi) - F(lo))))
    c = min(max(v, float(F(lo))), float(F(hi)))
    q = (c - float(F(lo))) * resolution
    return int(math.floor(q + 0.5)) + 1, abs(q - math.floor(q) - 0.5), resolution


def _gaussian64(x, sigma):
    return 1.0 / (math.sqrt(2.0 * math.pi) * sigma) * math.exp(-0.5 * x * x / (sigma * sigma))


def _tsdf_ray64(limits, o32, p, t32, free_space):
    """One return's ray as the host builds it: (range in float64, begin and end superscaled
    cells), or None for a return closer than the truncation."""
    res, max_x, max_y, _, _ = limits
    sres = res / SUBPIXEL
    rx, ry = F(p[0] - o32[0]), F(p[1] - o32[1])
    range32 = F(math.sqrt(float(F(F(rx * rx) + F(ry * ry)))))   # the host's float range
    if range32 < t32:
        return None
    ratio = F(t32 / range32)
    # the mask ends: host float arithmetic as the reference writes it
    bx = o32[0] if free_space else F(o32[0] + F(F(F(1) - ratio) * rx))
    by = o32[1] if free_space else F(o32[1] + F(F(F(1) - ratio) * ry))
    ex = F(o32[0] + F(F(F(1) + ratio) * rx))
    ey = F(o32[1] + F(F(F(1) + ratio) * ry))
    b = cell_index_exact(sres, max_x, max_y, bx, by)
    e = cell_index_exact(sres, max_x, max_y, ex, ey)
    assert b[2] and e[2], "a mask end within the double error bound of a tie"
    return math.hypot(float(rx), float(ry)), b[:2], e[:2]


def tsdf_pair64(limits, origin, rng, X, Y, truncation, w_range, sigma):
    """(update tsd, update weight, error bound) of one (ray, cell) pair in float64."""
    res, max_x, max_y, _, _ = limits
    ox, oy = float(F(origin[0])), float(F(origin[1]))
    t = float(F(truncation))
    cx = max_x - res * (Y + 0.5)
    cy = max_y - res * (X + 0.5)
    ut = min(max(rng - math.hypot(cx - ox, cy - oy), -t), t)
    uw = w_range * (_gaussian64(ut, sigma) if sigma else 1.0)
    err = F32_ERROR_ULPS * _ulp32(max(rng, abs(cx), abs(cy), abs(ox), abs(oy)))
    return ut, uw, err


def tsdf_expected(limits, origin, returns, truncation, max_weight, range_exponent=0, sigma=0.0,
                  free_space=False):
    """TSDFRangeDataInserter2D::Insert into an empty grid whose limits are already grown,
    without normals: {(x, y): (tsd value, weight value, decided)} for every cell some pair
    claims.  A cell's winner is the first ray in input order whose float32 weight is non-zero;
    a cell is undecided where a claim or a quantised value is within the float32 error bound of
    a boundary."""
    o32 = np.asarray(origin, F)
    t32 = F(truncation)
    t = float(t32)
    sigma = float(F(sigma))
    least = 2.0 ** -149   # float32 rounds a weight below half of it to 0
    out = {}
    for p in np.asarray(returns, F).reshape(-1, 3):
        ray = _tsdf_ray64(limits, o32, p, t32, free_space)
        if ray is None:
            continue
        rng, b, e = ray
        w_range = 1.0 / rng ** range_exponent if range_exponent else 1.0
        for cell in geometric_mask(b, e):
            if cell in out and out[cell][3]:
                continue   # an earlier ray's decided claim wins
            ut, uw, err = tsdf_pair64(limits, origin, rng, cell[0], cell[1], t, w_range, sigma)
            claim = True
            value_ok = True
            if sigma:
                w_hi = w_range * _gaussian64(max(abs(ut) - err, 0.0), sigma)
                w_lo = w_range * _gaussian64(min(abs(ut) + err, t), sigma)
                if w_hi < least / 4:
                    continue   # claims nothing, whatever float32 does
                claim = w_lo > least
                # a subnormal ut * uw loses the relative precision the average divides back
                value_ok = w_lo > 2.0 ** -100
            else:
                value_ok = True
            if cell in out:   # after an undecided claim the winner is unknown
                continue
            tv, tdist, tres = tsdf_value64(ut, -t, t)
            wv, wdist, wres = tsdf_value64(min(uw, float(F(max_weight))), 0.0, max_weight)
            # the weight's relative error: its own float32 steps, and the update's error
            # through the distance kernel's slope |ut| / sigma^2
            w_rel = F32_ERROR_ULPS * 2.0 ** -24 * (2 + range_exponent)
            if sigma:
                w_rel += (abs(ut) + err) * err / (sigma * sigma)
            decided = (claim and value_ok and tdist > err * tres and
                       wdist > w_rel * uw * wres)
            out[cell] = (tv, wv, decided, claim)
    return {k: v[:3] for k, v in out.items()}


def round_f32(q):
    """The float32 nearest the exact Fraction q (ties to even): what one rounded float32
    operation gives for the exact result q."""
    x = F(float(q))
    cands = [np.nextafter(x, F(-np.inf)), x, np.nextafter(x, F(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q),
                                     int(np.frombuffer(F(c).tobytes(), np.uint32)[0]) & 1))
    return F(best)


def fmaf(a, b, c):
    """fmaf in exact arithmetic: a * b + c rounded once to float32."""
    return round_f32(Fraction(float(F(a))) * Fraction(float(F(b))) + Fraction(float(F(c))))


def tsdf_conversion(truncation, max_weight):
    """(tsd scale, tsd bias, weight scale, weight bias) of the value -> float decode, in float32
    as TSDValueConverter computes them."""
    def conv(lo, hi):
        scale = F(F(F(hi) - F(lo)) / F(VALUE_COUNT - 2))
        return scale, F(F(lo) - scale)
    ts, tb = conv(-F(truncation), F(truncation))
    ws, wb = conv(F(0), F(max_weight))
    return ts, tb, ws, wb


FUSIONS = ("first", "second")   # which product of tsd * w + ut * uw a multiply-add takes


def tsdf_update32(tv, wv, ut, uw, truncation, max_weight, fused=None):
    """UpdateCell of one cell whose values are (tv, wv), both non-zero, with the update
    (ut, uw), as float32 operations; the (tsd value, weight value) it stores, with lround.
    `fused` (one of FUSIONS) contracts as a multiply-add would: both decodes become fmaf, and so
    does the sum tsd * w + ut * uw with its first product (fmaf(tsd, w, ut * uw)) or its second
    (fmaf(ut, uw, tsd * w)); nvcc emits the second for sm_90a."""
    ts, tb, ws, wb = tsdf_conversion(truncation, max_weight)
    ut, uw = F(ut), F(uw)
    if fused:
        assert fused in FUSIONS
        tsd = fmaf(tv, ts, tb)
        w = fmaf(wv, ws, wb)
        num = fmaf(tsd, w, F(ut * uw)) if fused == "first" else fmaf(ut, uw, F(tsd * w))
    else:
        tsd = F(F(F(tv) * ts) + tb)
        w = F(F(F(wv) * ws) + wb)
        num = F(F(tsd * w) + F(ut * uw))
    uwt = F(w + uw)
    sdf = F(num / uwt)
    uwt = min(F(max_weight), uwt)

    def value(v, lo, hi):
        lo, hi = F(lo), F(hi)
        c = min(max(v, lo), hi)
        res = F(F(VALUE_COUNT - 2) / F(hi - lo))
        q = F(F(c - lo) * res)
        return int(math.floor(float(q) + 0.5)) + 1
    return value(sdf, -F(truncation), F(truncation)), value(uwt, 0, max_weight)


# ---------------------------------------------------------------------------------------------
# Launch shapes and grids
# ---------------------------------------------------------------------------------------------
LANE_PATTERNS = ("lane0", "lane31", "partial_warp_last", "last_block")


def extreme_index(pattern, n):
    """The index of the one point that decides the touched box under a pattern: lane 0 of the
    last warp, lane 31 of the last full warp, the last lane of a partial last warp (the last
    point), or the first point of the last 256-thread block."""
    if pattern == "lane0":
        return ((n - 1) // 32) * 32
    if pattern == "lane31":
        full = n // 32
        return (full - 1) * 32 + 31 if full else n - 1
    if pattern == "last_block":
        return ((n - 1) // 256) * 256
    return n - 1


def grid_with_flat_count(target, ny):
    """(nx, ny) of a grid with ny rows whose pitch * ny is `target`: nx is a multiple of 8, so
    that the pitch (nx rounded up to 8 cells) is nx itself."""
    nx = target // ny
    assert nx * ny == target and nx % 8 == 0
    return nx, ny
