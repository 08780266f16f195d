"""The 2D map-writing references of tests/map_writing2d_refs.py against brute force and the
restatements, on the CPU: the geometric ray mask against RayToPixelMask's integer walk, the
exact cell index against the restatement's, the set-based grid state against
Inserter.insert, the float64 TSDF cells against TsdfInserter.insert, the slot reservation
against exact totals and against the product's SlotReservation, and the two contraction
orders of the TSDF average."""
import math
from fractions import Fraction

import numpy as np
import pytest

from tests import insert2d_oracle as O
from tests import insert_tsdf2d_oracle as T
from tests import map_writing2d_refs as R

F = np.float32
S = R.SUBPIXEL


def _walk(b, e):
    m = O.ray_to_pixel_mask(b, e, S)
    assert len(m) == len(set(m)), "the walk emits a pixel twice"
    return set(m)


def _brute_mask(b, e):
    """Every pixel of the bounding box whose open square the segment meets, by solving for the
    segment's parameter on each axis exactly."""
    (bx, by), (ex, ey) = [(Fraction(2 * v[0] + 1, 2), Fraction(2 * v[1] + 1, 2)) for v in (b, e)]
    out = set()
    for X in range(min(b[0], e[0]) // S, max(b[0], e[0]) // S + 1):
        for Y in range(min(b[1], e[1]) // S, max(b[1], e[1]) // S + 1):
            lo, hi = Fraction(0), Fraction(1)
            lo_open = hi_open = False
            ok = True
            for p0, d, a in ((bx, ex - bx, X * S), (by, ey - by, Y * S)):
                if d == 0:
                    ok = ok and a < p0 < a + S
                    continue
                t0, t1 = sorted(((a - p0) / d, (a + S - p0) / d))
                if t0 >= lo:
                    lo, lo_open = t0, True
                if t1 <= hi:
                    hi, hi_open = t1, True
            if ok and (lo < hi or (lo == hi and not lo_open and not hi_open)):
                out.add((X, Y))
    return out


def _random_rays(rng, k, span):
    b = rng.randint(0, span, size=(k, 2))
    e = np.clip(b + rng.randint(-6 * S, 6 * S + 1, size=(k, 2)), 0, None)
    return [(tuple(int(v) for v in p), tuple(int(v) for v in q)) for p, q in zip(b, e)]


def _special_rays():
    rays = []
    for b in ((500, 500), (0, 0), (999, 999), (1000, 1000), (1499, 2501), (2000, 999)):
        for d in ((3000, 3000), (3000, -3000) if b[1] >= 3000 else (3000, 0), (0, 4000),
                  (4000, 0), (0, 0), (2000, 1000), (-999, 1998) if b[0] >= 999 else (999, 1998),
                  (1, 0), (0, 1), (1, 1)):
            e = (b[0] + d[0], b[1] + d[1])
            if min(e) >= 0:
                rays.append((b, e))
    # exact corner crossings: through (k s, l s) in subpixel units from b + 1/2
    for k in range(1, 4):
        rays.append(((499, 499), (499 + 2 * k * S, 499 + 2 * k * S)))
        rays.append(((499, 3 * S + 499), (499 + 2 * k * S, 3 * S + 499 - k * S)))
        rays.append(((S - 1, 2 * S - 1), (S - 1 + k * S, 2 * S - 1 + 2 * k * S)))
    # +-1/2 subpixel neighbours of borders: ends at k s - 1 and k s (centres k s -+ 1/2)
    for a in (S - 1, S, 2 * S - 1, 2 * S):
        for c in (S - 1, S, 3 * S - 1, 3 * S):
            rays.append(((a, 5), (c, 3 * S + 7)))
            rays.append(((5, a), (3 * S + 7, c)))
            rays.append(((a, c), (a + 2 * S, c + S)))
    return rays


def test_geometric_mask_equals_brute_force_and_the_walk_on_special_rays():
    for b, e in _special_rays():
        g = R.geometric_mask(b, e)
        assert g == _brute_mask(b, e), (b, e)
        assert g == _walk(b, e), (b, e)
        assert len(g) <= R.count_bound(b, e)
        assert (b[0] // S, b[1] // S) in g and (e[0] // S, e[1] // S) in g


def test_geometric_mask_equals_the_walk_on_random_rays():
    rng = np.random.RandomState(1)
    for b, e in _random_rays(rng, 3000, 20 * S):
        g = R.geometric_mask(b, e)
        assert g == _walk(b, e), (b, e)
        assert len(g) <= R.count_bound(b, e)
    for b, e in _random_rays(rng, 200, 20 * S):
        assert R.geometric_mask(b, e) == _brute_mask(b, e), (b, e)


def test_corner_rays_fill_three_pixels_of_their_bound():
    """A ray of L1 much smaller than a cell across a pixel corner: 3 pixels, the bound exactly."""
    for b, e in (((999, 999), (1000, 1000)), ((999, 1000), (1000, 999)), ((998, 999), (1001, 1000)),
                 ((1000, 999), (999, 1000))):
        g = R.geometric_mask(b, e)
        assert g == _walk(b, e)
    assert R.geometric_mask((998, 999), (1001, 1001)) == {(0, 0), (0, 1), (1, 1)}
    assert R.count_bound((998, 999), (1001, 1001)) == 3
    # through the corner exactly: two pixels, the diagonal step
    assert R.geometric_mask((999, 999), (1000, 1000)) == {(0, 0), (1, 1)}


def test_cell_index_exact_matches_the_restatement_where_decided():
    rng = np.random.RandomState(2)
    undecided = 0
    for res in (0.05, 1.0, 0.1, float(F(0.05)), 0.025):
        for sres in (res, res / S):
            g = O.Grid(sres, 3.7 + 600 * rng.rand(), -2.1 - 600 * rng.rand(), 10, 10)
            _, max_x, max_y, _, _ = g.limits
            pts = np.concatenate([
                np.column_stack([max_x - rng.rand(300) * 40, max_y - rng.rand(300) * 40]),
                # cell borders and centres in float32, and their ulp neighbours
                np.column_stack([max_x - sres * np.arange(60) / 2,
                                 max_y - sres * np.arange(60) / 2])])
            pts = pts.astype(F)
            pts = np.concatenate([pts, np.nextafter(pts, F(np.inf)), np.nextafter(pts, F(-np.inf))])
            for px, py in pts:
                ix, iy, ok = R.cell_index_exact(sres, max_x, max_y, px, py)
                if not ok:
                    undecided += 1
                    continue
                assert g.cell_index(px, py) == (ix, iy)
    assert undecided < 200


def test_cell_index_exact_flags_exact_ties():
    # (max - p) / res - 0.5 exactly an integer + 1/2: the double computation decides the cell
    ix, iy, ok = R.cell_index_exact(1.0, 5.0, 5.0, F(3.0), F(3.0))
    assert (ix, iy) == (2, 2) and not ok
    ix, iy, ok = R.cell_index_exact(1.0, 5.0, 5.0, F(3.25), F(2.75))
    assert (ix, iy) == (2, 1) and ok


def _seeded_scan(rng, origin, n, m, spread):
    ret = np.column_stack([origin[0] + rng.uniform(-spread, spread, n),
                           origin[1] + rng.uniform(-spread, spread, n), np.zeros(n)]).astype(F)
    mis = np.column_stack([origin[0] + rng.uniform(-spread, spread, m),
                           origin[1] + rng.uniform(-spread, spread, m), np.zeros(m)]).astype(F)
    return ret, mis


@pytest.mark.parametrize("free_space", [True, False])
def test_set_based_grid_equals_the_restatement_on_seeded_scans(free_space):
    rng = np.random.RandomState(3)
    ins = O.Inserter(0.55, 0.49, free_space)
    tables = ins.tables()
    g = O.Grid.create_grid([0.3, -0.2], 0.05)
    limits, cells, box = g.limits, g.cells, g.known_box
    for k in range(6):
        # off the cell corners, so that every index is decided by the exact quotient
        origin = np.float32([0.3 + 0.1 * k + 0.0137, -0.2 + 0.05 * k + 0.0211, 0])
        ret, mis = _seeded_scan(rng, origin, 60, 20, 2.0 + 1.5 * k)   # grows on later scans
        want = R.expected_probability_grid(limits, cells, box, origin, ret, mis, tables,
                                           free_space)
        ins.insert(origin, ret, g, mis)
        limits, cells, box, decided = want
        assert decided
        assert g.limits == limits
        np.testing.assert_array_equal(g.cells, cells)
        assert g.known_box == box


def test_set_based_grid_on_a_grid_made_from_cells_and_refusals():
    rng = np.random.RandomState(4)
    ins = O.Inserter(0.6, 0.4, True)
    cells = np.zeros((37, 45), np.uint16)
    cells[5:9, 30:33] = rng.randint(1, 32768, size=(4, 3))
    g = O.Grid(0.05, 1.0, 2.0, 45, 37, cells)
    origin = np.float32([0.1, 1.1, 0])
    ret, mis = _seeded_scan(rng, origin, 40, 10, 0.8)
    want = R.expected_probability_grid(g.limits, g.cells, R.nonzero_box(cells), origin, ret, mis,
                                       ins.tables())
    ins.insert(origin, ret, g, mis)
    assert g.limits == want[0] and g.known_box == want[2] and want[3]
    np.testing.assert_array_equal(g.cells, want[1])
    # the guard: 100 cells double to 25 600 and no further
    lim = (0.05, 2.5, 2.5, 100, 100)
    assert R.grow_limits(lim, [(F(2.5 - 0.05 * 12799), F(0.0))])[0][3] == 25600
    assert R.grow_limits(lim, [(F(2.5 - 0.05 * 25599 - 200.0), F(0.0))]) is None


def test_tsdf_float64_cells_equal_the_restatement_where_decided():
    from cartographer_b200.scan_matching import TSDFRangeDataInserterOptions2D as Opts
    rng = np.random.RandomState(5)
    checked = 0
    for exponent, sigma, free_space in ((0, 0.0, False), (1, 0.0, True), (2, 0.1, False),
                                        (0, 0.02, False)):
        opts = Opts(truncation_distance=0.3, maximum_weight=10.0, update_free_space=free_space,
                    project_sdf_distance_to_scan_normal=False, update_weight_range_exponent=exponent,
                    update_weight_angle_scan_normal_to_ray_kernel_bandwidth=0.0,
                    update_weight_distance_cell_to_hit_kernel_bandwidth=sigma)
        g = T.TsdfGrid.create_grid([0.2, 0.1], 0.05, 0.3, 10.0)
        origin = np.float32([0.2137, 0.1211, 0])
        a = rng.uniform(0, 2 * math.pi, 80)
        r = rng.uniform(0.2, 2.2, 80)
        ret = np.column_stack([origin[0] + r * np.cos(a), origin[1] + r * np.sin(a),
                               np.zeros(80)]).astype(F)
        want = R.tsdf_expected(g.limits, origin, ret, 0.3, 10.0, exponent, sigma, free_space)
        assert T.TsdfInserter(opts).insert(origin, ret, g)
        tsd, weight = g.arrays()
        claimed = {(x, y) for y, x in zip(*np.nonzero(weight))}
        for (x, y), (tv, wv, ok) in want.items():
            if ok:
                assert (int(tsd[y, x]), int(weight[y, x])) == (tv, wv), (x, y)
                checked += 1
        decided_cells = {c for c, v in want.items() if v[2]}
        assert decided_cells <= claimed
        assert claimed <= set(want)
    assert checked > 2000


def test_tsdf_update_fused_model():
    """fmaf rounds once; the unfused model rounds the product first."""
    a, b, c = F(1 + 2 ** -12), F(1 + 2 ** -12), F(-1)
    assert R.fmaf(a, b, c) == F(2 ** -11 + 2 ** -24)
    assert F(F(a * b) + c) == F(2 ** -11)
    assert R.round_f32(Fraction(1, 3)) == F(1 / 3)
    assert R.round_f32(Fraction(1) + Fraction(1, 2 ** 24)) == F(1)   # tie to even
    # the two contraction orders of tsd * w + ut * uw are different models: with ut * uw
    # inexact, some cells store different values under them
    rng = np.random.RandomState(12)
    differ = 0
    for _ in range(3000):
        tv, wv = (int(v) for v in rng.randint(1, 32768, 2))
        ut, uw = F(rng.uniform(-0.3, 0.3)), F(rng.uniform(0.01, 3.0))
        first, second = (R.tsdf_update32(tv, wv, ut, uw, 0.3, 10.0, f) for f in R.FUSIONS)
        differ += first != second
    assert differ > 0


def test_slot_reservation_equals_the_product_function():
    """The Python copy against csm::SlotReservation in the product library, called through its
    exported C++ symbol, on lengths around the rounding of the 1e-9 margin and the 2^31 - 1
    cap."""
    import ctypes as C
    from cartographer_b200 import _lib
    fn = _lib.lib()._ZN3csm15SlotReservationEddi
    fn.restype = C.c_longlong
    fn.argtypes = [C.c_double, C.c_double, C.c_int]
    rng = np.random.RandomState(13)
    cases = [(0.0, 0.05, 1), (1e12, 0.05, 3), (0.05 * (2 ** 31 - 4), 0.05, 1),
             (0.05 * (2 ** 31 - 5), 0.05, 1), (3.0, float(F(0.05)), 65537)]
    cases += [(float(l1), float(res), int(n)) for l1, res, n in
              zip(rng.uniform(0, 1e6, 300), rng.choice([0.05, float(F(0.05)), 0.025, 1.0], 300),
                  rng.randint(1, 1 << 20, 300))]
    # exact multiples of the resolution, where the 1e-9 margin decides the floor
    cases += [(k * 0.05, 0.05, 7) for k in (1, 3, 10, 12345, 10 ** 6)]
    for l1, res, n in cases:
        assert R.slot_reservation(l1, res, n) == fn(l1, res, n), (l1, res, n)


def test_slot_reservation_bounds_brute_force_totals():
    rng = np.random.RandomState(6)
    for res in (0.05, 1.0, float(F(0.05)), 0.025):
        g = O.Grid(res, 10.0 + 600 * rng.rand(), -5.0 + 600 * rng.rand(), 400, 400)
        lim = g.limits
        _, max_x, max_y, _, _ = lim
        centre = (max_x - 200 * res, max_y - 200 * res)
        for trial in range(20):
            n = rng.randint(1, 200)
            origin = np.float32([centre[0] + rng.uniform(-1, 1) * res,
                                 centre[1] + rng.uniform(-1, 1) * res, 0])
            if trial % 2:   # near pixel corners, far shorter than a cell
                k = rng.randint(-100, 100, size=(n, 2))
                pts = np.column_stack([max_x - (k[:, 0] + 100) * res + rng.uniform(-1e-4, 1e-4, n),
                                       max_y - (k[:, 1] + 100) * res + rng.uniform(-1e-4, 1e-4, n),
                                       np.zeros(n)]).astype(F)
                origin = pts[0].copy()
                pts[:, :2] = origin[:2] + rng.uniform(-res / 40, res / 40, (n, 2)).astype(F)
            else:
                pts = np.column_stack([centre[0] + rng.uniform(-8, 8, n),
                                       centre[1] + rng.uniform(-8, 8, n), np.zeros(n)]).astype(F)
            o, ends, _ = R.superscaled_ends(lim, origin, pts)
            total = R.exact_slot_total(o, ends)
            cap = R.slot_reservation(R.l1_sum(origin, pts), res, n)
            assert total <= cap
            # the brute-force total is the walk's pixel count bound, ray by ray
            for e in ends[:5]:
                assert len(_walk(o, e)) <= R.count_bound(o, e)
    assert R.slot_reservation(1e12, 0.05, 3) == 2 ** 31 - 1


def test_keep_patterns_and_flat_grids():
    assert R.extreme_index("lane0", 257) == 256
    assert R.extreme_index("lane31", 257) == 255
    assert R.extreme_index("lane31", 31) == 30
    assert R.extreme_index("last_block", 65537) == 65536
    assert R.extreme_index("last_block", 4097) == 4096
    assert R.extreme_index("last_block", 255) == 0
    assert R.extreme_index("partial_warp_last", 33) == 32
    for target in (1 << 14, (1 << 14) - 8, (1 << 14) + 8):
        nx, ny = R.grid_with_flat_count(target, {1 << 14: 128, (1 << 14) - 8: 23,
                                                 (1 << 14) + 8: 683}[target])
        assert nx * ny == target and nx % 8 == 0
