"""Scans whose consecutive points share cells, against exact sums.

For the tile form of the lowest-resolution pass, the 2D matcher also stores each discrete
scan as entries: a run of equal consecutive cells, cut every kMaxWeight (4) points, weighted
by its length.  The tile pass sums weight x value and flushes its packed u16 sums by weight,
so the cases below put runs across its 32-entry staging and its four-at-once path, with
cells of value 255 (the largest weight per flush).  Clouds repeat a point's exact
coordinates, so a run keeps its cell under every rotation.  Each case compares with the
oracle, which sums point by point: the lowest-resolution sums of every form
(csm_score_top2d), one branch step of every form at the top level and at h = 1
(csm_branch_step2d), the per-point discrete scans (csm_discretize2d) and caller-given scans
(csm_score_candidates2d), which keep reading points.
"""
import numpy as np
import pytest

from benchmarks import synthetic
from tests.test_gpu_branch_step_2d import World, _tight_bound, check_step
from tests.test_gpu_top_pass_2d import RES, centred, check_top

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def runs_cloud(rng, n, counts, radius_cells, far_every=0):
    """n points: random points, each repeated by the next entry of `counts` (cyclic); with
    far_every, every far_every-th run lies off the map, 10-15 m from the sensor (beyond
    the window tables of the maps below, while the search stays small)."""
    pts, i = [], 0
    while sum(len(p) for p in pts) < n:
        c = counts[i % len(counts)]
        xy = rng.uniform(-radius_cells, radius_cells, 2) * RES
        if far_every and i % far_every == far_every - 1:
            xy = rng.uniform(-1.0, 1.0, 2) * 2.0 + np.array([10.0, -7.0])
        pts.append(np.tile(np.array([xy[0], xy[1], 0.0]), (c, 1)))
        i += 1
    return np.concatenate(pts)[:n].astype(np.float32)


CLOUDS = {
    # runs far longer than the weight cap: 271 entries, 270 of weight 4
    "identical": lambda rng: np.tile(runs_cloud(rng, 1, [1], 3), (1081, 1)),
    # run lengths that put run ends on every residue of the tile pass's 32-entry staging
    "straddle": lambda rng: runs_cloud(rng, 1081, [3, 5, 7, 30, 33, 2, 1, 9, 64, 129], 6),
    "alternating": lambda rng: runs_cloud(rng, 1081, [1, 2, 1, 6, 1, 4, 1, 5], 6),
    "far_runs": lambda rng: runs_cloud(rng, 1081, [4, 1, 9, 3, 17], 6, far_every=3),
    "one_point": lambda rng: runs_cloud(rng, 1, [1], 3),
}


def _saturated(ny, nx):
    return np.ones((ny, nx), np.uint16)   # every cell at the highest probability: 255


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_top_pass_every_form(oracle, sm, name):
    xyz = CLOUDS[name](np.random.RandomState(len(name)))
    grid = centred(_saturated(150, 140))
    check_top(oracle, sm, grid, 4, xyz, lin=1.0, ang=0.2)
    check_top(oracle, sm, grid, 3, xyz, full=True)
    rng = np.random.RandomState(3)
    cells = rng.randint(1, 32768, size=(120, 110)).astype(np.uint16)
    check_top(oracle, sm, centred(cells), 4, xyz, full=True)


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_branch_step_every_form(oracle, sm, name):
    xyz = CLOUDS[name](np.random.RandomState(len(name)))
    for cells in (_saturated(90, 90),
                  np.random.RandomState(8).randint(1, 32768, size=(70, 80)).astype(np.uint16)):
        w = World(oracle, sm, cells, 4, xyz, lin=0.6, ang=0.1)
        try:
            for h in (3, 1):
                last = w.ds.shape[0] - 1
                par = w.parents(w.lattice(0, h)[:9] + w.lattice(last, h)[:33], h)
                check_step(w, par, h, np.float32(0.1), 0.1)
                check_step(w, par, h, _tight_bound(w, par, h), 0.1)
                # one live parent among dead ones: G = 32 lanes share its points
                p1 = par.copy()
                top = _tight_bound(w, par, h)
                p1["score"][1:] = np.nextafter(top, np.float32(-1))
                p1["score"][0] = max(p1["score"][0], top)
                check_step(w, p1, h, top, 0.1)
        finally:
            w.close()


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_discretize_per_point(oracle, sm, name):
    xyz = CLOUDS[name](np.random.RandomState(len(name)))
    grid = centred(np.random.RandomState(4).randint(1, 32768, size=(60, 70)).astype(np.uint16))
    m = sm.FastCorrelativeScanMatcher2D(grid, sm.FastCorrelativeScanMatcherOptions2D(1.0, 0.3, 4))
    try:
        og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
        fe = oracle.frontend2d(og, xyz, (0.0, 0.0, 0.0), lin=1.0, ang=0.3)
        ds, bounds = m.discretize(xyz, (0.0, 0.0, 0.0))
        np.testing.assert_array_equal(ds, fe["discrete_scans"])
        np.testing.assert_array_equal(bounds, fe["bounds"])
    finally:
        m.close()


def test_caller_scans_with_runs_beyond_the_clamp(oracle, sm):
    """Caller-given scans with runs of equal cells, runs off the map and runs of different
    cells beyond +-30000 that the engine clamps to one cell."""
    grid = centred(_saturated(40, 50))
    runs = [((3, 4), 7), ((40000, 2), 5), ((35000, 2), 3), ((-1, 5), 2), ((10, 10), 1),
            ((-31000, -45000), 9), ((-30500, -30001), 4), ((20, 30), 6), ((200, 7), 3)]
    scan = np.concatenate([np.tile(np.array(c, np.int32), (k, 1)) for c, k in runs])
    ds = np.stack([scan, scan[::-1].copy()])
    og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
    om = oracle.FastCorrelativeScanMatcher2D(og, 1.0, 0.3, 3)
    m = sm.FastCorrelativeScanMatcher2D(grid, sm.FastCorrelativeScanMatcherOptions2D(1.0, 0.3, 3))
    try:
        cand = np.array([(s, x, y) for s in (0, 1) for x in range(-12, 13, 3)
                         for y in range(-9, 10, 3)], np.int32)
        for level in (0, 2):
            want_scores, want_sums = om.score_candidates(level, ds, cand)
            got_scores, got_sums = m.score_candidates(level, ds, cand)
            np.testing.assert_array_equal(got_sums, want_sums)
            np.testing.assert_array_equal(got_scores.view(np.uint32), want_scores.view(np.uint32))
    finally:
        m.close()
