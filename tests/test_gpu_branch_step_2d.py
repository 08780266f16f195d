"""One branch step of the 2D fast matcher (csm_branch_step2d) against exact child sums.

The hook runs the batch's own level step (k_level_begin, the counting sort and either
k_expand, one warp per parent, or k_expand_lattice<4|8|16>) over parents the test
chooses, with the job's bound set first.  The reference is the oracle's ScoreCandidates
at level h - 1 (integer sums, float score bits) on the oracle's discrete scans:
  * a parent is live iff score >= B; a child is valid unless it lies past max_x / max_y;
  * at h >= 2 a valid child of a live parent is pushed iff score > min_score and
    score >= B, with the oracle's score bits; counters = (valid children of live
    parents, live parents) and the bound stays at B;
  * at h == 1 leaves raise the bound during the step: every recorded leaf carries its
    exact score, the final bound is max(B, best child score > min_score), every child
    at that maximum is recorded, and the counters lie between their values at the
    final bound and at B.
Outputs are compared as sorted multisets (atomics order them across warps); a lattice
work item of <= 32 parents of one scan runs in one warp, whose order is checked exactly:
row 2*j0 then row 2*j0+1, parents in queue order, x ascending within a parent.
The cases aim at the early exit (t_min - p_hi), the lane re-map (ballot, k-th leader,
shuffled sums, mx, p_hi, positions and x2/y2 flags) and the packed u16 accumulators.
"""
import numpy as np
import pytest

from benchmarks import synthetic

pytestmark = pytest.mark.gpu

RES = 0.05
FORMS = [("warp", 8), ("lattice", 4), ("lattice", 8), ("lattice", 16)]


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


class World:
    """A stack, a cloud and a local-window search, on the device and in the oracle."""

    def __init__(self, oracle, sm, grid, depth, cloud, lin=2.0, ang=0.3, pose=None):
        if isinstance(grid, np.ndarray):  # cells of a map centred on the world origin
            ny, nx = grid.shape
            grid = synthetic.GridSpec(grid, RES, 0.5 * ny * RES, 0.5 * nx * RES)
        self.grid = grid
        self.pose = np.zeros(3) if pose is None else np.asarray(pose, np.float64)
        self.cloud = np.ascontiguousarray(cloud, np.float32)
        self.lin, self.ang, self.depth = lin, ang, depth
        self.m = sm.FastCorrelativeScanMatcher2D(
            self.grid, sm.FastCorrelativeScanMatcherOptions2D(lin, ang, depth))
        og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
        self.om = oracle.FastCorrelativeScanMatcher2D(og, lin, ang, depth)
        fe = oracle.frontend2d(og, self.cloud, self.pose, lin=lin, ang=ang)
        self.ds, self.bounds = fe["discrete_scans"], fe["bounds"]
        self.sm = sm

    def close(self):
        self.m.close()

    def lattice(self, scan, h):
        """Every node of `scan`'s level-h lattice, x outer, y inner."""
        mnx, mxx, mny, mxy = self.bounds[scan]
        return [(scan, x, y) for x in range(mnx, mxx + 1, 1 << h)
                for y in range(mny, mxy + 1, 1 << h)]

    def scores(self, level, cand):
        cand = np.asarray(cand, np.int32).reshape(-1, 3)
        if not len(cand):
            return np.zeros(0, np.float32)
        return self.om.score_candidates(level, self.ds, cand)[0]

    def parents(self, nodes, h, loose=False):
        """Parents with their exact level-h score (or the top score, a looser p_hi)."""
        out = np.zeros(len(nodes), self.sm.NODE2D_DTYPE)
        if len(nodes):
            out["scan"], out["xo"], out["yo"] = np.asarray(nodes, np.int32).T
            out["score"] = np.float32(0.9) if loose else self.scores(h, nodes)
        return out


def _key(rows):
    return sorted((int(r["scan"]), int(r["xo"]), int(r["yo"]), int(np.float32(r["score"]).view(np.uint32)))
                  for r in rows)


def _children(w, parents, h, live):
    half = 1 << (h - 1)
    cand = []
    for p in parents[live]:
        for t in range(4):
            x, y = int(p["xo"]) + (t >> 1) * half, int(p["yo"]) + (t & 1) * half
            if x <= w.bounds[p["scan"], 1] and y <= w.bounds[p["scan"], 3]:
                cand.append((int(p["scan"]), x, y))
    return cand


def check_step(w, parents, h, B, min_score, forms=FORMS):
    """Runs every form on one case and compares with the exact reference.  Returns the
    reference children and scores (for the threshold cases)."""
    B, min_score = np.float32(B), np.float32(min_score)
    live = parents["score"] >= B
    cand = _children(w, parents, h, live)
    sc = w.scores(h - 1, cand)
    one_warp = len(parents) <= 32 and len(set(parents["scan"].tolist())) == 1
    for form, unroll in forms:
        tag = "%s/%d h=%d" % (form, unroll, h)
        got, final, ctr = w.m.branch_step(w.cloud, w.pose, False, min_score, h, parents, B, form,
                                          unroll)
        if h >= 2:
            kept = (sc > min_score) & (sc >= B)
            want = [(c[0], c[1], c[2], s) for c, s in zip(cand, sc) if s > min_score and s >= B]
            want_rows = np.array(want, w.sm.NODE2D_DTYPE) if want else np.zeros(0, w.sm.NODE2D_DTYPE)
            assert _key(got) == _key(want_rows), tag
            assert ctr == (len(cand), int(live.sum())), tag
            assert final == B, tag
            if form == "lattice" and one_warp:
                # documented push order of one warp
                half = 1 << (h - 1)
                by = {(c[1], c[2]): s for c, s, k in zip(cand, sc, kept) if k}
                order = []
                for iy in (0, 1):
                    for p in parents[live]:
                        for ix in (0, 1):
                            xy = (int(p["xo"]) + ix * half, int(p["yo"]) + iy * half)
                            if xy in by:
                                order.append(xy)
                assert [(int(r["xo"]), int(r["yo"])) for r in got] == order, tag
        else:
            ok = sc > min_score
            best = max(B, sc[ok].max()) if ok.any() else B
            assert final == best, tag
            exact = {c: s for c, s in zip(cand, sc)}
            seen = set()
            for r in got:
                c = (int(r["scan"]), int(r["xo"]), int(r["yo"]))
                assert c in exact and c not in seen, tag
                seen.add(c)
                assert np.float32(r["score"]).view(np.uint32) == exact[c].view(np.uint32), tag
                assert r["score"] > min_score and r["score"] >= B, tag
            for c, s in exact.items():
                if s > min_score and s == best:
                    assert c in seen, (tag, c)
            live_f = parents["score"] >= best
            lo = (len(_children(w, parents, h, live_f)), int(live_f.sum()))
            hi = (len(cand), int(live.sum()))
            assert lo[0] <= ctr[0] <= hi[0] and lo[1] <= ctr[1] <= hi[1], (tag, ctr, lo, hi)
    return cand, sc


def _random_cells(rng, ny, nx, zero=0.3):
    cells = rng.randint(1, 32768, size=(ny, nx)).astype(np.uint16)
    cells[rng.uniform(size=cells.shape) < zero] = 0
    return cells


def _cloud(rng, n, radius_cells, far=0):
    """n points in a square of +-radius cells around the sensor, the last `far` of them
    hundreds of metres away (outside the map and the window table)."""
    xy = rng.uniform(-radius_cells, radius_cells, (n, 2)) * RES
    if far:
        xy[-far:] = rng.uniform(-1.0, 1.0, (far, 2)) * 300.0 + np.array([600.0, -450.0])
    return np.concatenate([xy, np.zeros((n, 1))], axis=1).astype(np.float32)


def _tight_bound(w, parents, h):
    """B at the best valid child of all parents (most parents are then ruled out early)."""
    cand = _children(w, parents, h, np.ones(len(parents), bool))
    return w.scores(h - 1, cand).max()


@pytest.fixture(scope="module")
def small_world(oracle, sm):
    rng = np.random.RandomState(11)
    w = World(oracle, sm, _random_cells(rng, 96, 80), 5, _cloud(rng, 1081, 30), lin=2.0, ang=0.3)
    yield w
    w.close()


@pytest.mark.parametrize("count", [1, 2, 3, 5, 9, 17, 31, 32, 33, 65])
def test_parents_per_scan(small_world, count):
    """Every starting G (32 / count rounded down to a power of two) and full and partial
    work items; one scan and two scans at once, at a loose and at a tight bound."""
    w = small_world
    rng = np.random.RandomState(count)
    for h in (1, 2, 4):
        for scans in ((0,), (1, w.ds.shape[0] - 1)):
            nodes = []
            for k in scans:
                lat = w.lattice(k, h)
                idx = np.sort(rng.choice(len(lat), min(count, len(lat)), replace=False))
                nodes += [lat[i] for i in idx]
            par = w.parents(nodes, h)
            check_step(w, par, h, np.float32(0.1), 0.1)
            check_step(w, par, h, _tight_bound(w, par, h), 0.1)


@pytest.mark.parametrize("pattern", ["lanes_0_5_17", "one_of_32", "quarter_of_9",
                                     "two_of_33", "edge_live"])
def test_remap_patterns(small_world, pattern):
    """Live parents that are not contiguous in the warp, exactly one live parent (G = 32),
    G growing fourfold in one re-map, and live parents on max_x / max_y (x2 or y2 false)
    among interior dead ones, so that the flags travel with the re-map."""
    w = small_world
    h = 2
    k = 3
    lat = w.lattice(k, h)
    mnx, mxx, mny, mxy = w.bounds[k]
    half = 1 << (h - 1)
    if pattern == "edge_live":
        edge = [c for c in lat if c[1] + half > mxx or c[2] + half > mxy]
        inner = [c for c in lat if not (c[1] + half > mxx or c[2] + half > mxy)]
        nodes = inner[:24] + edge[:8]
        nodes = [nodes[i] for i in np.random.RandomState(0).permutation(len(nodes))]
        live = np.array([(c in edge) for c in nodes])
        assert live.sum() >= 4
    else:
        n, on = {"lanes_0_5_17": (32, [0, 5, 17]), "one_of_32": (32, [13]),
                 "quarter_of_9": (9, [1, 4, 6, 8]), "two_of_33": (33, [0, 32])}[pattern]
        nodes = lat[:n]
        live = np.zeros(n, bool)
        live[on] = True
    par = w.parents(nodes, h)
    lo = np.float32(0.11)
    # dead parents score just below B; the live ones keep their exact score (>= B)
    B = min(lo, par["score"][live].min())
    par["score"][~live] = np.nextafter(B, np.float32(-1))
    check_step(w, par, h, B, 0.1)
    # again at the best child's score: the live parents are ruled out early one by one
    Bt =_tight_bound(w, par[live], h)
    par2 = par.copy()
    par2["score"][~live] = np.nextafter(Bt, np.float32(-1))
    par2["score"][live] = np.maximum(par2["score"][live], Bt)
    check_step(w, par2, h, Bt, 0.1)


@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 255, 256, 257, 1081])
def test_point_counts(oracle, sm, n):
    """Point counts around the 128-point early-exit tests and the chunk staging."""
    rng = np.random.RandomState(1000 + n)
    w = World(oracle, sm, _random_cells(rng, 64, 72, zero=0.1), 4, _cloud(rng, n, 20),
              lin=1.0, ang=0.2)
    try:
        for h in (3, 2, 1):
            for k in (0, w.ds.shape[0] // 2):
                lat = w.lattice(k, h)
                par = w.parents(lat[:40], h)
                check_step(w, par, h, np.float32(0.1), 0.1)
                check_step(w, par, h, _tight_bound(w, par, h), 0.1)
    finally:
        w.close()


def test_bound_and_min_score_at_exact_thresholds(small_world):
    """B = ToScore(s) keeps a child of exact sum s, nextafter(B, +inf) drops it; min_score
    is strict: min_score = ToScore(s) drops it, nextafter(.., -inf) keeps it."""
    w = small_world
    lo = np.float32(0.05)  # below every score (an empty child scores min_score = 0.1)

    def pushed(min_score, B, h, par):
        got, final, _ = w.m.branch_step(w.cloud, w.pose, False, min_score, h, par, B, "lattice")
        return {(int(r["xo"]), int(r["yo"])) for r in got}, final

    for h in (3, 2, 1):
        lat = w.lattice(2, h)
        par = w.parents(lat[:32], h)
        cand = _children(w, par, h, np.ones(len(par), bool))
        sc = w.scores(h - 1, cand)
        for pick in (int(np.argmax(sc)), int(np.argsort(sc)[len(sc) // 2])):
            s, xy = sc[pick], (cand[pick][1], cand[pick][2])
            up = np.nextafter(s, np.float32(2))
            down = np.nextafter(s, np.float32(-1))
            # parents stay live at B = s (a parent's sum bounds its children's)
            check_step(w, par, h, s, lo)
            check_step(w, par, h, up, lo)
            check_step(w, par, h, lo, s)
            check_step(w, par, h, lo, down)
            if h >= 2:
                assert xy in pushed(lo, s, h, par)[0]
                assert xy not in pushed(lo, up, h, par)[0]
                assert xy not in pushed(s, lo, h, par)[0]
                assert xy in pushed(down, lo, h, par)[0]
            else:
                assert pushed(lo, s, h, par)[1] >= s


def test_loose_parent_scores(small_world):
    """A parent score above its true sum (a looser p_hi) changes nothing."""
    w = small_world
    for h in (4, 2, 1):
        lat = w.lattice(1, h)[:33]
        exact = w.parents(lat, h)
        loose = w.parents(lat, h, loose=True)
        B = _tight_bound(w, exact, h)
        for form, unroll in FORMS:
            a = w.m.branch_step(w.cloud, w.pose, False, 0.1, h, exact, B, form, unroll)
            b = w.m.branch_step(w.cloud, w.pose, False, 0.1, h, loose, B, form, unroll)
            assert _key(a[0]) == _key(b[0]) and a[1] == b[1]
        check_step(w, loose, h, B, 0.1)


def test_points_outside_window_table(oracle, sm):
    """A third of the points lie hundreds of metres off the map (cell indices far outside
    every level's window table)."""
    rng = np.random.RandomState(5)
    w = World(oracle, sm, _random_cells(rng, 50, 60), 4, _cloud(rng, 400, 18, far=130),
              lin=1.0, ang=0.2)
    try:
        for h in (3, 2, 1):
            par = w.parents(w.lattice(0, h)[:33] + w.lattice(w.ds.shape[0] - 1, h)[:17], h)
            check_step(w, par, h, np.float32(0.1), 0.1)
            check_step(w, par, h, _tight_bound(w, par, h), 0.1)
    finally:
        w.close()


@pytest.mark.parametrize("n", [257, 1081, 9000])
def test_saturated_grid(oracle, sm, n):
    """Every cell at the highest probability: all children tie at 255 n, the early exit's
    bound is tight (c_t + p_hi - mx == t_min at every test) and the packed u16 sums come
    closest to overflowing (9000 points: > 256 per lane in the warp form)."""
    cells = np.ones((90, 90), np.uint16)
    w = World(oracle, sm, cells, 4, _cloud(np.random.RandomState(n), n, 12), lin=0.6, ang=0.1)
    try:
        assert (oracle.precompute_grid2d(cells, w.grid.min_cost, w.grid.max_cost, 1) == 255).all()
        for h in (3, 2, 1):
            par = w.parents(w.lattice(0, h)[:9] + w.lattice(1, h)[:32], h)
            top = _tight_bound(w, par, h)
            check_step(w, par, h, top, 0.1)
            check_step(w, par, h, np.float32(0.1), 0.1)
            # dense ties with re-maps: 3 parents live at the tied maximum
            p2 = par.copy()
            dead = np.ones(len(p2), bool)
            dead[[0, len(p2) // 2, len(p2) - 2]] = False
            p2["score"][dead] = np.nextafter(top, np.float32(-1))
            check_step(w, p2, h, top, 0.1)
    finally:
        w.close()


def test_every_level_on_config2_stack(oracle, sm):
    """Every h from depth - 1 down to 1 on a 1000 x 1000 depth-7 stack (the config-2
    layout) with a 1081-beam scan, at a loose and at the tight bound, 65 parents on each
    of three scans."""
    grid, occ = synthetic.make_grid2d(0, 1000)
    rng = np.random.RandomState(1)
    pose = synthetic.random_free_pose(occ, grid, rng)
    scan = synthetic.cast_scan(occ, grid, pose, seed=1)
    w = World(oracle, sm, grid, 7, scan, lin=3.0, ang=0.05,
              pose=pose + np.array([0.3, -0.2, 0.05]))
    try:
        S = w.ds.shape[0]
        for h in range(6, 0, -1):
            nodes = []
            for k in (0, S // 2, S - 1):
                lat = w.lattice(k, h)
                idx = np.random.RandomState(h * 10 + k).choice(len(lat), min(65, len(lat)),
                                                              replace=False)
                nodes += [lat[i] for i in np.sort(idx)]
            par = w.parents(nodes, h)
            check_step(w, par, h, np.float32(0.1), 0.1)
            check_step(w, par, h, _tight_bound(w, par, h), 0.1)
    finally:
        w.close()


@pytest.mark.parametrize("shape,depth", [((1, 1), 3), ((3, 7), 3), ((3, 7), 2)])
def test_tiny_grids(oracle, sm, shape, depth):
    """1 x 1 and 7 x 3 grids: lattices and window tables of one or two cells."""
    rng = np.random.RandomState(depth + shape[0])
    cells = rng.randint(1, 32768, size=shape).astype(np.uint16)
    w = World(oracle, sm, cells, depth, _cloud(rng, 200, 3), lin=0.5, ang=0.3)
    try:
        for h in range(depth - 1, 0, -1):
            nodes = []
            for k in range(w.ds.shape[0]):
                nodes += w.lattice(k, h)
            par = w.parents(nodes, h)
            check_step(w, par, h, np.float32(0.1), 0.1)
            if len(par):
                check_step(w, par, h, _tight_bound(w, par, h), 0.1)
    finally:
        w.close()


def test_rejects_parents_off_the_lattice(small_world, sm):
    from cartographer_b200 import _lib
    w = small_world
    par = w.parents(w.lattice(0, 2)[:3], 2)
    par["xo"][1] += 1
    with pytest.raises(_lib.CsmError) as e:
        w.m.branch_step(w.cloud, w.pose, False, 0.1, 2, par, np.float32(0.1), "lattice")
    assert e.value.status == 1
    with pytest.raises(_lib.CsmError):
        w.m.branch_step(w.cloud, w.pose, False, 0.1, w.depth, par[:1], np.float32(0.1), "warp")


def test_reports_points_beyond_the_cell_index_range(oracle, sm):
    """A point more than 30000 cells from the grid origin cannot be held in the int16
    cell indices: both hooks return CSM_E_CAPACITY, as a match does, instead of scoring
    a clamped scan."""
    from cartographer_b200 import _lib
    rng = np.random.RandomState(3)
    xyz = _cloud(rng, 200, 10)
    xyz[-1, :2] = (1600.0, -1400.0)  # ~42000 cells away
    w = World(oracle, sm, _random_cells(rng, 40, 40), 3, xyz, lin=0.5, ang=0.0)
    try:
        par = w.parents(w.lattice(0, 2)[:4], 2, loose=True)
        for form in ("warp", "lattice"):
            with pytest.raises(_lib.CsmError) as e:
                w.m.branch_step(w.cloud, w.pose, False, 0.1, 2, par, np.float32(0.1), form)
            assert e.value.status == 3
        with pytest.raises(_lib.CsmError) as e:
            w.m.score_top(w.cloud, w.pose)
        assert e.value.status == 3
        with pytest.raises(_lib.CsmError) as e:
            w.m.Match(w.pose, w.cloud, 0.1)
        assert e.value.status == 3
    finally:
        w.close()
