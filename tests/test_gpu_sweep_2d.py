"""The 2D branch-and-bound sweep around its branch step, against the oracle and an
exact numpy replay.

A. Greedy dives (k_job_best, k_dive) through csm_dives2d, replayed exactly: per scan
   the argmax of the lowest-resolution sums (lowest slot i * nyc + j on ties), the two
   gates (top score > min_score; not float32(best) < float32(ratio) * float32(job_best)),
   the greedy descent (highest child sum, lowest t = (dx << 1) | dy on ties, a child
   valid unless past max_x / max_y), the bound (max of min_score and every leaf score
   > min_score) and the counters (valid children scored, dives run).
B. The top queue (k_filter_top, k_top_as_leaves at depth 1): every lowest-resolution
   candidate with score > min_score and score >= the bound after the dives, each scan's
   run in row-major order (y outer, x inner); at depth 1 the leaves are the queue and
   the bound its maximum.
C. The chunked level loop: every case under small chunks, with and without the lattice
   kernel on split chunks, and without dives, gives the oracle's result bit for bit and
   the default run's leaves_tied; the trace shows the continuation sweeps ran.
D. Exactly tied optima: the inline read-back overflow, the sort replay of tied
   lowest-resolution candidates, leaf compaction between sweeps, and both capacity
   refusals (after which the same matcher matches again).
E. A batch mixing depths, min_scores, local and full-submap jobs and repeated handles,
   equal to the oracle in job order whole, one job per sub-batch and with small chunks.
"""
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import worlds

pytestmark = pytest.mark.gpu

RES = 0.05


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _bits(v):
    return int(np.float32(v).view(np.uint32))


class Case:
    """One match (stack, cloud, search) on the device and in the oracle."""

    def __init__(self, oracle, sm, grid, depth, cloud, pose=(0.0, 0.0, 0.0), lin=1.0, ang=0.3,
                 full=False, min_score=0.1):
        if isinstance(grid, np.ndarray):  # cells of a map centred on the world origin
            ny, nx = grid.shape
            grid = synthetic.GridSpec(grid, RES, 0.5 * ny * RES, 0.5 * nx * RES)
        self.oracle, self.sm, self.grid = oracle, sm, grid
        self.depth, self.lin, self.ang, self.full = depth, lin, ang, full
        self.min_score = np.float32(min_score)
        self.pose = np.asarray(pose, np.float64)
        self.cloud = np.ascontiguousarray(cloud, np.float32)
        self.m = sm.FastCorrelativeScanMatcher2D(
            grid, sm.FastCorrelativeScanMatcherOptions2D(lin, ang, depth))
        self.dcloud = sm.DeviceCloud(self.cloud)
        self.og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
        self.om = oracle.FastCorrelativeScanMatcher2D(self.og, lin, ang, depth)
        self._fe = None
        self._want = None
        self._top = None

    def close(self):
        self.m.close()
        self.dcloud.close()

    @property
    def fe(self):
        if self._fe is None:
            fe = self.oracle.frontend2d(self.og, self.cloud, self.pose, full=self.full,
                                        lin=self.lin, ang=self.ang)
            self._fe = (fe["discrete_scans"], fe["bounds"])
        return self._fe

    def want(self):
        """The oracle's match (cached: every limit variant compares against one run)."""
        if self._want is None:
            if self.full:
                self._want = self.om.match_full_submap(self.cloud, self.min_score)
            else:
                self._want = self.om.match(self.pose, self.cloud, self.min_score)
        return self._want

    def job(self, min_score=None):
        jobs = np.zeros(1, self.sm.JOB2D_DTYPE)
        jobs["full_submap"] = int(self.full)
        jobs["initial_pose"] = self.pose
        jobs["min_score"] = self.min_score if min_score is None else min_score
        return jobs

    def run(self, limits=None):
        res, st = self.sm.match_batch([self.m], [self.dcloud], self.job(), self.lin, self.ang,
                                      limits)
        return res[0], st

    def dives(self, min_score, ratio):
        return self.m.dives(self.cloud, self.pose, self.full, min_score, ratio)

    def scores(self, level, cand):
        cand = np.asarray(cand, np.int32).reshape(-1, 3)
        if not len(cand):
            return np.zeros(0, np.float32), np.zeros(0, np.int32)
        return self.om.score_candidates(level, self.fe[0], cand)

    def top(self):
        """Per scan: the lowest-resolution lattice (x outer, y inner: slot order), its sums
        and scores."""
        if self._top is not None:
            return self._top
        h = self.depth - 1
        lat = []
        for k, (mnx, mxx, mny, mxy) in enumerate(self.fe[1]):
            lat.append([(k, x, y) for x in range(mnx, mxx + 1, 1 << h)
                        for y in range(mny, mxy + 1, 1 << h)])
        sc, su = self.scores(h, [c for l in lat for c in l])
        out, o = [], 0
        for l in lat:
            out.append((l, su[o:o + len(l)], sc[o:o + len(l)]))
            o += len(l)
        self._top = out
        return out


def replay_dives(case, min_score, ratio):
    """-> (job_best, bound after the dives, candidates scored, dives run)."""
    min_score, ratio = np.float32(min_score), np.float32(ratio)
    top = case.top()
    job_best = max([int(su.max()) for _, su, _ in top if len(su)] + [0])
    divers = []  # [scan, x, y, sum, score]
    for lat, su, sc in top:
        if not len(su):
            continue
        slot = int(np.argmax(su))  # first maximum: the lowest slot
        if not sc[slot] > min_score:
            continue
        if np.float32(su[slot]) < ratio * np.float32(job_best):
            continue
        divers.append(list(lat[slot]) + [int(su[slot]), sc[slot]])
    bounds = case.fe[1]
    scored = 0
    for h in range(case.depth - 1, 0, -1):
        half = 1 << (h - 1)
        cand, owner = [], []
        for d, (k, x, y, _, _) in enumerate(divers):
            for t in range(4):
                cx, cy = x + (t >> 1) * half, y + (t & 1) * half
                if cx <= bounds[k, 1] and cy <= bounds[k, 3]:
                    cand.append((k, cx, cy))
                    owner.append(d)
        sc, su = case.scores(h - 1, cand)
        scored += len(cand)
        best = {}
        for c, o, s, f in zip(cand, owner, su, sc):
            if o not in best or s > best[o][1]:  # ties keep the lowest t (generation order)
                best[o] = (c, int(s), f)
        for o, (c, s, f) in best.items():
            divers[o] = [c[0], c[1], c[2], s, f]
    bound = min_score
    for d in divers:
        if d[4] > min_score:
            bound = max(bound, d[4])
    return job_best, np.float32(bound), scored, len(divers)


def expected_queue(case, min_score, bound):
    """Per scan: the kept lowest-resolution candidates in row-major order."""
    out = {}
    for lat, su, sc in case.top():
        keep = [(c[2], c[1], _bits(s)) for c, s in zip(lat, sc) if s > min_score and s >= bound]
        if keep:
            out[lat[0][0]] = [(x, y, b) for y, x, b in sorted(keep)]
    return out


def check_dives(case, min_score, ratio):
    min_score = np.float32(min_score)
    job_best, (b_dive, b_top), ctr, queue = case.dives(min_score, ratio)
    want = replay_dives(case, min_score, ratio)
    tag = (case.depth, float(min_score), float(ratio))
    assert job_best == want[0], tag
    assert _bits(b_dive) == _bits(want[1]), (tag, b_dive, want[1])
    assert ctr == (want[2], want[3]), (tag, ctr, want[2:])
    # B: the top queue
    exp = expected_queue(case, min_score, b_dive)
    got = {}
    for r in queue:
        got.setdefault(int(r["scan"]), []).append((int(r["xo"]), int(r["yo"]), _bits(r["score"])))
    assert got == exp, tag
    assert len(queue) == sum(len(v) for v in exp.values())
    if case.depth == 1 and len(queue):
        assert _bits(b_top) == _bits(max(b_dive, queue["score"].max())), tag
    else:
        assert _bits(b_top) == _bits(b_dive), tag
    return want


def _random_cells(rng, ny, nx, zero=0.3):
    cells = rng.randint(1, 32768, size=(ny, nx)).astype(np.uint16)
    cells[rng.uniform(size=cells.shape) < zero] = 0
    return cells


def _cloud(rng, n, radius_cells):
    xy = rng.uniform(-radius_cells, radius_cells, (n, 2)) * RES
    return np.concatenate([xy, np.zeros((n, 1))], axis=1).astype(np.float32)


def _uniform_case(oracle, sm, depth, lin=1.0, ang=0.5, n=40):
    """Every cell at the highest probability and every point of every candidate inside
    the map at every level: every candidate of every level ties."""
    cloud = _cloud(np.random.RandomState(depth), n, 20)
    return Case(oracle, sm, np.ones((200, 200), np.uint16), depth, cloud, lin=lin, ang=ang)


DIVE_CASES = {
    # windows that are not multiples of 2^h: children fall off the lattice
    "random_d5": dict(shape=(96, 80), depth=5, lin=1.3, ang=0.3),
    "random_d2": dict(shape=(96, 80), depth=2, lin=0.55, ang=0.3),
    "random_d1": dict(shape=(60, 70), depth=1, lin=0.3, ang=0.2),
    "one_scan": dict(shape=(96, 80), depth=4, lin=1.1, ang=0.0),
    "one_slot": dict(shape=(60, 60), depth=3, lin=0.0, ang=0.3),
    "few_slots": dict(shape=(60, 60), depth=3, lin=0.2, ang=0.3),
    "many_slots": dict(shape=(96, 96), depth=3, lin=2.0, ang=0.1),
    "full_submap": dict(full=True, depth=5),
    "plateau": dict(plateau=True, depth=4, lin=0.6, ang=0.2),
    "plateau_d1": dict(plateau=True, depth=1, lin=0.3, ang=0.1),
}


@pytest.fixture(scope="module")
def dive_cases(oracle, sm):
    made = {}

    def get(name):
        if name not in made:
            p = DIVE_CASES[name]
            rng = np.random.RandomState(len(made) + 7)
            if p.get("full"):
                grid, occ, pose, scan = worlds.small_world(203, size_cells=100, beams=91)
                made[name] = Case(oracle, sm, grid, p["depth"], scan, lin=1.0, ang=0.3, full=True)
            elif p.get("plateau"):
                made[name] = _uniform_case(oracle, sm, p["depth"], p["lin"], p["ang"])
            else:
                made[name] = Case(oracle, sm, _random_cells(rng, *p["shape"]), p["depth"],
                                  _cloud(rng, 500, 25), lin=p["lin"], ang=p["ang"])
        return made[name]

    yield get
    for c in made.values():
        c.close()


@pytest.mark.parametrize("name", sorted(DIVE_CASES))
def test_dives_and_top_queue(dive_cases, name):
    """A and B: every ratio gate (0, the default, 1 and > 1), at a low min_score and at
    min_score equal to a top score."""
    case = dive_cases(name)
    top = case.top()
    scores = np.concatenate([sc for _, _, sc in top])
    sums = [su for _, su, _ in top]
    assert len(scores) >= 1
    if name == "one_slot":
        assert all(len(s) == 1 for s in sums)
    if name == "few_slots":
        assert all(1 < len(s) < 32 for s in sums)
    if name == "many_slots":
        assert all(len(s) > 32 for s in sums)
    if name.startswith("plateau"):
        assert len(set(scores.tolist())) == 1
    ratios = [0.0, 0.97, 1.0, 1.5]
    lows = [np.float32(0.05), np.float32(np.median(scores))]
    for min_score in lows:
        n_dives = []
        for ratio in ratios:
            n_dives.append(check_dives(case, min_score, ratio)[3])
        # ratio 0 dives from every scan that clears min_score; > 1 from none
        assert n_dives[3] == 0
        assert n_dives[0] >= n_dives[1] >= n_dives[2]


@pytest.mark.parametrize("name", ["random_d5", "many_slots", "full_submap"])
def test_dives_gate_at_exact_product(dive_cases, name):
    """A ratio whose float32 product with job_best equals a scan's best exactly: the scan
    dives (the gate is a strict <), and one ulp more ratio is replayed as well."""
    case = dive_cases(name)
    sums = [su for _, su, _ in case.top()]
    job_best = np.float32(max(int(s.max()) for s in sums))
    found = 0
    for s in sorted({int(s.max()) for s in sums}):
        if s >= job_best:
            continue
        for r in (np.float32(np.float32(s) / job_best),):
            for c in (r, np.nextafter(r, np.float32(2)), np.nextafter(r, np.float32(0))):
                if np.float32(c) * job_best == np.float32(s):
                    at = check_dives(case, 0.05, c)[3]
                    above = check_dives(case, 0.05, np.nextafter(c, np.float32(2)))[3]
                    assert at >= above
                    found += 1
                    break
        if found >= 2:
            break
    if not found:
        pytest.skip("no float32 ratio hits a scan's best exactly")


# ---- C: the chunked level loop ----------------------------------------------
def _local_case(oracle, sm, seed):
    grid, occ, pose, scan = worlds.small_world(100 + seed)
    rng = np.random.RandomState(seed)
    init = pose + np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-0.3, 0.3)])
    return Case(oracle, sm, grid, 3 + seed % 4, scan, init, 2.0, 0.5, min_score=0.3)


def _full_case(oracle, sm, seed):
    grid, occ, pose, scan = worlds.small_world(200 + seed, size_cells=160, beams=121)
    return Case(oracle, sm, grid, 5, scan, lin=1.0, ang=0.3, full=True, min_score=0.4)


FAST_CLOUD = np.array([[-2.5, 0.5, 0], [-2.0, 0.5, 0], [0.0, -0.5, 0], [0.5, -1.6, 0],
                       [2.5, 0.5, 0], [2.5, 1.7, 0]], np.float32)


def _transform(cloud, pose):
    c, s = math.cos(pose[2]), math.sin(pose[2])
    out = cloud.copy()
    out[:, 0] = c * cloud[:, 0] - s * cloud[:, 1] + pose[0]
    out[:, 1] = s * cloud[:, 0] + c * cloud[:, 1] + pose[1]
    return out.astype(np.float32)


def _sparse_case(oracle, sm, k):
    """The reference's correct-pose test: a sparse cloud on a near-empty map (many ties)."""
    rng = np.random.RandomState(42)
    for _ in range(k + 1):
        u = rng.uniform(-1.0, 1.0, 3)
    expected = (2.0 * u[0], 2.0 * u[1], 0.5 * u[2])
    og = worlds.insert_range_data(oracle, 200, 200, 0.05, 5.0, 5.0, expected[:2],
                                  _transform(FAST_CLOUD, expected))
    grid = synthetic.GridSpec(og.cells, 0.05, 5.0, 5.0)
    return Case(oracle, sm, grid, 3, FAST_CLOUD, lin=3.0, ang=1.0, min_score=0.1)


def _large_case(oracle, sm):
    grid, occ = synthetic.make_grid2d(0, 1000)
    rng = np.random.RandomState(1)
    pose = synthetic.random_free_pose(occ, grid, rng)
    scan = synthetic.cast_scan(occ, grid, pose, seed=1)
    return Case(oracle, sm, grid, 7, scan, pose + np.array([1.5, -2.0, 0.2]), lin=7.0,
                ang=math.radians(30.0), min_score=0.55)


SWEEP_CASES = (["local%d" % s for s in range(8)] + ["full%d" % s for s in range(4)] +
               ["sparse%d" % k for k in range(4)] + ["large"])


@pytest.fixture(scope="module")
def sweep_cases(oracle, sm):
    made = {}

    def get(name):
        if name not in made:
            if name == "large":
                made[name] = _large_case(oracle, sm)
            else:
                kind, k = name.rstrip("0123456789"), int(name[len(name.rstrip("0123456789")):])
                made[name] = {"local": _local_case, "full": _full_case,
                              "sparse": _sparse_case}[kind](oracle, sm, k)
        return made[name]

    yield get
    for c in made.values():
        c.close()


def check_result(case, res, st, ref=None):
    """The oracle's result bit for bit; `ref` (the default run) for leaves_tied."""
    want = case.want()
    assert bool(res["found"]) == want["found"]
    if want["found"]:
        assert _bits(res["score"]) == _bits(want["score"])
        np.testing.assert_array_equal(res["pose_estimate"], want["pose"])
        assert (int(res["best_scan_index"]), int(res["best_x_offset"]), int(res["best_y_offset"])) == (
            want["best_scan_index"], want["best_x_offset"], want["best_y_offset"])
    if ref is not None:
        assert int(res["leaves_tied"]) == int(ref["leaves_tied"])
        for k in ("found", "score", "best_scan_index", "best_x_offset", "best_y_offset"):
            assert res[k] == ref[k], k


def _variants(name, nodes):
    v = []
    if nodes <= 4000:
        v += [{"chunk": 1}, {"chunk": 2}]
    v += [{"chunk": c} for c in (31, 32, 33, 1000)]
    v += [{"chunk": c, "lattice_min": 1} for c in ((2, 31, 33, 1000) if nodes <= 4000 else
                                                    (31, 33, 1000))]
    v += [{"dive_ratio": 2.0}, {"dive_ratio": 2.0, "chunk": 33}]
    if name == "large":
        v += [{"chunk": c} for c in (16383, 16384, 16385)]
        v += [{"chunk": c, "dive_ratio": 2.0} for c in (16383, 16384, 16385)]
    return v


@pytest.mark.parametrize("name", SWEEP_CASES)
def test_chunked_level_loop(sweep_cases, name):
    case = sweep_cases(name)
    ref, st0 = case.run()
    check_result(case, ref, st0)
    assert st0["sweep_trace"][0] >= 1
    assert st0["host_syncs"] == st0["sweep_trace"][0] + (st0["sweep_trace"][3] > 4096)
    top_default = case.dives(case.min_score, 0.97)[3]
    top_loose = case.dives(case.min_score, 2.0)[3]
    continued = 0
    for lim in _variants(name, st0["nodes_expanded"]):
        res, st = case.run(lim)
        check_result(case, res, st, ref)
        trace = st["sweep_trace"]
        top = top_loose if lim.get("dive_ratio", 0.97) > 1 else top_default
        if len(top) > lim.get("chunk", 1 << 23):
            # the top level held more than one chunk: the host continued
            assert trace[0] > 1, (lim, trace, len(top))
            continued += 1
        assert st["host_syncs"] == trace[0] + (trace[3] > 4096), (lim, trace)
        assert trace[3] == st["leaves_tied"] or not res["found"]
    assert continued >= 1


# ---- D: leaves and ties -----------------------------------------------------
@pytest.fixture(scope="module")
def uniform_cases(oracle, sm):
    made = {}

    def get(depth):
        if depth not in made:
            made[depth] = _uniform_case(oracle, sm, depth)
        return made[depth]

    yield get
    for c in made.values():
        c.close()


def _all_leaves(case):
    b = case.fe[1].astype(np.int64)
    return int(((b[:, 1] - b[:, 0] + 1) * (b[:, 3] - b[:, 2] + 1)).sum())


@pytest.mark.parametrize("depth", [1, 3, 5])
def test_uniform_grid_ties(uniform_cases, depth):
    """Every leaf ties: more optimal leaves than the inline read-back holds (one more host
    sync), the DFS-first leaf through the sort replay of tied lowest-resolution
    candidates."""
    case = uniform_cases(depth)
    n = _all_leaves(case)
    assert n > 4096
    for lim in (None, {"inline_best": 0}, {"inline_best": 1}, {"inline_best": 4096},
                {"chunk": 1000}, {"chunk": 33, "lattice_min": 1}):
        res, st = case.run(lim)
        check_result(case, res, st)
        trace = st["sweep_trace"]
        assert res["leaves_tied"] == n and trace[3] == n, lim
        assert st["host_tie_resolves"] >= 1, lim
        inline = 4096 if lim is None else lim.get("inline_best", 4096)
        assert st["host_syncs"] == trace[0] + 1 and n > inline, (lim, st["host_syncs"], trace)
        if lim and "chunk" in lim and depth > 1:
            assert trace[0] > 1, (lim, trace)


def test_few_ties_read_back_inline(sweep_cases):
    """Optimal leaves within inline_best come back with the collect; one more than
    inline_best costs one more sync."""
    case = sweep_cases("sparse0")
    ref, st = case.run()
    n = int(ref["leaves_tied"])
    assert n >= 1 and st["host_syncs"] == st["sweep_trace"][0]
    for inline, extra in ((n, 0), (n - 1, 1), (0, 1)):
        res, st = case.run({"inline_best": inline})
        check_result(case, res, st, ref)
        assert st["host_syncs"] == st["sweep_trace"][0] + extra, (inline, st)


@pytest.mark.parametrize("name", ["random_d5", "many_slots", "one_scan"])
def test_leaf_compaction(dive_cases, name):
    """No dives, one node per chunk and an 8-leaf buffer: the bound rises leaf by leaf,
    the non-optimal leaves fill the buffer and are compacted away between sweeps (a
    continuation adds at most 4 leaves to at most 4 kept ones, so nothing overflows)."""
    case = dive_cases(name)
    ref, _ = case.run()
    res, st = case.run({"chunk": 1, "leaf_cap": 8, "dive_ratio": 2.0})
    check_result(case, res, st, ref)
    trace = st["sweep_trace"]
    assert trace[1] >= 1, trace
    assert trace[2] <= 8


def test_too_many_tied_leaves_is_refused(uniform_cases):
    from cartographer_b200 import _lib
    case = uniform_cases(3)
    with pytest.raises(_lib.CsmError) as e:
        # all leaves tie and stay; one continuation adds at most 256 to at most 256
        case.run({"chunk": 64, "leaf_cap": 512})
    assert e.value.status == 3 and "too many tied leaves" in str(e.value)
    res, st = case.run()
    check_result(case, res, st)
    assert res["leaves_tied"] == _all_leaves(case)


def test_depth1_top_overflow_is_refused(uniform_cases):
    """Depth 1: every queued candidate is a leaf, and all of them tie here."""
    from cartographer_b200 import _lib
    for case in (uniform_cases(1),):
        top = len(case.dives(case.min_score, 0.97)[3])
        assert top > 2
        with pytest.raises(_lib.CsmError) as e:
            case.run({"leaf_cap": max(2, top - 1)})
        assert e.value.status == 3
        res, st = case.run({"leaf_cap": top})
        check_result(case, res, st)
        res, st = case.run()
        check_result(case, res, st)


# ---- E: batches -------------------------------------------------------------
def test_mixed_batch(oracle, sm):
    rng = np.random.RandomState(9)
    worlds_ = [worlds.small_world(300 + i, size_cells=120, beams=91, max_range=5.0)
               for i in range(2)]
    depths = [1, 2, 5, 7]
    lin, ang = 0.6, 0.2
    stacks, ostacks = [], []
    for d in depths:
        for g, _, _, _ in worlds_:
            stacks.append(sm.FastCorrelativeScanMatcher2D(
                g, sm.FastCorrelativeScanMatcherOptions2D(lin, ang, d)))
            og = oracle.Grid2D(g.cells, g.resolution, g.max_x, g.max_y)
            ostacks.append(oracle.FastCorrelativeScanMatcher2D(og, lin, ang, d))
    clouds = [sm.DeviceCloud(w[3]) for w in worlds_]
    jobs = []
    for k in range(22):
        si = int(rng.randint(len(stacks)))
        ci = si % 2 if k % 5 else 1 - si % 2  # mostly the stack's own world
        full = k % 7 == 3
        # every third job asks for more than any pose scores: found = 0 between found jobs
        ms = 0.97 if k % 3 == 1 else float(rng.choice([0.1, 0.3, 0.45]))
        init = worlds_[ci][2] + rng.uniform(-0.3, 0.3, 3) * [1, 1, 0.3]
        jobs.append((si, ci, full, init, ms))
    jarr = np.zeros(len(jobs), sm.JOB2D_DTYPE)
    for k, (si, ci, full, init, ms) in enumerate(jobs):
        jarr[k]["stack_index"], jarr[k]["cloud_index"] = si, ci
        jarr[k]["full_submap"], jarr[k]["initial_pose"], jarr[k]["min_score"] = full, init, ms
    assert len({stacks[si].options.branch_and_bound_depth for si, *_ in jobs}) == 4
    try:
        res, st = sm.match_batch(stacks, clouds, jarr, lin, ang)
        found = []
        for k, (si, ci, full, init, ms) in enumerate(jobs):
            om = ostacks[si]
            cloud = worlds_[ci][3]
            want = om.match_full_submap(cloud, ms) if full else om.match(init, cloud, ms)
            assert bool(res[k]["found"]) == want["found"], k
            found.append(want["found"])
            if want["found"]:
                assert _bits(res[k]["score"]) == _bits(want["score"]), k
                np.testing.assert_array_equal(res[k]["pose_estimate"], want["pose"])
                assert (int(res[k]["best_scan_index"]), int(res[k]["best_x_offset"]),
                        int(res[k]["best_y_offset"])) == (
                    want["best_scan_index"], want["best_x_offset"], want["best_y_offset"]), k
        # jobs that find nothing sit between jobs that do
        assert any(not f and any(found[:k]) and any(found[k + 1:]) for k, f in enumerate(found))
        for lim in ({"max_points": 1}, {"chunk": 7}, {"max_points": 1, "chunk": 7}):
            got, st2 = sm.match_batch(stacks, clouds, jarr, lin, ang, lim)
            assert got.tobytes() == res.tobytes(), lim
            if "max_points" in lim:
                assert st2["sweep_trace"][0] >= len(jobs)
    finally:
        for m in stacks:
            m.close()
        for c in clouds:
            c.close()
