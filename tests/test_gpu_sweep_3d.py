"""The 3D branch-and-bound sweep around its branch step, against the oracle and numpy.

A. The top queue (k3_filter_top) through csm_top_queue3d, compared as a set with a numpy
   filter of csm_score_top3d's lowest-resolution sums: every candidate with
   ToScore(sum) > min_score and >= the bound after the dives, with its score bits; with
   dives, without dives (the bound is min_score), on a saturated world whose bound ties
   many candidates, and with min_score equal to a candidate's score.
B. The chunked level loop (k3_level_begin, continuation sweeps, Collect3D): parity,
   random-voxel, tie and full-submap worlds under chunks of 1 .. 65535 and the default,
   with and without dives, give the oracle's Result bit for bit and the default run's
   leaves_tied; the trace shows the continuation sweeps ran.
C. The leaf list's capacity: where the dives already reach the optimum the recorded leaves
   are exactly the T tied ones, so leaf_cap = T matches and T - 1 is refused with
   CSM_E_CAPACITY, after which the same matcher matches again, alone and in a batch.
D. The optimal-leaf read-back: T-way ties (T = 0, 1, 2, 255, 256, 257) under inline_best
   0, 1, T - 1, T, T + 1 give one result, and host_syncs counts the extra copy exactly.
E. Batches mixing depths, full_resolution_depths, local and full-submap jobs, min_scores,
   repeated matchers and nodes and an empty histogram, under 1, 3 and 24 workers (more
   than the 16 lanes) and small chunks, equal to the single calls and the oracle; a batch
   with a refused job, and the one after it; the sharded queues on a world-1 context.
"""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import worlds3d
from tests.test_gpu_parity_3d import _building_case
from tests.test_gpu_score3d import _saturated_world, world

pytestmark = pytest.mark.gpu

RES = 0.1
IDENT = [0, 0, 0, 1, 0, 0, 0]
POSE = [0.03, -0.02, 0.01, 1, 0, 0, 0]
NO_DIVES = 2.0   # k3_dive's gate: best < 2 * TopBest for every scan with a non-zero sum
CHUNKS = [1, 2, 7, 8, 9, 64, 4096, 65535, None]


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _bits(v):
    return int(np.float32(v).view(np.uint32))


class Case3:
    """One 3D match (matcher, node, poses) on the device and in the oracle."""

    def __init__(self, oracle, sm, hi, lo, od, node, node_pose=POSE, submap_pose=IDENT,
                 full=False, min_score=0.2, hist=None):
        self.sm, self.od, self.node, self.full = sm, od, node, full
        self.node_pose = np.asarray(node_pose, np.float64)
        self.submap_pose = np.asarray(submap_pose, np.float64)
        self.min_score = np.float32(min_score)
        self.om, self.m = worlds3d.make_pair(oracle, sm, hi, lo, od, hist=hist)
        self.en = worlds3d.engine_node(sm, node)
        self._want = None

    def close(self):
        self.m.close()

    def want(self):
        if self._want is None:
            if self.full:
                self._want = self.om.match_full_submap(self.node_pose[3:], self.submap_pose[3:],
                                                       self.node, self.min_score)
            else:
                self._want = self.om.match(self.node_pose, self.submap_pose, self.node,
                                           self.min_score)
        return self._want

    def job(self, matcher_index=0, node_index=0, min_score=None):
        return (matcher_index, node_index, self.full, self.node_pose, self.submap_pose,
                self.min_score if min_score is None else min_score)

    def run(self, **limits):
        """One job through csm_match3d_batch_limits -> (result, stats incl. sweep_trace)."""
        res, st = self.sm.match_batch3d([self.m], [self.en], [self.job()], limits=limits)
        return res[0], st

    def single(self):
        return self.m.match_raw(self.full, self.node_pose, self.submap_pose, self.en,
                                self.min_score)

    def top(self):
        return self.m.score_top(self.full, self.node_pose, self.submap_pose, self.en,
                                self.min_score)

    def top_queue(self, ratio, min_score=None):
        ms = self.min_score if min_score is None else min_score
        return self.m.top_queue(self.full, self.node_pose, self.submap_pose, self.en, ms, ratio)


def check_result(got, want):
    """Every Result field bit for bit with the oracle's."""
    assert (got is not None) == want["found"]
    if got is None:
        return
    assert _bits(got["score"]) == _bits(want["score"])
    np.testing.assert_array_equal(got["pose_estimate"], want["pose"])
    assert _bits(got["rotational_score"]) == _bits(want["rotational_score"])
    assert _bits(got["low_resolution_score"]) == _bits(want["low_resolution_score"])
    assert (got["best_scan_index"],) + got["best_offset"] == (
        want["best_scan_index"], want["best_x"], want["best_y"], want["best_z"])


def same_result(a, b):
    assert (a is None) == (b is None)
    if a is None:
        return
    assert _bits(a["score"]) == _bits(b["score"])
    np.testing.assert_array_equal(a["pose_estimate"], b["pose_estimate"])
    assert _bits(a["rotational_score"]) == _bits(b["rotational_score"])
    assert _bits(a["low_resolution_score"]) == _bits(b["low_resolution_score"])
    assert a["best_scan_index"] == b["best_scan_index"] and a["best_offset"] == b["best_offset"]
    assert a["leaves_tied"] == b["leaves_tied"]


# ---- worlds -------------------------------------------------------------------------------
def building_case(oracle, sm, seed=11):
    """test_gpu_parity_3d's building world: a lidar scan of a synthetic building."""
    hi, lo, cloud, low, hn, hs, node_pose = _building_case(seed)
    od = worlds3d.fast_options(depth=6, frd=3, xy=1.5, z=0.5, angular=0.25, min_rot=0.3,
                               min_low=0.25)
    node = worlds3d.node_data(cloud, low=low, hist=hn)
    rng = np.random.RandomState(seed)
    init = node_pose.copy()
    init[:3] += rng.uniform(-0.8, 0.8, 3) * [1, 1, 0.3]
    yaw = 2 * math.atan2(node_pose[6], node_pose[3]) + rng.uniform(-0.15, 0.15)
    init[3:] = [math.cos(yaw / 2), 0, 0, math.sin(yaw / 2)]
    return Case3(oracle, sm, hi, lo, od, node, node_pose=init, min_score=0.3, hist=hs)


def random_case(oracle, sm, seed=4, depth=5, frd=3, min_score=0.15, hist=None, node_hist=None):
    """test_gpu_score3d's random-voxel world."""
    rng, hi, lo, node = world(seed, 300, n_vox=30000)
    if node_hist is not None:
        node["rotational_scan_matcher_histogram"] = node_hist
    od = worlds3d.fast_options(depth=depth, frd=frd, xy=0.7, z=0.3, angular=0.06, min_low=0.14)
    return Case3(oracle, sm, hi, lo, od, node, min_score=min_score, hist=hist)


def tie_case(oracle, sm, seed, holes, min_low):
    """test_gpu_score3d's tie worlds: a saturated box (with holes) and a cloud inside it, so
    the optimum is tied among many leaves (holes: their ancestors differ; min_low: the
    gate rejects some)."""
    rng = np.random.RandomState(seed)
    hi, lo = _saturated_world(rng, 26, 4, holes)
    cloud = worlds3d.random_cloud(rng, 40, 0.8)
    node = worlds3d.node_data(cloud, low=worlds3d.random_cloud(rng, 30, 1.5))
    od = worlds3d.fast_options(depth=3, frd=2, xy=0.3, z=0.1, angular=0.06, min_low=min_low)
    return Case3(oracle, sm, hi, lo, od, node, min_score=0.2)


def full_submap_case(oracle, sm, seed=9, depth=7):
    """MatchFullSubmap (the whole grid, every angle) of a sparse saturated grid by a cloud
    of its own voxel centres: one sharp optimum at offset 0, angle 0."""
    rng = np.random.RandomState(seed)
    idx = np.unique(rng.randint(-6, 6, size=(150, 3)), axis=0).astype(np.int32)
    hi = synthetic.HybridGridSpec(RES, idx, np.full(len(idx), 32767, np.uint16))
    lo = worlds3d.random_voxels(rng, 200, 3, 0.45)
    cloud = (idx[:80] * RES + 0.01).astype(np.float32)
    node = worlds3d.node_data(cloud, low=cloud)
    od = worlds3d.fast_options(depth=depth, frd=3, xy=0.7, z=0.3, angular=0.06)
    return Case3(oracle, sm, hi, lo, od, node, node_pose=IDENT, full=True, min_score=0.5)


def point_case(oracle, sm, T, seed=0, wxy=5, wz=2, depth=3):
    """A one-point cloud over a grid whose only occupied voxels are T saturated ones under
    T offsets of the window: exactly T leaves tie at the optimum, every gate passes, and
    since no voxel lies outside the window the dives reach the optimum."""
    rng = np.random.RandomState(1000 + seed)
    p = np.array([[0.013, -0.021, 0.017]], np.float32)
    node = worlds3d.node_data(p, low=p)
    # the point's cell under POSE (k3_discretize: lround((p + t) / resolution))
    c = np.floor((p[0].astype(np.float64) + POSE[:3]) / RES + 0.5).astype(np.int64)
    offs = np.array([(x, y, z) for z in range(-wz, wz + 1) for y in range(-wxy, wxy + 1)
                     for x in range(-wxy, wxy + 1)])
    pick = offs[rng.choice(len(offs), T, replace=False)] + c if T else np.array([[90, 90, 90]])
    hi = synthetic.HybridGridSpec(RES, pick.astype(np.int32), np.full(len(pick), 32767, np.uint16))
    lo = worlds3d.random_voxels(rng, 300, 4, 0.45)
    od = worlds3d.fast_options(depth=depth, frd=depth, xy=wxy * RES, z=wz * RES, angular=0.0)
    case = Case3(oracle, sm, hi, lo, od, node, min_score=0.2)
    case.T = T
    return case


# ---- A. the top queue -----------------------------------------------------------------------
def expected_queue(case, top, bound, min_score):
    """numpy k3_filter_top over csm_score_top3d's sums (scan-major, z, y, x)."""
    sums = top["sums"]
    n = len(case.node["high_resolution_point_cloud"])
    sc = worlds3d.to_score(sums, n)
    keep = (sc > np.float32(min_score)) & (sc >= np.float32(bound))
    s, kz, ky, kx = np.nonzero(keep)
    step = 1 << (case.od["branch_and_bound_depth"] - 1)
    wxy, wz = worlds3d.search_window(case.od, RES)
    out = np.zeros(len(s), case.sm.BNB_NODE3D_DTYPE)
    out["scan"], out["x"], out["y"], out["z"] = s, -wxy + kx * step, -wxy + ky * step, -wz + kz * step
    out["score"] = sc[keep]
    return out, sc


def as_set(q):
    order = np.lexsort((q["x"], q["y"], q["z"], q["scan"]))
    return q[order]


def check_queue(case, ratio, min_score=None):
    ms = case.min_score if min_score is None else np.float32(min_score)
    top = case.m.score_top(case.full, case.node_pose, case.submap_pose, case.en, ms)
    bound, q = case.top_queue(ratio, ms)
    if ratio > 1:
        assert _bits(bound) == _bits(ms)
    else:
        assert _bits(bound) == _bits(top["bound"])    # score_top runs the default 0.97
    want, sc = expected_queue(case, top, bound, ms)
    got = as_set(q)
    want = as_set(want)
    assert len(got) == len(want)
    for f in ("scan", "x", "y", "z"):
        np.testing.assert_array_equal(got[f], want[f])
    np.testing.assert_array_equal(got["score"].view(np.uint32), want["score"].view(np.uint32))
    return bound, q, sc


@pytest.mark.parametrize("world_name", ["building", "random3", "random4"])
def test_top_queue_with_and_without_dives(oracle, sm, world_name):
    """Depth 3 and 4 give the random world 32 and 12 lowest-resolution candidates per scan;
    the building (depth 6) has one."""
    if world_name == "building":
        case = building_case(oracle, sm)
    else:
        case = random_case(oracle, sm, depth=int(world_name[-1]), frd=2)
    bound, q, sc = check_queue(case, 0.97)
    assert bound > case.min_score            # the dives raised the bound
    bound2, q2, _ = check_queue(case, NO_DIVES)
    assert len(q2) == (sc > case.min_score).sum() >= len(q)
    case.close()


def test_top_queue_keeps_candidates_tied_with_the_bound(oracle, sm):
    """A saturated box: the dives end at 255 n, so the bound equals the score of many
    lowest-resolution candidates, and every one of them is queued (>=, not >)."""
    case = tie_case(oracle, sm, 2, 0.0, 0.0)
    bound, q, sc = check_queue(case, 0.97)
    tied = (sc == bound).sum()
    assert tied > 1 and len(q) == tied
    assert np.all(q["score"] == bound)
    case.close()


def test_top_queue_drops_candidates_at_min_score(oracle, sm):
    """min_score equal to a candidate's score: without dives (bound = min_score) that
    candidate passes >= bound but not > min_score, so it is absent."""
    case = random_case(oracle, sm, seed=5, depth=3, frd=2)
    top = case.top()
    n = len(case.node["high_resolution_point_cloud"])
    sc = np.sort(np.unique(worlds3d.to_score(top["sums"], n)))
    ms = sc[len(sc) // 2]
    bound, q, scores = check_queue(case, NO_DIVES, ms)
    assert (scores == ms).sum() >= 1
    assert not np.any(q["score"] == ms) and len(q) == (scores > ms).sum() > 0
    # with dives, the same min_score
    check_queue(case, 0.97, ms)
    case.close()


# ---- B. the chunked level loop ------------------------------------------------------------
B_WORLDS = ["building", "random", "holes", "gate", "full_submap"]


def make_world(oracle, sm, name):
    if name == "building":
        return building_case(oracle, sm)
    if name == "random":
        return random_case(oracle, sm)
    if name == "holes":
        return tie_case(oracle, sm, 3, 0.02, 0.0)
    if name == "gate":
        return tie_case(oracle, sm, 4, 0.0, 0.5)
    return full_submap_case(oracle, sm)


@pytest.mark.parametrize("name", B_WORLDS)
def test_chunked_level_loop_equals_the_oracle(oracle, sm, name):
    case = make_world(oracle, sm, name)
    want = case.want()
    assert want["found"]
    base, st0 = case.run()
    check_result(base, want)
    same_result(base, case.single()[0])
    assert st0["sweep_trace"][2] == base["leaves_tied"]
    if name in ("holes", "gate"):
        assert base["leaves_tied"] > 1
    for ratio in (0.97, NO_DIVES):
        queue = len(case.top_queue(ratio)[1])
        for chunk in CHUNKS:
            lim = {"dive_ratio": ratio}
            if chunk is not None:
                lim["chunk"] = chunk
            got, st = case.run(**lim)
            tag = (name, ratio, chunk)
            check_result(got, want)
            assert got["leaves_tied"] == base["leaves_tied"], tag
            collects, most, n_best = st["sweep_trace"]
            assert n_best == base["leaves_tied"], tag
            assert st["host_syncs"] == collects + (n_best > 256) + (n_best > 1), tag
            if chunk is not None and queue > chunk:
                assert collects > 1, tag
    case.close()


def test_default_collects_of_realistic_matches(oracle, sm):
    """The collects (1 + continuation sweeps) and the most leaves recorded, under the default
    limits, of the B full-submap job and of the config-3 and config-5 nodes (16 x 2048 and
    64 x 1024 lidar points against a 40 m submap, depth 8), each equal to its single call;
    printed for the record."""
    case = full_submap_case(oracle, sm)
    got, st = case.run()
    check_result(got, case.want())
    print("\nfull-submap job: sweep_trace", st["sweep_trace"])
    case.close()
    o3 = sm.FastCorrelativeScanMatcherOptions3D(min_rotational_score=0.45)
    for name, rings, az, seed in (("config 3", 16, 2048, 40), ("config 5", 64, 1024, 41)):
        hi, lo, sub_hist, wld = synthetic.make_submap3d(seed, 40.0, rings, az, 20.0)
        rng = np.random.RandomState(500 + seed)
        n = synthetic.make_node3d(wld, rng, rings, az, 20.0, seed=7000)
        rng = np.random.RandomState(9)
        init = n["pose"].copy()
        init[:3] += rng.uniform(-1, 1, 3) * [2.0, 2.0, 0.3]
        yaw = 2 * math.atan2(n["pose"][6], n["pose"][3]) + rng.uniform(-1, 1) * math.radians(8)
        init[3:] = [math.cos(yaw / 2), 0, 0, math.sin(yaw / 2)]
        m = sm.FastCorrelativeScanMatcher3D(hi, lo, sub_hist, o3)
        node = sm.TrajectoryNodeData3D(n["cloud"], n["low"], n["hist"])
        res, st = sm.match_batch3d([m], [node], [(0, 0, False, init, IDENT, 0.55)], limits={})
        same_result(res[0], m.match_raw(False, init, IDENT, node, 0.55)[0])
        print("%s node (%d points): sweep_trace %s, nodes_expanded %d" % (
            name, len(n["cloud"]), st["sweep_trace"], st["nodes_expanded"]))
        assert st["sweep_trace"][1] < (1 << 20)
        m.close()


# ---- C. leaf capacity ---------------------------------------------------------------------
@pytest.mark.parametrize("T", [2, 257])
def test_leaf_capacity_at_the_tie_count(oracle, sm, T):
    from cartographer_b200._lib import CsmError
    case = point_case(oracle, sm, T)
    want = case.want()
    assert want["found"]
    top = case.top()
    best = worlds3d.to_score(255, 1)
    assert _bits(top["bound"]) == _bits(best)       # the dives reach the optimum
    base, st = case.run()
    check_result(base, want)
    assert base["leaves_tied"] == T and st["sweep_trace"][1] == T
    for chunk in (None, 1):
        lim = {} if chunk is None else {"chunk": chunk}
        got, st = case.run(leaf_cap=T, **lim)
        same_result(got, base)
        assert st["sweep_trace"][1] == T
        with pytest.raises(CsmError) as e:
            case.run(leaf_cap=T - 1, **lim)
        assert e.value.status == 3 and "capacity" in str(e.value)
        # the same matcher, alone and in a batch, right after the refusal
        same_result(case.single()[0], base)
        res, _ = sm.match_batch3d([case.m], [case.en], [case.job(), case.job()])
        same_result(res[0], base)
        same_result(res[1], base)
    case.close()


# ---- D. the optimal-leaf read-back ----------------------------------------------------------
@pytest.mark.parametrize("T", [0, 1, 2, 255, 256, 257])
def test_inline_read_back_of_tied_leaves(oracle, sm, T):
    case = point_case(oracle, sm, T, seed=T)
    want = case.want()
    assert want["found"] == (T > 0)
    base, st = case.run()
    check_result(base, want)
    if T == 1:
        assert st["host_syncs"] == 1             # unique optimum, one sweep
    for ib in sorted({0, 1, max(0, T - 1), min(T, 256), min(T + 1, 256), 256}):
        for chunk in (None, 1):
            lim = {"inline_best": ib} if chunk is None else {"inline_best": ib, "chunk": chunk}
            got, st = case.run(**lim)
            tag = (T, ib, chunk)
            same_result(got, base)
            collects, most, n_best = st["sweep_trace"]
            assert n_best == T, tag
            if chunk is None:
                assert collects == 1, tag
            assert st["host_syncs"] == collects + (T > ib) + (T > 1), tag
    case.close()


# ---- E. batches ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed_batch(oracle, sm):
    """Matchers of depth 2 .. 7 and several full_resolution_depths on one random world, the
    building, the full-submap job, an empty-histogram matcher and node, and a T = 257 tie;
    jobs repeat matchers and nodes and mix min_scores."""
    rng, hi, lo, node = world(4, 300, n_vox=30000)
    cases = []
    for depth, frd in ((2, 1), (3, 3), (4, 2), (5, 3), (6, 8), (7, 3)):
        od = worlds3d.fast_options(depth=depth, frd=frd, xy=0.7, z=0.3, angular=0.06,
                                   min_low=0.14)
        cases.append(Case3(oracle, sm, hi, lo, od, node, min_score=0.15))
    cases.append(building_case(oracle, sm))
    cases.append(full_submap_case(oracle, sm))
    cases.append(random_case(oracle, sm, seed=7, depth=4, frd=2, hist=np.zeros(0, np.float32),
                             node_hist=np.zeros(0, np.float32)))
    cases.append(point_case(oracle, sm, 257))
    matchers = [c.m for c in cases]
    nodes = [c.en for c in cases]   # cases 0 .. 5 share node 0; nodes 1 .. 5 stay unused
    jobs, wants = [], []
    for k, c in enumerate(cases):
        for ms in ((c.min_score, np.float32(0.12)) if k < 6 else (c.min_score,)):
            jobs.append((k, 0 if k < 6 else k) + c.job(min_score=ms)[2:])
            wants.append(c)
    # repeats: a job of each kind again, and a local job of the full-submap matcher
    jobs += [jobs[3], jobs[12], (7, 7, False, POSE, IDENT, 0.5)]
    wants += [wants[3], wants[12], cases[7]]
    yield cases, matchers, nodes, jobs, wants
    for c in cases:
        c.close()


def _want(c, job):
    _, _, full, npose, spose, ms = job
    if full:
        return c.om.match_full_submap(npose[3:], spose[3:], c.node, ms)
    return c.om.match(npose, spose, c.node, ms)


@pytest.mark.parametrize("workers,limits", [(1, None), (3, None), (24, None), (24, {"chunk": 7}),
                                            (3, {"chunk": 2, "dive_ratio": NO_DIVES})])
def test_mixed_batch_equals_single_calls_and_oracle(sm, mixed_batch, workers, limits):
    cases, matchers, nodes, jobs, wants = mixed_batch
    got, st = sm.match_batch3d(matchers, nodes, jobs, max_concurrency=workers, limits=limits)
    assert len(got) == len(jobs)
    found = 0
    for j, (job, g) in enumerate(zip(jobs, got)):
        mi, ni, full, npose, spose, ms = job
        single, _ = matchers[mi].match_raw(full, npose, spose, nodes[ni], ms)
        same_result(g, single)
        check_result(g, _want(wants[j], job))
        found += g is not None
    assert found >= len(jobs) // 2
    if limits is not None:
        assert st["sweep_trace"][0] > len(jobs)


def test_batch_with_a_refused_job_then_a_right_one(sm, mixed_batch):
    from cartographer_b200._lib import CsmError
    cases, matchers, nodes, jobs, wants = mixed_batch
    with pytest.raises(CsmError) as e:
        sm.match_batch3d(matchers, nodes, jobs, max_concurrency=24, limits={"leaf_cap": 256})
    assert e.value.status == 3
    got, _ = sm.match_batch3d(matchers, nodes, jobs, max_concurrency=24)
    for j, (job, g) in enumerate(zip(jobs, got)):
        check_result(g, _want(wants[j], job))


# ---- E. the sharded queues on a world-1 context ---------------------------------------------
def _raw_cb3d(sm, ctx, matchers, nodes, jobs, owner):
    """csm_cb_batch3d_run into a results array filled with 0xA5 -> (status, raw bytes)."""
    holders = [sm._NodeHolder(n) for n in nodes]
    c_nodes = (sm.CsmNode3D * len(holders))(*[h.c for h in holders])
    c_m = (C.c_void_p * len(matchers))(*[(m._h if m is not None else None) for m in matchers])
    c_jobs = (sm.CsmJob3D * len(jobs))()
    for k, (mi, ni, full, npose, spose, ms) in enumerate(jobs):
        c_jobs[k].matcher_index, c_jobs[k].node_index = mi, ni
        c_jobs[k].full_submap, c_jobs[k].min_score = int(full), float(ms)
        c_jobs[k].global_node_pose = (C.c_double * 7)(*[float(v) for v in npose])
        c_jobs[k].global_submap_pose = (C.c_double * 7)(*[float(v) for v in spose])
    res = (sm.CsmResult3D * len(jobs))()
    C.memset(res, 0xA5, C.sizeof(res))
    own = None if owner is None else np.ascontiguousarray(owner, np.int32)
    st = sm._lib.lib().csm_cb_batch3d_run(
        ctx._h, c_m, C.c_int32(len(matchers)), c_nodes, C.c_int32(len(holders)), c_jobs,
        C.c_int32(len(jobs)), None if own is None else own.ctypes.data_as(C.POINTER(C.c_int32)),
        C.c_int32(0), res, None)
    return st, bytes(res)


def _raw_cb2d(sm, ctx, matchers, clouds, jobs, owner, lin, ang):
    hs = (C.c_void_p * len(matchers))(*[(m._h if m is not None else None) for m in matchers])
    cs = (C.c_void_p * len(clouds))(*[c._h for c in clouds])
    res = np.full(len(jobs) * sm.RESULT2D_DTYPE.itemsize, 0xA5, np.uint8)
    own = None if owner is None else np.ascontiguousarray(owner, np.int32)
    st = sm._lib.lib().csm_cb_batch2d_run(
        ctx._h, hs, C.c_int32(len(matchers)), cs, C.c_int32(len(clouds)),
        jobs.ctypes.data_as(C.c_void_p), C.c_int32(len(jobs)),
        None if own is None else own.ctypes.data_as(C.POINTER(C.c_int32)), C.c_double(lin),
        C.c_double(ang), res.ctypes.data_as(C.c_void_p), None)
    return st, res.tobytes()


def test_sharded_queues_on_a_world_one_context(sm, mixed_batch):
    cases, matchers, nodes, jobs, _ = mixed_batch
    ctx = sm.MultiGpuContext(1, 0, 0)
    try:
        # 3D: equal to the unsharded batch job for job
        want, _ = sm.match_batch3d(matchers, nodes, jobs, max_concurrency=3)
        for owner in (None, np.zeros(len(matchers), np.int32)):
            got, _ = sm.match_batch3d(matchers, nodes, jobs, ctx=ctx, submap_owner=owner)
            for g, w in zip(got, want):
                same_result(g, w)
        assert sm.match_batch3d(matchers, nodes, [], ctx=ctx)[0] == []
        untouched = bytes([0xA5]) * (C.sizeof(sm.CsmResult3D) * len(jobs))
        for owner in ([1] * len(matchers), [-1] * len(matchers)):
            assert _raw_cb3d(sm, ctx, matchers, nodes, jobs, owner) == (1, untouched)
        missing = list(matchers)
        missing[jobs[-1][0]] = None
        assert _raw_cb3d(sm, ctx, missing, nodes, jobs, None) == (1, untouched)
        assert b"an owned submap has no matcher" in sm._lib.lib().csm_last_error_string()

        # 2D
        rng = np.random.RandomState(0)
        ms2, clouds, poses = [], [], []
        opts = sm.FastCorrelativeScanMatcherOptions2D(1.0, 0.3, 5)
        for seed in (11, 12):
            grid, occ = synthetic.make_grid2d(seed, size_cells=200)
            pose = synthetic.random_free_pose(occ, grid, rng, margin_cells=10)
            scan = synthetic.cast_scan(occ, grid, pose, beams=181, max_range=8.0, seed=seed)
            ms2.append(sm.FastCorrelativeScanMatcher2D(grid, opts))
            clouds.append(sm.DeviceCloud(scan))
            poses.append(pose)
        jobs2 = np.zeros(6, sm.JOB2D_DTYPE)
        for k in range(6):
            jobs2[k]["stack_index"], jobs2[k]["cloud_index"] = k % 2, (k // 2) % 2
            jobs2[k]["full_submap"] = int(k == 5)
            jobs2[k]["initial_pose"] = poses[(k // 2) % 2] + [0.2, -0.1, 0.05]
            jobs2[k]["min_score"] = 0.3 + 0.05 * (k % 3)
        want2, _ = sm.match_batch(ms2, clouds, jobs2, 1.0, 0.3)
        assert want2["found"].sum() >= 1
        for owner in (None, np.zeros(2, np.int32)):
            got2, _ = sm.match_batch_sharded(ctx, ms2, clouds, jobs2, 1.0, 0.3, submap_owner=owner)
            assert got2.tobytes() == want2.tobytes()
        got2, _ = sm.match_batch_sharded(ctx, ms2, clouds, jobs2[:0], 1.0, 0.3)
        assert len(got2) == 0
        untouched2 = bytes([0xA5]) * (sm.RESULT2D_DTYPE.itemsize * len(jobs2))
        for owner in ([1, 0], [0, -1]):
            assert _raw_cb2d(sm, ctx, ms2, clouds, jobs2, owner, 1.0, 0.3) == (1, untouched2)
        assert _raw_cb2d(sm, ctx, [ms2[0], None], clouds, jobs2, None, 1.0, 0.3) == (
            1, untouched2)
        assert b"an owned submap has no stack" in sm._lib.lib().csm_last_error_string()
        for m in ms2:
            m.close()
        for c in clouds:
            c.close()
    finally:
        ctx.close()
