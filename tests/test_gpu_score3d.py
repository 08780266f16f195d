"""The 3D fast matcher's scoring kernels against exact sums: k3_score_list (ScoreOct at
every depth) through csm_score_candidates3d, and the lowest-resolution pass, the
rotational filter and the greedy dives through csm_score_top3d, both run by the match's
own launch code.  Every sum is compared for equality with the oracle's ScoreCandidates
hook and every score by its bits; the dives are replayed in numpy.  Ends with matches
whose optimum is tied among many leaves (the host's tie resolution), compared bit for
bit with the oracle, and the depth-1 refusal."""
import ctypes as C

import numpy as np
import pytest

from tests import worlds3d

pytestmark = pytest.mark.gpu

RES = 0.1
IDENT = [0, 0, 0, 1, 0, 0, 0]
POSE = [0.03, -0.02, 0.01, 1, 0, 0, 0]


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def profiled(fn):
    from cartographer_b200 import _lib
    lib = _lib.lib()
    lib.csm_profile_enable(1)
    try:
        out = fn()
        buf = C.create_string_buffer(8192)
        lib.csm_profile_read(buf, 8192)
    finally:
        lib.csm_profile_enable(0)
    return out, {ln.split()[0] for ln in buf.value.decode().splitlines() if ln.strip()}


def world(seed, n_hi, n_lo=60, extent=24, hi_values=None, cloud_center=(0.0, 0.0, 0.0),
          radius=2.0, n_vox=3000):
    rng = np.random.RandomState(seed)
    hi = worlds3d.random_voxels(rng, n_vox, extent, RES, values=hi_values)
    lo = worlds3d.random_voxels(rng, 400, 8, 0.45)
    node = worlds3d.node_data(worlds3d.random_cloud(rng, n_hi, radius, cloud_center),
                              low=worlds3d.random_cloud(rng, n_lo, radius))
    return rng, hi, lo, node


def check_candidates(oracle, sm, om, m, od, node, cand_by_depth):
    """Engine sums and score bits == the oracle's, for every depth's candidate list."""
    rows = [np.concatenate([c, np.full((len(c), 1), d)], axis=1)
            for d, c in cand_by_depth.items()]
    allc = np.concatenate(rows).astype(np.int32)
    (sums, scores), names = profiled(
        lambda: m.score_candidates(False, POSE, IDENT, worlds3d.engine_node(sm, node), allc))
    assert "k3_score_list" in names
    k = 0
    for d, c in cand_by_depth.items():
        ws, wsc, _ = om.score_candidates(False, POSE, IDENT, node, d, c)
        np.testing.assert_array_equal(sums[k:k + len(c)], ws, err_msg="depth %d" % d)
        np.testing.assert_array_equal(scores[k:k + len(c)].view(np.uint32), wsc.view(np.uint32))
        k += len(c)
    return sums


def window_candidates(rng, S, wxy, wz, m):
    """m random candidates of the window plus its eight corners (negative offsets)."""
    c = np.stack([rng.randint(0, S, m), rng.randint(-wxy, wxy + 1, m),
                  rng.randint(-wxy, wxy + 1, m), rng.randint(-wz, wz + 1, m)], axis=1)
    corners = np.array([(S - 1, x, y, z) for z in (-wz, wz) for y in (-wxy, wxy)
                        for x in (-wxy, wxy)])
    return np.concatenate([c, corners]).astype(np.int32)


# ---- k3_score_list / ScoreOct ------------------------------------------------------------
# n_hi straddles the 512-thread CTA stride and the 16-warp reduction; each case also takes
# another depth / full_resolution_depth / window so that the low-resolution indices are
# exercised with odd windows that are not multiples of 2^h (0.0 m: wz = 0).
@pytest.mark.parametrize("n_hi,depth,frd,xy,z", [
    (1, 2, 1, 0.7, 0.3), (31, 3, 2, 0.5, 0.0), (32, 4, 3, 0.9, 0.5), (511, 5, 3, 0.7, 0.3),
    (512, 6, 8, 1.3, 0.5), (513, 7, 3, 1.1, 0.7), (1024, 8, 3, 0.7, 0.3),
    (1537, 5, 1, 0.7, 0.2)])
def test_score_candidates_every_depth(oracle, sm, n_hi, depth, frd, xy, z):
    rng, hi, lo, node = world(n_hi + depth, n_hi)
    od = worlds3d.fast_options(depth=depth, frd=frd, xy=xy, z=z, angular=0.03)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od)
    wxy, wz = worlds3d.search_window(od, RES)
    S = len(om.discrete_scans(False, POSE, IDENT, node)[0])
    sums = check_candidates(oracle, sm, om, m, od, node,
                            {d: window_candidates(rng, S, wxy, wz, 120) for d in range(depth)})
    assert sums.max() > 0
    m.close()


def test_score_candidates_64k_point_node(oracle, sm):
    """A node of 65 536 points (config 5's size): one ulp of score is more than one unit of
    sum there, so only the integer sums can show an off-by-one."""
    rng, hi, lo, node = world(5, 65536)
    od = worlds3d.fast_options(depth=8, frd=3, xy=0.9, z=0.3, angular=0.0)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od)
    wxy, wz = worlds3d.search_window(od, RES)
    check_candidates(oracle, sm, om, m, od, node,
                     {d: window_candidates(rng, 1, wxy, wz, 12) for d in range(8)})
    m.close()


def test_score_candidates_outside_and_saturated(oracle, sm):
    """A cloud wholly outside the grid sums to 0 (score exactly 0.1); one inside a saturated
    box sums to 255 n at every depth."""
    rng = np.random.RandomState(3)
    g = np.stack(np.meshgrid(*[np.arange(-30, 30)] * 3, indexing="ij"), -1).reshape(-1, 3)
    from benchmarks import synthetic
    hi = synthetic.HybridGridSpec(RES, g.astype(np.int32), np.full(len(g), 32767, np.uint16))
    lo = worlds3d.random_voxels(rng, 100, 8, 0.45)
    od = worlds3d.fast_options(depth=5, frd=2, xy=0.7, z=0.3, angular=0.0)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od)
    wxy, wz = worlds3d.search_window(od, RES)
    for center, radius, want in (((0.0, 0.0, 0.0), 1.2, 255), ((60.0, -60.0, 40.0), 1.0, 0)):
        node = worlds3d.node_data(worlds3d.random_cloud(rng, 700, radius, center))
        cand = {d: window_candidates(rng, 1, wxy, wz, 40) for d in range(5)}
        sums = check_candidates(oracle, sm, om, m, od, node, cand)
        assert np.all(sums == want * 700)
        if want == 0:
            _, scores = m.score_candidates(False, POSE, IDENT, worlds3d.engine_node(sm, node),
                                           np.array([[0, 0, 0, 0, 0]], np.int32))
            assert scores[0] == np.float32(0.1)
    m.close()


# ---- k3_score_top, k3_dive, k3_select_scans ------------------------------------------------
def replay_dives(om, node, od, top, min_score, ratio=np.float32(0.97)):
    """k3_dive in numpy: per kept scan the first maximum of its lowest-resolution sums; scans
    with score <= min_score or best < ratio * TopBest (float) are skipped; greedy first-max
    descent over the window-clipped children; leaves above min_score go through the gate.
    -> (bound, candidates scored, gate evaluations)."""
    depth = od["branch_and_bound_depth"]
    wxy, wz = worlds3d.search_window(od, RES)
    n = len(node["high_resolution_point_cloud"])
    nxc = top["nxc"]
    bound, scored, gates = np.float32(min_score), 0, 0
    for s in range(len(top["angle"])):
        flat = top["sums"][s].ravel()
        bi = int(np.argmax(flat))   # first maximum
        best = int(flat[bi])
        if not worlds3d.to_score(best, n) > np.float32(min_score):
            continue
        if np.float32(best) < ratio * np.float32(top["top_best"]):
            continue
        h = depth - 1
        kz, r = divmod(bi, nxc * nxc)
        ky, kx = divmod(r, nxc)
        ox, oy, oz = -wxy + (kx << h), -wxy + (ky << h), -wz + (kz << h)
        leaf = best
        while h > 0:
            half = 1 << (h - 1)
            kids = [(t, ox + (t & 1) * half, oy + ((t >> 1) & 1) * half,
                     oz + ((t >> 2) & 1) * half) for t in range(8)]
            kids = [k for k in kids if k[1] <= wxy and k[2] <= wxy and k[3] <= wz]
            sums, _, _ = om.score_candidates(False, POSE, IDENT, node, h - 1,
                                             [(s, x, y, z) for _, x, y, z in kids])
            b = 0
            for i in range(1, len(kids)):
                if sums[i] > sums[b]:
                    b = i
            scored += len(kids)
            _, ox, oy, oz = kids[b]
            leaf = int(sums[b])
            h -= 1
        score = worlds3d.to_score(leaf, n)
        if score > np.float32(min_score):
            gates += 1
            _, _, low = om.score_candidates(False, POSE, IDENT, node, 0, [(s, ox, oy, oz)])
            if float(low[0]) >= od["min_low_resolution_score"]:
                bound = max(bound, score)
    return bound, scored, gates


def check_top(sm, om, m, od, node, min_score):
    """csm_score_top3d of a local match: every lowest-resolution sum == the oracle's (scan
    major, then z, y, x), TopBest == their maximum, angle indices increasing."""
    top, names = profiled(lambda: m.score_top(False, POSE, IDENT,
                                              worlds3d.engine_node(sm, node), min_score))
    S, nxc, nzc = len(top["angle"]), top["nxc"], top["nzc"]
    step = 1 << (od["branch_and_bound_depth"] - 1)
    wxy, wz = worlds3d.search_window(od, RES)
    assert nxc == (2 * wxy + step) // step and nzc == (2 * wz + step) // step
    if S:
        assert "k3_score_top" in names and "k3_dive" in names
        kz, ky, kx = np.meshgrid(np.arange(nzc), np.arange(nxc), np.arange(nxc), indexing="ij")
        lat = np.stack([-wxy + kx.ravel() * step, -wxy + ky.ravel() * step,
                        -wz + kz.ravel() * step], axis=1)
        cand = np.concatenate([np.concatenate([np.full((len(lat), 1), s), lat], axis=1)
                               for s in range(S)])
        want, _, _ = om.score_candidates(False, POSE, IDENT, node, od["branch_and_bound_depth"] - 1,
                                         cand)
        np.testing.assert_array_equal(top["sums"].ravel(), want)
        assert top["top_best"] == top["sums"].max()
        assert np.all(np.diff(top["angle"]) > 0)
    return top


@pytest.mark.parametrize("seed,depth,frd,xy,z,min_score,saturated", [
    (1, 5, 3, 0.7, 0.3, 0.15, False), (2, 6, 2, 0.9, 0.0, 0.2, False),
    (3, 4, 9, 0.5, 0.5, 0.1, False), (4, 5, 3, 0.7, 0.3, 0.15, False),
    (5, 3, 1, 0.3, 0.2, 0.12, 1.4)])
def test_top_pass_and_dives_vs_replay(oracle, sm, seed, depth, frd, xy, z, min_score,
                                      saturated):
    """Every lowest-resolution sum of the kept scans, TopBest, and the dive bound and
    counters of a numpy replay.  The saturated grids (a cloud of radius `saturated` in a
    box whose voxels are all 255 or empty) make the top sums of a scan tie, so the first
    maximum matters."""
    rng, hi, lo, node = world(seed, 300, hi_values=32767 if saturated else None, n_vox=30000)
    if saturated:
        node["high_resolution_point_cloud"] = worlds3d.random_cloud(rng, 300, saturated)
    od = worlds3d.fast_options(depth=depth, frd=frd, xy=xy, z=z, angular=0.06, min_low=0.14)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od)
    top = check_top(sm, om, m, od, node, min_score)
    assert len(top["angle"]) >= 3
    bound, scored, gates = replay_dives(om, node, od, top, min_score)
    assert top["bound"].view(np.uint32) == bound.view(np.uint32)
    assert top["counters"] == (scored, gates)
    assert gates > 0
    if saturated:
        flat = top["sums"].reshape(len(top["angle"]), -1)
        assert any((f == f.max()).sum() > 1 for f in flat)
    m.close()


def _filter_node(rng, far_range, hist_n=24, empty_hist=False):
    near = worlds3d.random_cloud(rng, 12, 1.0)
    far = np.array([[far_range * 0.6, far_range * 0.8, 0.0]], np.float32)
    cloud = np.concatenate([near, far])
    hist = np.zeros(0, np.float32) if empty_hist else rng.uniform(0, 5, hist_n).astype(np.float32)
    return worlds3d.node_data(cloud, low=near, hist=hist)


@pytest.mark.parametrize("far_range,min_angles", [(20.0, 1025), (35.0, 2049)])
def test_rotational_filter_beyond_one_chunk(oracle, sm, far_range, min_angles):
    """Full-submap nodes of 20 m and 35 m range have more than 1024 / 2048 angles, so
    k3_select_scans compacts in two / three chunks.  With every angle kept the angle
    indices are 0 .. A-1; with min_rotational_score equal to a kept score exactly the kept
    set is the angles whose score is not below it; a threshold above 1 keeps nothing."""
    rng = np.random.RandomState(int(far_range))
    hi = worlds3d.random_voxels(rng, 2000, 20, RES)
    lo = worlds3d.random_voxels(rng, 200, 6, 0.45)
    node = _filter_node(rng, far_range)
    hist = rng.uniform(0, 5, 24).astype(np.float32)
    rot = [0, 0, 0, 0.96, 0, 0, 0.28]
    od = worlds3d.fast_options(depth=8, frd=3, min_rot=0.0)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od, hist=hist)
    en = worlds3d.engine_node(sm, node)
    top = m.score_top(True, rot, IDENT, en, 0.1)
    A = len(top["angle"])
    assert A >= min_angles
    np.testing.assert_array_equal(top["angle"], np.arange(A))
    _, _, wr = om.discrete_scans(True, rot, IDENT, node)
    np.testing.assert_array_equal(top["rot"].view(np.uint32), wr.view(np.uint32))
    assert top["top_best"] == top["sums"].max()
    all_rot = top["rot"]
    thr = np.sort(all_rot)[A // 3]
    m.close()
    od2 = dict(od, min_rotational_score=float(thr))
    om2, m2 = worlds3d.make_pair(oracle, sm, hi, lo, od2, hist=hist)
    top2 = m2.score_top(True, rot, IDENT, en, 0.1)
    np.testing.assert_array_equal(top2["angle"], np.nonzero(~(all_rot < thr))[0])
    assert thr in top2["rot"]
    gc, gp, gr = m2.discretize(True, rot, IDENT, en)
    wc, wp, wr = om2.discrete_scans(True, rot, IDENT, node)
    np.testing.assert_array_equal(gr.view(np.uint32), wr.view(np.uint32))
    np.testing.assert_array_equal(gp.view(np.uint32), wp.view(np.uint32))
    np.testing.assert_array_equal(gc, wc)
    np.testing.assert_array_equal(top2["rot"].view(np.uint32), wr.view(np.uint32))
    m2.close()
    od3 = dict(od, min_rotational_score=1.5)
    _, m3 = worlds3d.make_pair(oracle, sm, hi, lo, od3, hist=hist)
    top3 = m3.score_top(True, rot, IDENT, en, 0.1)
    assert len(top3["angle"]) == 0 and top3["counters"] == (0, 0)
    assert m3.MatchFullSubmap(rot[3:], IDENT[3:], en, 0.1) is None
    m3.close()


def test_rotational_filter_empty_histogram(oracle, sm):
    """Without histograms every rotational score is 1 (k3_fill); min_rotational_score 1
    keeps every angle."""
    rng = np.random.RandomState(9)
    hi = worlds3d.random_voxels(rng, 2000, 20, RES)
    lo = worlds3d.random_voxels(rng, 200, 6, 0.45)
    node = _filter_node(rng, 3.0, empty_hist=True)
    od = worlds3d.fast_options(depth=4, frd=2, xy=0.4, z=0.2, angular=0.3, min_rot=1.0,
                               min_low=0.12)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od, hist=np.zeros(0, np.float32))
    top = check_top(sm, om, m, od, node, 0.12)
    A = len(top["angle"])
    assert A > 10
    np.testing.assert_array_equal(top["angle"], np.arange(A))
    assert np.all(top["rot"] == np.float32(1.0))
    _, _, wr = om.discrete_scans(False, POSE, IDENT, node)
    assert len(wr) == A
    bound, scored, gates = replay_dives(om, node, od, top, 0.12)
    assert top["bound"].view(np.uint32) == bound.view(np.uint32)
    assert top["counters"] == (scored, gates)
    m.close()


# ---- tie resolution on the host (Run3D), end to end ------------------------------------------
def _saturated_world(rng, extent, lo_extent, holes=0.0):
    """A saturated high-resolution box, with a fraction `holes` of its 2x2x2 blocks empty,
    and a random low-resolution box."""
    g = np.stack(np.meshgrid(*[np.arange(-extent, extent)] * 3, indexing="ij"), -1).reshape(-1, 3)
    nb = extent
    empty = rng.uniform(size=(nb, nb, nb)) < holes
    b = (g + extent) >> 1
    keep = ~empty[b[:, 0], b[:, 1], b[:, 2]]
    from benchmarks import synthetic
    hi = synthetic.HybridGridSpec(RES, g[keep].astype(np.int32),
                                  np.full(keep.sum(), 32767, np.uint16))
    gl = np.stack(np.meshgrid(*[np.arange(-lo_extent, lo_extent)] * 3, indexing="ij"),
                  -1).reshape(-1, 3)
    lo = synthetic.HybridGridSpec(0.45, gl.astype(np.int32),
                                  rng.randint(1, 32768, len(gl)).astype(np.uint16))
    return hi, lo


@pytest.mark.parametrize("seed,holes,xy,z,angular,min_low,expect", [
    (1, 0.0, 0.2, 0.1, 0.0, 0.0, "few"),        # one scan, 75 tied leaves
    (2, 0.0, 0.4, 0.2, 0.12, 0.0, "many"),      # > 256 tied leaves (kInlineBest)
    (3, 0.02, 0.3, 0.1, 0.06, 0.0, "any"),      # holes: ancestors differ
    (4, 0.0, 0.3, 0.1, 0.06, 0.5, "any"),       # a strict gate rejects some ties
])
def test_tied_optimum_resolved_as_reference(oracle, sm, seed, holes, xy, z, angular, min_low,
                                            expect):
    rng = np.random.RandomState(seed)
    hi, lo = _saturated_world(rng, 26, 4, holes)
    cloud = worlds3d.random_cloud(rng, 40, 0.8)
    node = worlds3d.node_data(cloud, low=worlds3d.random_cloud(rng, 30, 1.5))
    od = worlds3d.fast_options(depth=3, frd=2, xy=xy, z=z, angular=angular, min_low=min_low)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od)
    want = om.match(POSE, IDENT, node, 0.2)
    got = m.Match(POSE, IDENT, worlds3d.engine_node(sm, node), 0.2)
    st = m.last_stats
    assert (got is not None) == want["found"]
    assert want["found"]
    assert got["score"] == want["score"]
    assert got["best_scan_index"] == want["best_scan_index"]
    assert got["best_offset"] == (want["best_x"], want["best_y"], want["best_z"])
    np.testing.assert_array_equal(got["pose_estimate"], want["pose"])
    assert got["low_resolution_score"] == want["low_resolution_score"]
    assert st["leaves_tied"] > 1
    if expect == "few":
        assert 1 < st["leaves_tied"] <= 256 and st["host_tie_resolves"] >= 1
    elif expect == "many":
        assert st["leaves_tied"] > 256 and st["host_tie_resolves"] >= 1
    m.close()


def test_depth_one_is_refused(oracle, sm):
    """branch_and_bound_depth == 1 (allowed by the reference) returns CSM_E_INVALID."""
    from cartographer_b200._lib import CsmError
    rng, hi, lo, node = world(1, 20)
    od = worlds3d.fast_options(depth=1, frd=1)
    _, m = worlds3d.make_pair(oracle, sm, hi, lo, od)
    with pytest.raises(CsmError) as e:
        m.Match(POSE, IDENT, worlds3d.engine_node(sm, node), 0.1)
    assert e.value.status == 1
    assert "branch_and_bound_depth == 1 is not supported" in str(e.value)
    m.close()
