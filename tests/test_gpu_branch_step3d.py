"""One level of the 3D branch step (k3_level_begin + k3_expand, with the low-resolution
gate at level 1) over caller-given parents, through csm_branch_step3d: the match's own
launch code.  Children are compared with the oracle's exact child sums (as a sorted
multiset, score bits included); at level 1 the final bound, the recorded leaves with
their gate scores, and the counters are checked against what any execution order allows.
Cases: window clipping (wz = 0, windows smaller than the child step, parents on the last
lattice node), thresholds set exactly equal to child scores, the gate's chunked float sum
and its 0x7fff mask, and frontiers of more than one 65 536-parent chunk."""
import numpy as np
import pytest

from tests import worlds3d

pytestmark = pytest.mark.gpu

RES = 0.1
IDENT = [0, 0, 0, 1, 0, 0, 0]
POSE = [0.03, -0.02, 0.01, 1, 0, 0, 0]
K_CHUNK = 1 << 16


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def setup(oracle, sm, seed, depth, frd, xy, z, n_hi=300, n_lo=60, low_values=None,
          min_low=0.0, angular=0.03, lo_far=0.0):
    rng = np.random.RandomState(seed)
    hi = worlds3d.random_voxels(rng, 3000, 24, RES)
    lo = worlds3d.random_voxels(rng, 400, 6, 0.45, values=low_values)
    low_cloud = worlds3d.random_cloud(rng, n_lo, 2.0)
    if lo_far:   # some low-resolution points outside the low-resolution box
        low_cloud[::7] += np.float32(lo_far)
    node = worlds3d.node_data(worlds3d.random_cloud(rng, n_hi, 2.0), low=low_cloud)
    od = worlds3d.fast_options(depth=depth, frd=frd, xy=xy, z=z, angular=angular,
                               min_low=min_low)
    om, m = worlds3d.make_pair(oracle, sm, hi, lo, od)
    S = len(om.discrete_scans(False, POSE, IDENT, node)[0])
    return rng, od, om, m, node, S


def lattice(h, wxy, wz):
    """The nodes of level h's lattice per axis: -w + k 2^h <= w."""
    return np.arange(-wxy, wxy + 1, 1 << h), np.arange(-wz, wz + 1, 1 << h)


def children(parents, h, wxy, wz):
    """The reference's three `break` loops (:412-430): z outer, y, x inner, a child exists
    while its offset stays inside the window.  -> rows {parent index, scan, x, y, z}."""
    half = 1 << (h - 1)
    out = []
    for i, (s, x, y, z) in enumerate(parents):
        for dz in (0, half):
            if z + dz > wz:
                break
            for dy in (0, half):
                if y + dy > wxy:
                    break
                for dx in (0, half):
                    if x + dx > wxy:
                        break
                    out.append((i, s, x + dx, y + dy, z + dz))
    return np.array(out, np.int64).reshape(-1, 5)


def some_parents(rng, S, h, wxy, wz, n):
    """n random level-h lattice nodes plus every node on the last lattice node of an axis."""
    xs, zs = lattice(h, wxy, wz)
    p = [(int(rng.randint(S)), int(rng.choice(xs)), int(rng.choice(xs)), int(rng.choice(zs)))
         for _ in range(n)]
    p += [(S - 1, xs[-1], int(rng.choice(xs)), int(rng.choice(zs))),
          (0, int(rng.choice(xs)), xs[-1], int(rng.choice(zs))),
          (0, int(rng.choice(xs)), int(rng.choice(xs)), zs[-1]),
          (S - 1, xs[-1], xs[-1], zs[-1])]
    return np.array(p, np.int64)


def records(p, scores):
    from cartographer_b200 import scan_matching as sm
    out = np.zeros(len(p), sm.BNB_NODE3D_DTYPE)
    out["scan"], out["x"], out["y"], out["z"] = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
    out["score"] = scores
    return out


def key(rec):
    return sorted(zip(rec["scan"].tolist(), rec["x"].tolist(), rec["y"].tolist(),
                      rec["z"].tolist(), rec["score"].view(np.uint32).tolist()))


def step(sm, m, node, min_score, h, parents, bound):
    from tests.test_gpu_score3d import profiled
    (out, final, ctr), names = profiled(lambda: m.branch_step(
        False, POSE, IDENT, worlds3d.engine_node(sm, node), min_score, h, parents, bound))
    if len(parents):
        assert "k3_expand" in names
    return out, final, ctr


# ---- k3_expand, level >= 2 ---------------------------------------------------------------
@pytest.mark.parametrize("seed,depth,frd,xy,z,h", [
    (1, 5, 3, 0.7, 0.3, 2), (2, 6, 2, 0.9, 0.0, 3), (3, 5, 9, 0.3, 0.1, 4),
    (4, 7, 3, 1.1, 0.5, 2), (5, 4, 1, 0.2, 0.0, 3), (6, 8, 3, 3.3, 0.7, 6)])
def test_expand_pushes_exact_children(oracle, sm, seed, depth, frd, xy, z, h):
    """Pushed children == the valid children of parents with score >= B whose score is
    > min_score and >= B; B, min_score and some parent scores are exactly child scores."""
    rng, od, om, m, node, S = setup(oracle, sm, seed, depth, frd, xy, z)
    wxy, wz = worlds3d.search_window(od, RES)
    par = some_parents(rng, S, h, wxy, wz, 150)
    kids = children(par, h, wxy, wz)
    _, ks, _ = om.score_candidates(False, POSE, IDENT, node, h - 1, kids[:, 1:])
    order = np.sort(ks)
    B = order[len(order) // 2]
    min_score = order[len(order) // 4]
    choice = np.concatenate([order, [B, B, np.nextafter(B, np.float32(0)),
                                     np.nextafter(B, np.float32(1))]]).astype(np.float32)
    ps = rng.choice(choice, len(par)).astype(np.float32)
    ps[:3] = B
    live = ps >= B
    keep = live[kids[:, 0]] & (ks > min_score) & (ks >= B)
    want = records(kids[keep, 1:], ks[keep])
    got, final, ctr = step(sm, m, node, float(min_score), h, records(par, ps), float(B))
    assert key(got) == key(want)
    assert final.view(np.uint32) == B.view(np.uint32)
    assert ctr == (int(live[kids[:, 0]].sum()), int(live.sum()), 0)
    assert 0 < keep.sum() < len(kids)
    if z == 0.0:
        assert np.all(kids[:, 4] == 0)
    m.close()


# ---- k3_expand, level 1 (leaves and the gate) ----------------------------------------------------
def check_leaves(sm, om, m, od, node, par, B, min_score):
    """Leaves of one level-1 step against what any order of the parents allows: the final
    bound F = max(B, best gate-passing child > min_score of a parent >= B); every such child
    at F is recorded with its exact score and gate bits; every record is a gate-passing
    child > min_score and >= B; counters lie between their values at F and at B."""
    wxy, wz = worlds3d.search_window(od, RES)
    _, ps, _ = om.score_candidates(False, POSE, IDENT, node, 1, par)
    kids = children(par, 1, wxy, wz)
    _, ks, lows = om.score_candidates(False, POSE, IDENT, node, 0, kids[:, 1:])
    assert np.all(ks <= ps[kids[:, 0]])   # the precomputation bound
    B, min_score = np.float32(B), np.float32(min_score)
    gate = lows.astype(np.float64) >= od["min_low_resolution_score"]
    pl = ps[kids[:, 0]]
    ok = (pl >= B) & (ks > min_score) & (ks >= B) & gate
    F = max(B, ks[ok].max()) if ok.any() else B
    got, final, ctr = step(sm, m, node, float(min_score), 1, records(par, ps), float(B))
    assert final.view(np.uint32) == F.view(np.uint32)
    allowed = {}
    for k in np.nonzero(ok)[0]:
        r = (int(kids[k, 1]), int(kids[k, 2]), int(kids[k, 3]), int(kids[k, 4]),
             int(ks[k].view(np.uint32)), int(lows[k].view(np.uint32)))
        allowed[r] = allowed.get(r, 0) + 1
    seen = {}
    for g in got:
        r = (int(g["scan"]), int(g["x"]), int(g["y"]), int(g["z"]),
             int(g["score"].view(np.uint32)), int(g["low"].view(np.uint32)))
        seen[r] = seen.get(r, 0) + 1
    assert all(seen[r] <= allowed.get(r, 0) for r in seen), "a leaf outside the allowed set"
    for r, c in allowed.items():
        if r[4] == int(F.view(np.uint32)):
            assert seen.get(r, 0) == c, "a gate-passing leaf at the final bound is missing"
    n_at = lambda thr: (int((pl >= thr).sum()), int((ps >= thr).sum()),
                        int(((pl >= thr) & (ks > min_score) & (ks >= thr)).sum()))
    lo, hi = n_at(F), n_at(B)
    assert all(lo[i] <= ctr[i] <= hi[i] for i in range(3)), (ctr, lo, hi)
    return F, ks, lows, ok


@pytest.mark.parametrize("seed,depth,frd,xy,z", [
    (11, 4, 2, 0.7, 0.3), (12, 5, 1, 0.5, 0.0), (13, 3, 9, 0.3, 0.2), (14, 6, 3, 0.9, 0.5)])
def test_level_one_leaves_and_bound(oracle, sm, seed, depth, frd, xy, z):
    rng, od, om, m, node, S = setup(oracle, sm, seed, depth, frd, xy, z, min_low=0.3)
    wxy, wz = worlds3d.search_window(od, RES)
    par = some_parents(rng, S, 1, wxy, wz, 120)
    kids = children(par, 1, wxy, wz)
    _, ks, _ = om.score_candidates(False, POSE, IDENT, node, 0, kids[:, 1:])
    order = np.sort(ks)
    for B, min_score in ((order[0], order[0]), (order[len(order) // 2], order[len(order) // 3]),
                         (order[-1], order[len(order) // 2])):
        check_leaves(sm, om, m, od, node, par, B, min_score)
    m.close()


@pytest.mark.parametrize("n_lo", [1, 511, 512, 513, 1025])
def test_gate_at_its_threshold(oracle, sm, n_lo):
    """The gate's ordered float sum in 512-point chunks: n_lo around the chunk size, low
    values with bit 15 set, points outside the low-resolution box.  min_low_resolution_score
    is set exactly to a leaf's gate score chosen so that the best leaf fails the gate and a
    lower one passes at equality."""
    seed = 100 + n_lo
    rng = np.random.RandomState(seed)
    lowv = rng.randint(1, 32768, 5000) | np.where(rng.uniform(size=5000) < 0.5, 0x8000, 0)
    args = dict(seed=seed, depth=4, frd=2, xy=0.5, z=0.2, n_lo=n_lo, lo_far=3.0)
    _, od, om, m, node, S = setup(oracle, sm, low_values=lowv[:400], **args)
    m.close()
    wxy, wz = worlds3d.search_window(od, RES)
    par = some_parents(rng, S, 1, wxy, wz, 80)
    kids = children(par, 1, wxy, wz)
    _, ks, lows = om.score_candidates(False, POSE, IDENT, node, 0, kids[:, 1:])
    best = int(np.argmax(ks))
    lower = [k for k in np.argsort(-ks, kind="stable") if ks[k] < ks[best] and lows[k] > lows[best]]
    thr = lows[lower[0]] if lower else lows[best]
    _, od, om, m, node, S = setup(oracle, sm, low_values=lowv[:400], min_low=float(thr), **args)
    F, ks, lows, ok = check_leaves(sm, om, m, od, node, par, ks.min(), 0.0)
    assert ok.any() and (lows[ok] == thr).any()
    if lower:
        assert F < ks.max()
    m.close()


# ---- chunks: k3_level_begin takes 65 536 parents at a time from the end of the queue -----------------
@pytest.mark.parametrize("n", [K_CHUNK, K_CHUNK + 1, 2 * K_CHUNK + 1])
def test_frontier_larger_than_one_chunk(oracle, sm, n):
    """Dead parents (score below B) fill the queue; live ones sit at its first and last
    places and around the chunk boundaries.  Every live parent is expanded exactly once."""
    rng, od, om, m, node, S = setup(oracle, sm, 7, 4, 2, 0.7, 0.3, n_hi=64)
    wxy, wz = worlds3d.search_window(od, RES)
    h = 2
    base = some_parents(rng, S, h, wxy, wz, 20)
    _, bs, _ = om.score_candidates(False, POSE, IDENT, node, h, base)
    B = np.float32(0.1)
    par = np.repeat(base[:1], n, axis=0)
    ps = np.full(n, np.nextafter(B, np.float32(0)), np.float32)
    spots = sorted({0, 1, K_CHUNK - 1, K_CHUNK, K_CHUNK + 1, 2 * K_CHUNK, n - 2, n - 1} &
                   set(range(n)))
    for j, i in enumerate(spots):
        par[i] = base[j % len(base)]
        ps[i] = bs[j % len(base)]
    live = ps >= B
    kids = children(par[live], h, wxy, wz)
    _, ks, _ = om.score_candidates(False, POSE, IDENT, node, h - 1, kids[:, 1:])
    keep = ks > B
    want = records(kids[keep, 1:], ks[keep])
    got, final, ctr = step(sm, m, node, 0.1, h, records(par, ps), float(B))
    assert key(got) == key(want)
    assert ctr == (len(kids), int(live.sum()), 0)
    assert final == B
    m.close()
