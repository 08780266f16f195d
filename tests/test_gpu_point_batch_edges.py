"""The point-batch processors (voxel_filter.cu, outlier3d.cu, xray.cu and the tables of
point_batch.cuh) at the edges where their kernels go wrong.  After every call each case compares
the device output bit for bit with the CPU restatements (tests/*_oracle.cc): kept indices, voxels
after phases 1 and 2, columns, box and pixels.  Wherever the independent references of
tests/point_batch_refs.py decide the result, the device must equal them too."""
import functools

import numpy as np
import pytest

from tests import outlier_removal_oracle as ORO
from tests import point_batch_refs as R
from tests import voxel_filter_oracle as VFO
from tests import xray_oracle as XO

pytestmark = pytest.mark.gpu

F = np.float32
LAUNCH_SIZES = [1, 31, 32, 33, 255, 256, 257, 65537]


@pytest.fixture(scope="module")
def S():
    from cartographer_b200 import sensor
    return sensor


@pytest.fixture(scope="module")
def P():
    from cartographer_b200 import points_processing
    return points_processing


def _positions(n):
    """Where the deciding point goes: lane 0, lane 31, the last point (a partial warp unless
    n % 32 == 0) and the first point of the last block."""
    return sorted({p for p in (0, 31, n - 1, (n - 1) // 256 * 256) if p < n})


# ---------------------------------------------------------------------------------------------
# Voxel filter
# ---------------------------------------------------------------------------------------------
def _check_vf(S, clouds, res):
    """One device batch against the restatement and, where it decides, the reference."""
    got, st = S.voxel_filter_batch(clouds, res)
    assert st["host_syncs"] == 1 and len(got) == len(clouds)
    for c, r, g in zip(clouds, res, got):
        np.testing.assert_array_equal(g, VFO.voxel_filter(c, r)[0])
        keys, ok = R.cloud_keys(c, r)
        if ok:
            np.testing.assert_array_equal(g, R.voxel_filter(keys)[0])
    return got


def _check_avf(S, clouds, opts):
    got, st = S.adaptive_voxel_filter_batch(clouds, [S.AdaptiveVoxelFilterOptions(*o)
                                                     for o in opts])
    assert st["host_syncs"] == 1 and len(got) == len(clouds)
    searches = []
    for c, o, g in zip(clouds, opts, got):
        want, st = VFO.adaptive_voxel_filter(c, *o)
        np.testing.assert_array_equal(g, want)
        ref, s = R.adaptive_voxel_filter(c, *o)
        if s["decided"]:
            np.testing.assert_array_equal(g, ref)
            assert s["trials"] == st["trials"]
        searches.append(s)
    return got, searches


def _tail(num_voxels=3000, per_voxel=3, y=40.0):
    """Small voxels after a heavy one: their draws have k <= per_voxel, so a wrong shift E
    changes which of their points are kept, where a heavy voxel's own draws would rarely show
    it.  Round robin, so their calls interleave."""
    x = 2.0 * np.arange(num_voxels, dtype=np.float64) + 6.0
    return np.concatenate([np.stack([x + 0.1 * j, np.full(num_voxels, y),
                                     np.full(num_voxels, 0.3)], 1)
                           for j in range(per_voxel)]).astype(F)


@functools.lru_cache(maxsize=None)
def _heavy(n):
    """n points in voxel (0, 0, 0) at resolution 2, then the tail; with the reference's kept
    indices and rejection trace, and the restatement's kept indices."""
    rng = np.random.RandomState(n % 1000)
    cloud = np.vstack([rng.uniform(0.1, 0.9, (n, 3)).astype(F), _tail()])
    keys, ok = R.cloud_keys(cloud, 2.0)
    assert ok
    kept, trace = R.voxel_filter(keys)
    want, st = VFO.voxel_filter(cloud, 2.0)
    np.testing.assert_array_equal(kept, want)
    assert sum(r for _, r in trace) == st["rejections"]
    return cloud, want, trace


# The 63rd, 64th and 65th extra draws of one voxel fall on calls 746 093, 747 943 and 750 882
# (test_point_batch_refs_cpu re-derives them): n points make calls 0 .. n - 2.
@pytest.mark.parametrize("n,extra,last_call", [
    (747944, 63, 746093),      # inside the 64-shift window to the end
    (747945, 64, 747943),      # the 64th extra draw on the heavy voxel's last call
    (747946, 64, 747943),      # one call stepped past the window
    (750883, 64, 747943),      # many calls stepped, none rejecting
    (750884, 65, 750882),      # a rejection in the stepped calls, on the last heavy call
])
def test_rejection_window_boundaries(S, n, extra, last_call):
    cloud, want, trace = _heavy(n)
    assert sum(r for _, r in trace) == extra and trace[-1][0] == last_call
    (got,), _ = S.voxel_filter_batch([cloud], [2.0])
    np.testing.assert_array_equal(got, want)
    # the same cloud in the middle of three
    rng = np.random.RandomState(1)
    a = rng.uniform(-5, 5, (5000, 3)).astype(F)
    b = rng.uniform(-5, 5, (777, 3)).astype(F)
    got = _check_vf(S, [a, cloud, b], [0.5, 2.0, 0.25])
    np.testing.assert_array_equal(got[1], want)


def test_two_rejecting_calls_inside_one_window(S):
    n = 122568
    rng = np.random.RandomState(2)
    cloud = np.vstack([rng.uniform(0.1, 0.9, (n, 3)).astype(F), _tail()])
    keys, ok = R.cloud_keys(cloud, 2.0)
    kept, trace = R.voxel_filter(keys)
    assert ok and trace == [(1310, 1), (122566, 1)]
    got = _check_vf(S, [cloud], [2.0])
    np.testing.assert_array_equal(got[0], kept)


@pytest.mark.parametrize("n", LAUNCH_SIZES)
def test_vf_launch_shapes(S, n):
    """Every point in voxel A but one, in voxel B, at each deciding position: the fixed filter
    must keep it, and the adaptive search reaches two distinct voxels only through it."""
    rng = np.random.RandomState(n)
    for p in _positions(n):
        cloud = rng.uniform(0.05, 0.45, (n, 3)).astype(F)
        cloud[p] = F([3.2, -1.3, 0.2])
        got = _check_vf(S, [cloud], [1.0])
        assert p in got[0]
        far = cloud.copy()
        far[p] = F([30.0, 1.0, 2.0])               # beyond max_range 20
        _check_avf(S, [cloud, far, cloud], [(1.0, 2.0, 20.0), (1.0, 2.0, 20.0),
                                            (1.0, 2.0, 1.0)])


def _many_clouds(nc, seed):
    """Clouds on one shared lattice, so that clouds share voxel keys; cloud 1 (repeated at
    nc - 2) alternates points in voxel (0, 0, 0) with points beyond its max_range, so that its
    kept voxel and the inactive points share the sort key 0."""
    rng = np.random.RandomState(seed)
    clouds = []
    for c in range(nc):
        m = int(rng.randint(1, 40))
        clouds.append((rng.randint(-4, 4, (m, 3)) * 0.3 + 0.01).astype(F))
    near = rng.uniform(-0.2, 0.2, (15, 3))
    far = rng.uniform(-0.2, 0.2, (15, 3)) + 50.0
    clouds[1 % nc] = np.stack([near, far], 1).reshape(-1, 3).astype(F)
    empty = np.zeros((0, 3), F)
    for at in {0, nc // 2, nc - 1}:
        clouds[at] = empty
    if nc >= 4:
        clouds[nc - 2] = clouds[1]                  # the same cloud twice
    return clouds


@pytest.mark.parametrize("nc", [1, 255, 256, 257, 1025])
def test_vf_many_clouds(S, nc):
    clouds = _many_clouds(nc, nc)
    rng = np.random.RandomState(nc + 1)
    res = [float(F(v)) for v in rng.uniform(0.05, 1.0, nc)]
    opts = [(float(F(rng.uniform(0.5, 3))), float(F(rng.randint(0, 40))),
             float(F(rng.uniform(1, 6)))) for _ in range(nc)]
    if nc >= 4:
        res[1] = res[nc - 2] = 0.3
        opts[1] = opts[nc - 2] = (1.0, 1.0, 10.0)   # dense at the first length, 1.0
    got = _check_vf(S, clouds, res)
    agot, _ = _check_avf(S, clouds, opts)
    for at in {0, nc // 2, nc - 1}:
        assert len(got[at]) == 0 and len(agot[at]) == 0
    if nc >= 4:
        assert len(agot[1]) == 1
        np.testing.assert_array_equal(got[1], got[nc - 2])
        np.testing.assert_array_equal(agot[1], agot[nc - 2])


def _empty_key_margin(cloud, search, m):
    """(trial length, ~0-key points) of the trial where counting each ~0-key point as new
    would have reached min_num_points m but the true distinct count does not."""
    for length, distinct in search["counts"]:
        keys, _ = R.cloud_keys(cloud, length)
        c0 = sum(k == R.EMPTY_KEY for k in keys)
        if distinct < m <= distinct + c0 - 1:
            return length, c0
    return None


def _others(d=20):
    return np.stack([3.0 * np.arange(d) + 10.0, np.full(d, 7.0), np.full(d, 3.0)], 1)


def test_empty_key_at_tried_lengths(S):
    d = 20
    trio = [[0, 0, -0.8], [0, 0, -1.0], [0, 0, -1.2]]
    # at max_length 1: (0, 0, -1) itself and two neighbours wrap to ~0
    first = np.vstack([_others(d), trio]).astype(F)
    # and (0, -1, 2^21 - 1) with them (the reference gives up on its tiny lengths)
    wrap = np.vstack([first, [[0, -1.0, 2.0 ** 21 - 1]]]).astype(F)
    # at max_length 1 the trio shares (0, 0, 0); at the first halving, 0.5, it wraps to ~0
    halving = np.vstack([_others(d), [[0, 0, -0.3], [0, 0, -0.35], [0, 0, -0.4]]]).astype(F)
    o = (1.0, d + 2.0, 1e9)
    for cloud, tried, c0_want in ((first, 1.0, 3), (wrap, 1.0, 4), (halving, 0.5, 3)):
        _, (s,) = _check_avf(S, [cloud], [o])
        assert s["decided"] or cloud is wrap
        # one ~0 point counted as new twice would have made that trial dense
        assert _empty_key_margin(cloud, s, F(o[1])) == (F(tried), c0_want)
    _check_avf(S, [first, wrap, halving] * 2, [o] * 6)


@functools.lru_cache(maxsize=None)
def _threshold_cloud():
    """400 distinct points and 20 repeats, so that some min_num_points is never reached."""
    c = np.random.RandomState(12).normal(0, 1.5, (400, 3)).astype(F)
    return np.vstack([c, c[:20]])


def _distinct(cloud, length):
    return len(set(R.cloud_keys(cloud, F(length))[0]))


def test_decide_thresholds_hit_exactly(S):
    cloud = _threshold_cloud()
    L = F(4.0)
    c_first, c_half, c_mid = (_distinct(cloud, L), _distinct(cloud, L / F(2)),
                              _distinct(cloud, (L / F(2) + L) / F(2)))
    assert c_first < c_mid <= c_half
    cases = {
        "first": (float(L), float(c_first), 1e9),             # distinct == m at max_length
        "halving": (float(L), float(c_half), 1e9),            # distinct == m at L / 2
        "bisection": (float(L), float(c_mid), 1e9),           # distinct == m at 3L / 4
        "keep_all": (float(L), float(len(cloud)), 1e9),       # num_active == m: <=, keep all
        "one_below": (float(L), float(len(cloud) - 1), 1e9),
    }
    _, searches = _check_avf(S, [cloud] * len(cases), list(cases.values()))
    s = dict(zip(cases, searches))
    assert all(v["decided"] for v in searches)
    assert s["first"]["trials"] == 1 and s["first"]["length"] == L
    assert s["halving"]["counts"][1] == (L / F(2), c_half) and s["halving"]["trials"] > 2
    assert s["bisection"]["counts"][2] == ((L / F(2) + L) / F(2), c_mid)
    assert s["keep_all"]["trials"] == 0 and s["one_below"]["trials"] > 0


def test_max_range_and_min_num_points_extremes(S):
    cloud = _threshold_cloud()
    opts = [(1.0, 50.0, float("inf")), (1.0, 50.0, -1.0), (1.0, 0.0, 1e9), (1.0, -3.0, 1e9),
            (1.0, 0.0, -1.0), (1.0, -3.0, -1.0)]
    got, searches = _check_avf(S, [cloud] * len(opts), opts)
    assert len(got[0]) > 0 and len(got[1]) == 0 and len(got[4]) == 0 and len(got[5]) == 0
    assert searches[2]["trials"] == 1 and searches[3]["trials"] == 1
    _check_avf(S, [np.zeros((0, 3), F)] * 2, opts[2:4])


@functools.lru_cache(maxsize=None)
def _options_by_path():
    """min_num_points values for _threshold_cloud at max_length 16, one per (halvings, trials)
    path the search takes."""
    cloud = _threshold_cloud()
    by = {}
    for m in range(0, len(cloud) + 2):
        s = R.adaptive_search(cloud, 16.0, float(m), 1e9)
        by.setdefault((s["halvings"], s["trials"]), (16.0, float(m), 1e9))
    return by


def test_clouds_finishing_at_each_trial(S):
    """One batch whose clouds finish at every point of the search: kept whole, at the first
    length, dense after each of the 7 halvings (then bisected), and at the last halving with
    nothing dense."""
    by = _options_by_path()
    paths = sorted(by)
    assert (0, 0) in paths and (0, 1) in paths and (7, 8) in paths
    assert {h for h, t in paths if t > h + 1} == set(range(1, 8))
    _, searches = _check_avf(S, [_threshold_cloud()] * len(paths), [by[p] for p in paths])
    assert [(s["halvings"], s["trials"]) for s in searches] == paths


# ---------------------------------------------------------------------------------------------
# Outlier remover
# ---------------------------------------------------------------------------------------------
def _outlier_device(P, calls, voxel_size, limit):
    """calls: lists of (origin, points) batches, one device call per list and phase.  Returns
    (hits, rays, kept) as the restatement's run() does, and the remover."""
    r = P.OutlierRemover(voxel_size, limit)
    for g in calls:
        r.add_hits([p for _, p in g])
    hits = r.voxels()
    for g in calls:
        r.count_rays([o for o, _ in g], [p for _, p in g])
    rays = r.voxels()
    kept = []
    for g in calls:
        kept += r.filter([p for _, p in g])[0]
    return (hits, rays, kept), r


def _check_outlier(P, calls, voxel_size, limit, need_decided=True):
    batches = [b for g in calls for b in g]
    got, r = _outlier_device(P, calls, voxel_size, limit)
    want = ORO.run(batches, voxel_size, limit)
    for a, b in zip(got[0], want[0]):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(got[1], want[1]):
        np.testing.assert_array_equal(a, b)
    assert len(got[2]) == len(want[2])
    for a, b in zip(got[2], want[2]):
        np.testing.assert_array_equal(a, b)
    ref = R.outlier_removal(batches, voxel_size, limit)
    assert ref["decided"] or not need_decided
    if ref["decided"]:
        for a, b in zip(got[0], R.voxel_arrays(ref["hits"])):
            np.testing.assert_array_equal(a, b)
        for a, b in zip(got[1], R.voxel_arrays(ref["rays"])):
            np.testing.assert_array_equal(a, b)
        for a, b in zip(got[2], ref["kept"]):
            np.testing.assert_array_equal(a, b)
    return got, r, ref


def _axis_rays(rng, num, max_len):
    """Rays from the origin along the six axis directions, ending 0.03 m past a multiple of
    1/8: every sample lands on a voxel centre at 0.125 m, so the reference decides them all."""
    axes = np.concatenate([np.eye(3), -np.eye(3)])
    d = axes[rng.randint(0, 6, num)]
    t = rng.randint(1, int(max_len * 8), num) / 8.0 + 0.03
    return (d * t[:, None]).astype(F)


def test_ray_tiles(P):
    rng = np.random.RandomState(3)
    pts = _axis_rays(rng, 4000, 37.0)
    pts[rng.randint(0, 4000, 200)] = 0.0             # zero-sample rays between long ones
    pts[:4] = F([[37.0, 0, 0], [0, -36.0, 0], [0, 0, 5.0], [1.0, 0, 0]])  # length == some x_k
    pts[4] = F([0, 0, 36.9])                          # 296 samples: more than one tile
    o = F([0, 0, 0])
    lengths = R.ray_lengths(o, pts)
    samples = sum(len(R.ray_samples(0.125, l)) for l in lengths)
    assert samples > 2 ** 19                          # past sm_count * 8 * 256 for any H100
    assert len(R.ray_samples(0.125, F(37.0))) == 296 and len(R.ray_samples(0.125, F(0))) == 0
    got, _, ref = _check_outlier(P, [[(o, pts)]], 0.125, 3.0)
    assert got[1][2].max() > 0 and len(got[2][0]) < len(pts)


def test_keep_at_exact_limit_ties(P):
    o = F([0, 0, 0])
    # voxel 2 along x (0.5 m at 0.25 m) has 1 hit and 3 rays; voxel (0, 2, 0) 2 hits, 1 ray
    pts = F([[0.5, 0, 0], [1.5, 0, 0], [1.75, 0, 0], [2.0, 0, 0],
             [0, 0.5, 0], [0, 0.5, 0], [0, 1.0, 0]])
    never_hit = F([[0, 0, 3.0], [0.5, 0, 0], [0, 0.5, 0]])
    for limit in (3.0, 0.5, 0.0, -1.0, 3.0 + 2.0 ** -40, 0.5 + 2.0 ** -40):
        r = P.OutlierRemover(0.25, limit)
        ref = ORO.Processor(0.25, limit)
        r.add_hits([pts])
        assert ref.add_hits(pts)
        r.count_rays([o], [pts])
        assert ref.count_rays(o, pts)
        for a, b in zip(r.voxels(), ref.voxels()):
            np.testing.assert_array_equal(a, b)
        (k, k2), _ = r.filter([pts, never_hit])
        np.testing.assert_array_equal(k, ref.filter(pts))
        np.testing.assert_array_equal(k2, ref.filter(never_hit))
        want = R.outlier_removal([(o, pts)], 0.25, limit)
        assert want["decided"] and want["rays"][(2, 0, 0)] == (1, 3)
        assert want["rays"][(0, 2, 0)] == (2, 1)
        np.testing.assert_array_equal(k, want["kept"][0])
        assert 0 not in k2                            # no hits: !(0 < limit * 0)
        assert (0 in k) == (3 < limit) and (4 in k) == (1 < 2 * limit)


def _points_of_keys(keys, voxel_size):
    """Points at the centres of the packed voxel keys."""
    k = np.array(keys, np.int64)
    idx = np.stack([(k & 0x3fff) - 8192, ((k >> 14) & 0x3fff) - 8192, (k >> 28) - 8192], 1)
    return (idx * voxel_size).astype(F)


def _chain_keys(slots, z, count_last=3, count_first=2):
    cand = [R.pack(x, y, z) for x in range(-150, 150) for y in range(-150, 150)]
    return R.keys_at_slot(cand, slots, count=count_last) + \
        R.keys_at_slot(cand, slots, slot=0, count=count_first)


def test_outlier_probe_chains_wrap(P):
    vs = 0.25
    c1 = _chain_keys(4096, 3)
    first = _points_of_keys(c1, vs)
    for k in c1[:3]:
        assert R.mix(k) & 4095 == 4095
    # the second call holds 3000 more points: the map grows to 8192 slots and rehashes
    rng = np.random.RandomState(4)
    c2 = _chain_keys(8192, -5)
    for k in c2[:3]:
        assert R.mix(k) & 8191 == 8191
    bulk = (rng.randint(-400, 400, (3000, 3)) * vs).astype(F)
    second = np.vstack([_points_of_keys(c2, vs), bulk])
    o1, o2 = F([0.1, 0.2, 0.3]), F([-0.3, 0.05, 0.2])
    calls = [[(o1, first)], [(o2, second), (o1, first)]]
    got, r, ref = _check_outlier(P, calls, vs, 3.0, need_decided=False)
    assert r.info()["slots"] == R.table_slots(4096, len(first) + len(second) + len(first))
    assert r.info()["slots"] == 8192
    # within one call: chains at the last slot of the initial table and nothing else
    got, r, _ = _check_outlier(P, [[(o1, first), (o2, first[::-1])]], vs, 1.0,
                               need_decided=False)
    assert r.info()["slots"] == 4096


def test_phase1_call_landing_on_half_the_slots(P):
    vs = 0.25
    chain = _chain_keys(4096, 7)
    rng = np.random.RandomState(5)
    rest = set(chain)
    while len(rest) < 2048:
        rest.add(R.pack(*[int(v) for v in rng.randint(-300, 300, 3)]))
    pts = _points_of_keys(sorted(rest), vs)
    assert len(pts) == 2048 and R.table_slots(4096, 0 + 2048) == 4096
    o = F([0.02, -0.01, 0.03])
    r = P.OutlierRemover(vs, 2.0)
    r.add_hits([pts])
    assert r.info() == {"phase": 1, "voxels": 2048, "slots": 4096}   # exactly half full
    got, r2, _ = _check_outlier(P, [[(o, pts)]], vs, 2.0, need_decided=False)
    assert r2.info()["slots"] == 4096
    r.add_hits([pts[:1]])                                # one more incoming: it grows
    assert r.info()["slots"] == 8192 and r.info()["voxels"] == 2048


@pytest.mark.parametrize("nb", [1, 2, 31, 257])
def test_batches_per_call(P, nb):
    rng = np.random.RandomState(nb)
    batches = []
    for b in range(nb):
        o = (rng.randint(-8, 8, 3) / 8.0).astype(F)
        m = int(rng.randint(0, 60)) if b % 5 else 0
        batches.append((o, (o + _axis_rays(rng, m, 6.0)).astype(F)))
    calls = [batches[:max(1, nb // 2)], batches[max(1, nb // 2):]] if nb > 1 else [batches]
    _check_outlier(P, [batches], 0.125, 2.0)
    _check_outlier(P, calls, 0.125, 2.0)


# ---------------------------------------------------------------------------------------------
# X-ray
# ---------------------------------------------------------------------------------------------
def _xray_state(x):
    lo, hi, empty = x.bounding_box()
    px, _ = x.draw()
    return (lo.copy(), hi.copy(), empty), x.voxels(), x.columns(), px


def _check_xray(x, o, batches, vs, factor=1.0, draw=True):
    """The device and the restatement after the same inserts, and the reference over every
    batch inserted so far."""
    lo, hi, empty = x.bounding_box()
    olo, ohi, oempty = o.bounding_box()
    assert empty == oempty
    np.testing.assert_array_equal(x.voxels(), o.voxels())
    yz, sums, counts = x.columns()
    oyz, osums, ocounts = o.columns()
    np.testing.assert_array_equal(yz, oyz)
    np.testing.assert_array_equal(sums.view(np.uint32), osums.view(np.uint32))
    np.testing.assert_array_equal(counts, ocounts)
    if not empty:
        np.testing.assert_array_equal(lo, olo)
        np.testing.assert_array_equal(hi, ohi)
    px = x.draw()[0] if draw else None
    if draw and not empty:
        np.testing.assert_array_equal(px, o.draw())
    ref = R.xray(batches, vs, factor)
    if ref["decided"] and not empty:
        assert ref["box"] == (tuple(lo), tuple(hi))
        np.testing.assert_array_equal(np.array(sorted(ref["voxels"], key=lambda v: v[::-1]),
                                               np.int32).reshape(-1, 3), x.voxels())
        cols = sorted(ref["columns"])
        np.testing.assert_array_equal(np.array(cols, np.int32).reshape(-1, 2), yz)
        np.testing.assert_array_equal(
            np.array([ref["columns"][c][:3] for c in cols], F).view(np.uint32),
            sums.view(np.uint32))
        np.testing.assert_array_equal([ref["columns"][c][3] for c in cols], counts)
        if draw:
            np.testing.assert_array_equal(px, ref["pixels"])
    return ref


@pytest.mark.parametrize("n", LAUNCH_SIZES)
def test_xray_cells_warp_edges(P, n):
    """The point that sets a face of the call's box at lane 0, lane 31, a partial warp and the
    last block; then refused calls whose outside point sits there, which change nothing."""
    rng = np.random.RandomState(n)
    vs = 0.1
    for p in _positions(n):
        pts = (rng.randint(-20, 20, (n, 3)) * vs + 0.02).astype(F)
        col = rng.uniform(0, 1, (n, 3)).astype(F)
        for face, v in ((0, -3.02), (1, 5.02), (2, -4.98)):
            q = pts.copy()
            q[p, face] = v
            x, o = P.XRay(vs), XO.Processor(vs)
            x.insert([q], [col])
            assert o.insert(q, col)
            _check_xray(x, o, [(q, col)], vs)
        x, o = P.XRay(vs), XO.Processor(vs)
        x.insert([pts], [col])
        assert o.insert(pts, col)
        before = _xray_state(x)
        bad = pts.copy()
        bad[p] = F([0, 0, 819.25])                    # cell 8192.5 -> 8193: outside
        from cartographer_b200._lib import CsmError
        with pytest.raises(CsmError):
            x.insert([bad], [col])
        assert not o.insert(bad, col)
        after = _xray_state(x)
        for a, b in zip(before[0], after[0]):
            np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(before[1], after[1])
        for a, b in zip(before[2], after[2]):
            np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(before[3], after[3])
        _check_xray(x, o, [(pts, col)], vs)


def test_xray_one_column_of_70000_points(P):
    rng = np.random.RandomState(7)
    n = 70000
    vs = 0.1
    pts = np.zeros((n, 3), F)
    pts[:, 0] = ((rng.randint(-3000, 3000, n)) * vs + 0.02).astype(F)
    pts[:, 1] = F(0.32)
    pts[:, 2] = F(-0.41)
    col = (rng.uniform(0, 1, (n, 3)) * 10.0 ** rng.randint(-5, 3, (n, 1))).astype(F)
    other = (rng.randint(-5, 5, (300, 3)) * vs + 0.02).astype(F)
    ocol = rng.uniform(0, 1, (300, 3)).astype(F)
    x, o = P.XRay(vs), XO.Processor(vs)
    x.insert([other[:150], pts, other[150:]], [ocol[:150], col, ocol[150:]])
    for p, c in ((other[:150], ocol[:150]), (pts, col), (other[150:], ocol[150:])):
        assert o.insert(p, c)
    ref = _check_xray(x, o, [(other[:150], ocol[:150]), (pts, col), (other[150:], ocol[150:])],
                      vs)
    assert ref["decided"] and ref["columns"][(3, -4)][3] >= n


def test_xray_probe_chains_wrap_in_both_tables(P):
    vs = 0.25
    vcand = [R.pack(x, y, z) for x in range(-100, 100) for y in range(-100, 100)
             for z in (1, 2, 3)]
    vkeys = R.keys_at_slot(vcand, 4096, count=3) + R.keys_at_slot(vcand, 4096, slot=0, count=2)
    ccand = [(y, z) for y in range(-300, 300) for z in range(-300, 300)]
    ckeys = np.array([R.column_key(y, z) for y, z in ccand], np.uint64)
    last = [ccand[i] for i in np.flatnonzero(
        (R.mix_array(ckeys) & np.uint64(4095)) == np.uint64(4095))[:3]]
    zero = [ccand[i] for i in np.flatnonzero(
        (R.mix_array(ckeys) & np.uint64(4095)) == np.uint64(0))[:2]]
    for y, z in last:
        assert R.mix(R.column_key(y, z)) & 4095 == 4095
    first = np.vstack([_points_of_keys(vkeys, vs),
                       np.array([[1, y, z] for y, z in last + zero]) * vs]).astype(F)
    rng = np.random.RandomState(9)
    col = rng.uniform(0, 1, (len(first), 3)).astype(F)
    # the second call grows both tables past 4096 slots; chains at the last slot of 8192
    vk2 = R.keys_at_slot(vcand[::-1], 8192, count=3)
    bulk = (rng.randint(-60, 60, (3000, 3)) * vs).astype(F)
    second = np.vstack([_points_of_keys(vk2, vs), bulk]).astype(F)
    col2 = rng.uniform(0, 1, (len(second), 3)).astype(F)
    x, o = P.XRay(vs), XO.Processor(vs)
    x.insert([first], [col])
    assert o.insert(first, col)
    _check_xray(x, o, [(first, col)], vs)
    x.insert([second], [col2])
    assert o.insert(second, col2)
    _check_xray(x, o, [(first, col), (second, col2)], vs)
    assert R.table_slots(4096, len(first) + len(second)) == 8192


def test_xray_widest_and_smallest_images(P):
    vs = 1.0
    ys = np.arange(-8192, 8192, dtype=np.float64)
    rng = np.random.RandomState(10)
    wide = np.stack([rng.randint(-3, 4, len(ys)), ys, np.zeros(len(ys))], 1).astype(F)
    extra = np.stack([np.full(500, 5.0), rng.randint(-8192, 8192, 500), np.zeros(500)],
                     1).astype(F)
    col = rng.uniform(0, 1, (len(wide), 3)).astype(F)
    x, o = P.XRay(vs), XO.Processor(vs)
    x.insert([wide, extra], [col, None])
    assert o.insert(wide, col) and o.insert(extra, None)
    _check_xray(x, o, [(wide, col), (extra, None)], vs)
    px, _ = x.draw()
    assert px.shape == (1, 16384)
    for pts in (F([[0.3, 0.2, -0.1]]), F([[0.3, 0.2, -0.1], [-2.2, 0.1, 0.2], [4.0, 0, 0]])):
        c = rng.uniform(0, 1, (len(pts), 3)).astype(F)
        x, o = P.XRay(vs), XO.Processor(vs)
        x.insert([pts], [c])
        assert o.insert(pts, c)
        _check_xray(x, o, [(pts, c)], vs)
        assert x.draw()[0].shape == (1, 1)


@pytest.mark.parametrize("factor", [0.0, -0.0, -1.5, -1e300, 1e-300, 7.5, 1e30, 1e300])
def test_xray_saturation_factor_extremes(P, factor):
    rng = np.random.RandomState(11)
    vs = 0.1
    pts = (rng.randint(-6, 6, (600, 3)) * vs + 0.02).astype(F)
    col = rng.uniform(0, 1.2, (600, 3)).astype(F)
    x, o = P.XRay(vs, saturation_factor=factor), XO.Processor(vs, factor)
    x.insert([pts[:300], pts[300:]], [col[:300], None])
    assert o.insert(pts[:300], col[:300]) and o.insert(pts[300:], None)
    ref = _check_xray(x, o, [(pts[:300], col[:300]), (pts[300:], None)], vs, factor)
    assert ref["decided"]


def test_xray_max_count_column_in_the_last_pixel(P):
    """The column with the most voxels is the last pixel (least y and z); black, so every
    saturation shows in the pixel."""
    vs = 1.0
    pts = [[x, -4, -3] for x in range(6)]                          # 6 voxels, the last pixel
    pts += [[x, 0, 0] for x in range(2)] + [[x, 2, -1] for x in range(3)] + [[0, 1, 1]]
    pts += [[x, -2, 1] for x in range(5)]
    pts = F(pts)
    x, o = P.XRay(vs), XO.Processor(vs)
    x.insert([pts])
    assert o.insert(pts)
    ref = _check_xray(x, o, [(pts, None)], vs)
    assert ref["counts"][-1, -1] == 6 == ref["counts"].max()
    assert len(np.unique(ref["pixels"])) >= 5
