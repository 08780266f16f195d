"""The real-time matchers' kernels candidate by candidate, at the edges where they go wrong.

k_rt_match (rt2d.cu) has three forms — the TMA-staged box, global gathers and TSDF — each
with 1 and 4 accumulators per lane; k_rt3_match (rt3d.cu) has one.  Every case here runs the
matches' own planning and launch code through the score hooks csm_rt_scores2d /
csm_rt_scores3d and compares

  * every candidate's weighted float32 score, bit for bit, with the oracle's Match (the
    scores max_element / the `score > best_score` loop sees), and
  * the match results (score bits, pose doubles, best indices, candidates scored),

and checks through csm_profile_read which kernel form ran.  The form a 2D batch gets is
restated below from PrepareJob's box arithmetic, so the tests also pin the planner.
Reference: real_time_correlative_scan_matcher_2d.cc:38-176,
real_time_correlative_scan_matcher_3d.cc:34-117."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic

pytestmark = pytest.mark.gpu

RES = 0.0625          # a power of two: cell centres, windows and ranges are exact
KERNEL = {"tma": "k_rt_match_tma", "gather": "k_rt_match_gather", "tsdf": "k_rt_match_tsdf"}


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def profiled(fn):
    """fn() with the per-kernel profile on -> (result, names of the kernels that ran)."""
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


def bits(x):
    return np.array(x, np.float32).view(np.uint32)


# ---- grids and clouds --------------------------------------------------------------------
def rand_cells(rng, ny, nx, unknown=0.25):
    cells = rng.randint(1, 32768, size=(ny, nx)).astype(np.uint16)
    cells[rng.uniform(size=(ny, nx)) < unknown] = 0
    return cells


def pgrid(cells, max_x=10.0, max_y=10.0, res=RES):
    return synthetic.GridSpec(cells, res, max_x, max_y)


def tgrid(rng, ny, nx, truncation=0.3, max_weight=10.0, max_x=10.0, max_y=10.0):
    tsd = rng.randint(1, 32768, size=(ny, nx)).astype(np.uint16)
    wgt = rng.randint(1, 32768, size=(ny, nx)).astype(np.uint16)
    unknown = rng.uniform(size=(ny, nx)) < 0.3
    tsd[unknown] = 0
    wgt[unknown] = 0
    wgt[rng.uniform(size=(ny, nx)) < 0.05] = 0
    return synthetic.TSDFGridSpec(tsd, wgt, RES, max_x, max_y, truncation, max_weight)


def world_of_cell(grid, ix, iy):
    """Centre of cell (ix, iy): index x <- world y, index y <- world x (map_limits.h:69-76)."""
    return (grid.max_x - (np.asarray(iy) + 0.5) * grid.resolution,
            grid.max_y - (np.asarray(ix) + 0.5) * grid.resolution)


def init_at(grid, ix, iy):
    wx, wy = world_of_cell(grid, ix, iy)
    return np.array([float(wx), float(wy), 0.0])


def cloud_at_cells(grid, init, cells):
    """Sensor-frame points (yaw 0) at the centres of the given (ix, iy) cells."""
    cells = np.asarray(cells, np.int64).reshape(-1, 2)
    wx, wy = world_of_cell(grid, cells[:, 0], cells[:, 1])
    return np.stack([wx - init[0], wy - init[1], np.zeros(len(cells))], 1).astype(np.float32)


def disk_cloud(rng, n, radius):
    r = radius * np.sqrt(rng.uniform(size=n))
    a = rng.uniform(-math.pi, math.pi, n)
    return np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-0.1, 0.1, n)], 1).astype(np.float32)


# ---- PrepareJob's box, restated -------------------------------------------------------------
def box_dims(nx, ny):
    pitch = (nx + 7) // 8 * 8
    bw = min(pitch, 256)
    bh = max(1, min(ny, 256, 100 * 1024 // (bw * 2)))
    return bw, bh


def job_fits(grid, cloud, init, lin_cells):
    """(fits the staged box, reach width after the 8-cell alignment, reach height) of one job
    as PrepareJob plans it (rt2d.cu): the cell of the initial translation +- (ceil(max range /
    resolution) + lin + 3), clipped to the grid; a reach that misses the grid fits any box."""
    ny, nx = grid.cells.shape if hasattr(grid, "cells") else grid.tsd_cells.shape
    bw, bh = box_dims(nx, ny)
    c, s = np.float32(math.cos(init[2])), np.float32(math.sin(init[2]))
    x = c * cloud[:, 0] - s * cloud[:, 1]
    y = s * cloud[:, 0] + c * cloud[:, 1]
    msr = max(float(np.float32(3.0 * grid.resolution)),
              float(np.sqrt(x * x + y * y, dtype=np.float32).max()))
    tx, ty = float(np.float32(init[0])), float(np.float32(init[1]))
    fx = (grid.max_y - ty) / grid.resolution - 0.5
    fy = (grid.max_x - tx) / grid.resolution - 0.5
    R = math.ceil(msr / grid.resolution) + lin_cells + 3
    rx0, rx1 = max(0, math.floor(fx - R)), min(nx - 1, math.ceil(fx + R))
    ry0, ry1 = max(0, math.floor(fy - R)), min(ny - 1, math.ceil(fy + R))
    if rx1 < rx0 or ry1 < ry0:
        return True, 0, 0
    w, h = rx1 - (rx0 & ~7) + 1, ry1 - ry0 + 1
    return w <= bw and h <= bh, w, h


# ---- the 2D check ---------------------------------------------------------------------------
def oracle_grid(oracle, grid):
    return oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)


def oracle_2d(oracle, grid, cloud, init, lin, ang, w_t, w_r):
    if hasattr(grid, "tsd_cells"):
        a = (grid.tsd_cells, grid.weight_cells, grid.resolution, grid.max_x, grid.max_y,
             grid.truncation_distance, grid.max_weight, cloud, init, lin, ang, w_t, w_r)
        return oracle.rt2d_scores_tsdf(*a), oracle.rt2d_match_tsdf(*a)
    og = oracle_grid(oracle, grid)
    a = (og, cloud, init, lin, ang, w_t, w_r)
    return oracle.rt2d_scores(*a), oracle.rt2d_match(*a)


def check_result(r, want):
    assert bits(r.score) == bits(want["score"]), (r.score, want["score"])
    np.testing.assert_array_equal(np.array(r.pose_estimate[:]), want["pose"])
    assert (r.best_scan_index, r.best_x_offset, r.best_y_offset) == (
        want["best_scan_index"], want["best_x_offset"], want["best_y_offset"])
    assert r.candidates_scored == want["candidates_scored"]
    assert r.num_scans == want["num_scans"]


def expected_form(grid, clouds, inits, lin_cells):
    if hasattr(grid, "tsd_cells"):
        return "tsdf"
    return "tma" if all(job_fits(grid, c, i, lin_cells)[0] for c, i in zip(clouds, inits)) \
        else "gather"


def check_2d(oracle, sm, grid, clouds, inits, lin_cells, ang, w_t=0.1, w_r=0.1, form=None,
             dg=None):
    """ScoresBatch against the oracle, candidate by candidate and result by result; the form
    that ran must be `form` (default: the restated plan's).  Returns (results, scores)."""
    lin = lin_cells * grid.resolution
    rt = sm.RealTimeCorrelativeScanMatcher2D(
        sm.RealTimeCorrelativeScanMatcherOptions(lin, ang, w_t, w_r))
    own = dg is None
    dg = sm.RealTimeGrid2D(grid) if own else dg
    try:
        (res, scores), names = profiled(lambda: rt.ScoresBatch(inits, clouds, dg))
    finally:
        if own:
            dg.close()
    want_form = expected_form(grid, clouds, inits, lin_cells)
    assert form is None or form == want_form, (form, want_form)
    assert KERNEL[want_form] in names, (want_form, names)
    assert not (set(KERNEL.values()) - {KERNEL[want_form]}) & names, names
    for j in range(len(clouds)):
        want_scores, want = oracle_2d(oracle, grid, clouds[j], inits[j], lin, ang, w_t, w_r)
        assert len(scores[j]) == len(want_scores), j
        np.testing.assert_array_equal(bits(scores[j]), bits(want_scores), err_msg="job %d" % j)
        check_result(res[j], want)
    return res, scores


def match_batch(oracle, sm, grid, clouds, inits, lin_cells, ang, w_t=0.1, w_r=0.1):
    """The public batch path alone (MatchBatch) against the oracle's Match."""
    lin = lin_cells * grid.resolution
    rt = sm.RealTimeCorrelativeScanMatcher2D(
        sm.RealTimeCorrelativeScanMatcherOptions(lin, ang, w_t, w_r))
    dg = sm.RealTimeGrid2D(grid)
    try:
        (_, _, st), names = profiled(lambda: rt.MatchBatch(inits, clouds, dg))
    finally:
        dg.close()
    for j in range(len(clouds)):
        check_result(rt.last_results[j], oracle_2d(oracle, grid, clouds[j], inits[j], lin, ang,
                                                    w_t, w_r)[1])
    return names, st


# ==== 2D: forms x accumulators x point counts x windows =======================================
POINT_COUNTS = (1, 31, 32, 33, 1081)      # the 32-point shuffle chunks
LIN_CELLS = (0, 1, 2, 3, 5, 8)            # 1 accumulator; 4 with 2, 4, partial; three r0 passes


def _batch(rng, grid, far):
    """Jobs of every point count and different ranges (so different num_scans) in one batch;
    `far` adds a 12 m point to the last job, whose reach then exceeds the staged box."""
    clouds, inits = [], []
    for k, n in enumerate(POINT_COUNTS):
        clouds.append(disk_cloud(rng, n, 0.5 + 0.9 * k))
        inits.append(np.array([rng.uniform(-1.0, 2.0), rng.uniform(-4.0, -1.0),
                               rng.uniform(-0.3, 0.3)]))
    if far:
        clouds[-1] = np.concatenate([clouds[-1], np.array([[12.0, 0.5, 0.0]], np.float32)])
    return clouds, inits


@pytest.mark.parametrize("lin_cells", LIN_CELLS)
@pytest.mark.parametrize("form", ["tma", "gather", "tsdf"])
def test_forms_point_counts_and_windows(oracle, sm, form, lin_cells):
    """Every form and accumulator count (per_scan <= 32 -> 1, else 4) over point counts 1, 31,
    32, 33 and 1081 in one launch, with one rotated scan per job and with many."""
    rng = np.random.RandomState(100 + 7 * lin_cells + {"tma": 0, "gather": 1, "tsdf": 2}[form])
    ny, nx = 300, 400    # box 256 x 200: short scans fit it, a 12 m point does not
    grid = tgrid(rng, ny, nx) if form == "tsdf" else pgrid(rand_cells(rng, ny, nx))
    for ang in (0.0, 0.1):
        clouds, inits = _batch(rng, grid, far=form == "gather")
        res, _ = check_2d(oracle, sm, grid, clouds, inits, lin_cells, ang,
                          form=None if form == "tsdf" else form)
        scans = {r.num_scans for r in res}
        assert scans == {1} if ang == 0.0 else len(scans) > 1


def test_unweighted_scores_are_float64_sums(oracle, sm):
    """w_t = w_r = 0: the weight is exp(-0) = 1, so each score is the ordered float32 sum of the
    probabilities over n; it lies within n * 2^-24 (relative) of the float64 sum of the same
    cells, read from the oracle's discrete scans."""
    rng = np.random.RandomState(7)
    grid = pgrid(rand_cells(rng, 200, 240))
    og = oracle_grid(oracle, grid)
    lin_cells, ang = 2, 0.2
    clouds, inits = [disk_cloud(rng, 1081, 3.0), disk_cloud(rng, 33, 1.0)], \
        [np.array([3.0, -2.0, 0.4]), np.array([1.0, -1.0, -1.0])]
    _, scores = check_2d(oracle, sm, grid, clouds, inits, lin_cells, ang, 0.0, 0.0, form="tma")
    table = oracle.value_to_cost_table(og.min_cost, og.max_cost)
    min_p = np.float32(oracle.constant(0))
    cells = grid.cells & 0x7fff
    prob = np.where(cells == 0, np.float32(1) - np.float32(og.max_cost),
                    np.float32(1) - table[cells]).astype(np.float64)
    w = 2 * lin_cells + 1
    for j, (cloud, init) in enumerate(zip(clouds, inits)):
        fe = oracle.frontend2d(og, cloud, init, False, lin_cells * RES, ang, rt_mode=True)
        ds = fe["discrete_scans"]
        n = len(cloud)
        ref = []
        for s in range(fe["num_scans"]):
            for xo in range(-lin_cells, lin_cells + 1):
                for yo in range(-lin_cells, lin_cells + 1):
                    x, y = ds[s, :, 0] + xo, ds[s, :, 1] + yo
                    inside = (x >= 0) & (x < grid.num_x) & (y >= 0) & (y < grid.num_y)
                    p = np.full(n, float(min_p))
                    p[inside] = prob[y[inside], x[inside]]
                    ref.append(p.sum() / n)
        ref = np.array(ref)
        assert len(ref) == len(scores[j]) == fe["num_scans"] * w * w
        np.testing.assert_array_less(np.abs(scores[j] - ref), n * 2.0 ** -24 * np.abs(ref) + 1e-30)


# ==== 2D: the staged box's edges ==============================================================
EDGES = ["width_bw", "width_bw_plus_1", "height_bh", "height_bh_plus_1", "overhang",
         "nx_not_multiple_of_8", "grid_smaller_than_box", "one_cell"]


def _edge_case(name):
    """(grid, clouds, inits, lin_cells, form) at one box edge, chosen with the restated plan."""
    rng = np.random.RandomState(200 + EDGES.index(name))
    lin_cells = 2
    if name in ("width_bw", "width_bw_plus_1"):
        # R = ceil(7.625 / RES) + 2 + 3 = 127: raw reach 255 cells; x0 = fx - 127 is 1 (2) past
        # an 8-cell boundary, so the aligned reach is exactly bw = 256 (257)
        grid = pgrid(rand_cells(rng, 150, 600))
        fx = 256 if name == "width_bw" else 257
        init = init_at(grid, fx, 75)
        cloud = np.concatenate([disk_cloud(rng, 200, 3.0),
                                np.array([[0.0, 7.625, 0.0], [7.0, 1.0, 0.0]], np.float32)])
        want = (True, 256) if name == "width_bw" else (False, 257)
        fits, w, _ = job_fits(grid, cloud, init, lin_cells)
        assert (fits, w) == want
    elif name in ("height_bh", "height_bh_plus_1"):
        # R = ceil(6.5625 / RES) + 5 = 110, clipped at row 0: height fy + 111 = 200 (201)
        grid = pgrid(rand_cells(rng, 400, 400))
        fy = 89 if name == "height_bh" else 90
        init = init_at(grid, 200, fy)
        cloud = np.concatenate([disk_cloud(rng, 200, 3.0),
                                np.array([[6.5625, 0.0, 0.0]], np.float32)])
        fits, _, h = job_fits(grid, cloud, init, lin_cells)
        assert (fits, h) == ((True, 200) if name == "height_bh" else (False, 201))
    elif name == "overhang":
        # box at x0 = 240, 256 wide, over a 300-cell row: the TMA fills past the edge with 0
        grid = pgrid(rand_cells(rng, 150, 300))
        init = init_at(grid, 250, 70)
        cloud = disk_cloud(rng, 300, 1.5)
    elif name == "nx_not_multiple_of_8":
        grid = pgrid(rand_cells(rng, 61, 203))
        init = init_at(grid, 150, 30)
        cloud = disk_cloud(rng, 300, 4.0)
    elif name == "grid_smaller_than_box":
        grid = pgrid(rand_cells(rng, 10, 20))
        init = init_at(grid, 10, 5)
        cloud = disk_cloud(rng, 100, 1.5)
    else:  # one_cell
        grid = pgrid(np.array([[1234]], np.uint16))
        init = init_at(grid, 0, 0)
        cloud = disk_cloud(rng, 40, 0.2)
    fits = job_fits(grid, cloud, init, lin_cells)[0]
    return grid, [cloud], [init], lin_cells, "tma" if fits else "gather"


@pytest.mark.parametrize("name", EDGES)
def test_box_edges(oracle, sm, name):
    grid, clouds, inits, lin_cells, form = _edge_case(name)
    want = {"width_bw_plus_1": "gather", "height_bh_plus_1": "gather"}.get(name, "tma")
    assert form == want
    check_2d(oracle, sm, grid, clouds, inits, lin_cells, 0.05, form=form)


# ==== 2D: batches ==============================================================================
def test_ctas_span_jobs_with_different_boxes(oracle, sm):
    """40 short-range jobs spread over a 1000 x 1000 grid, 3-7 scans each: a CTA's item range
    covers several jobs and restages the box between them.  The same jobs plus one whose
    reach exceeds the box run as global gathers."""
    rng = np.random.RandomState(11)
    grid = pgrid(rand_cells(rng, 1000, 1000), max_x=30.0, max_y=30.0)
    clouds, inits = [], []
    for k in range(40):
        clouds.append(disk_cloud(rng, int(rng.randint(1, 200)), rng.uniform(0.5, 2.0)))
        inits.append(np.array([rng.uniform(-28, 28), rng.uniform(-28, 28), rng.uniform(-3, 3)]))
    res, _ = check_2d(oracle, sm, grid, clouds, inits, 2, 0.15, form="tma")
    assert len({r.num_scans for r in res}) > 1
    clouds.append(disk_cloud(rng, 50, 20.0))
    inits.append(np.array([0.0, 0.0, 0.0]))
    check_2d(oracle, sm, grid, clouds, inits, 2, 0.15, form="gather")


def test_more_jobs_than_one_launch_takes(oracle, sm):
    """4097 jobs: two launches (kMaxJobs = 4096).  Per-job results and scores, summed stats."""
    rng = np.random.RandomState(12)
    grid = pgrid(rand_cells(rng, 64, 64), max_x=2.0, max_y=2.0)
    clouds = [disk_cloud(rng, 3, 0.1) for _ in range(4097)]
    inits = [np.array([rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5), 0.0]) for _ in range(4097)]
    names, st = match_batch(oracle, sm, grid, clouds, inits, 1, 0.0)
    assert KERNEL["tma"] in names
    assert st["candidates_scored"] == 4097 * 9 and st["host_syncs"] == 2
    check_2d(oracle, sm, grid, clouds, inits, 1, 0.0, form="tma")


# ==== 2D: ties ================================================================================
@pytest.mark.parametrize("tsdf", [False, True])
def test_ties_go_to_the_first_candidate(oracle, sm, tsdf):
    """A uniform grid that every candidate reads entirely.  w_t = w_r = 0: all candidates
    equal, candidate 0 wins.  w_t = 0, w_r > 0: the middle scan's candidates all carry the
    largest weight, and its first, (-lin, -lin), wins."""
    rng = np.random.RandomState(13)
    shape = (120, 120)
    if tsdf:
        grid = synthetic.TSDFGridSpec(np.full(shape, 20000, np.uint16),
                                      np.full(shape, 30000, np.uint16), RES, 3.0, 3.0, 0.3, 10.0)
    else:
        grid = pgrid(np.full(shape, 9000, np.uint16), max_x=3.0, max_y=3.0)
    clouds = [disk_cloud(rng, 100, 1.0)]
    inits = [np.array([-0.75, -0.75, 0.2])]
    lin_cells = 3
    res, scores = check_2d(oracle, sm, grid, clouds, inits, lin_cells, 0.3, 0.0, 0.0)
    assert len(set(bits(scores[0]).tolist())) == 1
    assert (res[0].best_scan_index, res[0].best_x_offset, res[0].best_y_offset) == (
        0, -lin_cells, -lin_cells)
    res, _ = check_2d(oracle, sm, grid, clouds, inits, lin_cells, 0.3, 0.0, 0.5)
    assert res[0].num_scans > 1
    assert (res[0].best_scan_index, res[0].best_x_offset, res[0].best_y_offset) == (
        (res[0].num_scans - 1) // 2, -lin_cells, -lin_cells)


def test_update_marker_cells(oracle, sm):
    """Cells with the update marker (0x8000) set, written through update(): the marker is not
    part of the value (ProbabilityGrid and TSDF2D)."""
    rng = np.random.RandomState(14)
    grid = pgrid(rand_cells(rng, 150, 150), max_x=5.0, max_y=5.0)
    dg = sm.RealTimeGrid2D(grid)
    try:
        cells2 = grid.cells.copy()
        mark = rng.uniform(size=cells2.shape) < 0.5
        cells2[mark] |= 0x8000
        dg.update(cells2)
        g2 = pgrid(cells2, max_x=5.0, max_y=5.0)
        check_2d(oracle, sm, g2, [disk_cloud(rng, 400, 3.0)], [np.array([0.3, 0.2, 1.0])], 3,
                 0.2, form="tma", dg=dg)
    finally:
        dg.close()
    t = tgrid(rng, 150, 150, max_x=5.0, max_y=5.0)
    dt = sm.RealTimeGrid2D(t)
    try:
        tsd2, w2 = t.tsd_cells.copy(), t.weight_cells.copy()
        tsd2[rng.uniform(size=tsd2.shape) < 0.5] |= 0x8000
        w2[rng.uniform(size=w2.shape) < 0.5] |= 0x8000
        dt.update(tsd2, w2)
        t2 = synthetic.TSDFGridSpec(tsd2, w2, RES, 5.0, 5.0, 0.3, 10.0)
        check_2d(oracle, sm, t2, [disk_cloud(rng, 400, 3.0)], [np.array([0.3, 0.2, 1.0])], 3,
                 0.2, dg=dt)
    finally:
        dt.close()


@pytest.mark.parametrize("tsdf", [False, True])
def test_scans_beside_and_outside_the_grid(oracle, sm, tsdf):
    """Initial poses beside each side and corner of the grid (scans partly inside) and far
    outside it (every read outside the limits)."""
    rng = np.random.RandomState(15)
    ny, nx = 80, 100
    grid = tgrid(rng, ny, nx, max_x=2.0, max_y=2.0) if tsdf else \
        pgrid(rand_cells(rng, ny, nx), max_x=2.0, max_y=2.0)
    clouds, inits = [], []
    for ix in (-3, nx // 2, nx + 2, -40, nx + 40):
        for iy in (-3, ny // 2, ny + 2, -40, ny + 40):
            if (ix, iy) == (nx // 2, ny // 2):
                continue
            inits.append(init_at(grid, ix, iy) + np.array([0.01, -0.02, rng.uniform(-1, 1)]))
            clouds.append(disk_cloud(rng, int(rng.randint(1, 80)), 1.0))
    check_2d(oracle, sm, grid, clouds, inits, 2, 0.3)


# ==== 2D: the single-call form's grid cache and the public ScoreCandidates ======================
def test_single_call_grid_cache(oracle, sm):
    """Match keeps one device grid per lane while the dimensions stay: two calls with the same
    dimensions but different limits and cells, then a switch to a TSDF2D of the same size, then
    back."""
    rng = np.random.RandomState(16)
    lin, ang = 2 * RES, 0.1
    rt = sm.RealTimeCorrelativeScanMatcher2D(
        sm.RealTimeCorrelativeScanMatcherOptions(lin, ang, 0.1, 0.1))
    cloud, init = disk_cloud(rng, 300, 2.0), np.array([0.5, -0.5, 0.3])
    g1 = pgrid(rand_cells(rng, 100, 120), max_x=3.0, max_y=3.0)
    g2 = pgrid(rand_cells(rng, 100, 120), max_x=2.5, max_y=4.0)
    t = tgrid(rng, 100, 120, max_x=3.0, max_y=2.0)
    for g in (g1, g2, t, g1):
        if hasattr(g, "tsd_cells"):
            score, pose = rt.MatchTSDF(init, cloud, g)
        else:
            score, pose = rt.Match(init, cloud, g)
        want = oracle_2d(oracle, g, cloud, init, lin, ang, 0.1, 0.1)[1]
        assert bits(score) == bits(want["score"])
        np.testing.assert_array_equal(pose, want["pose"])


def test_public_score_candidates(oracle, sm):
    """ScoreCandidates on caller-given candidates: offsets outside the search window and
    candidate counts that are not multiples of the 128-thread block."""
    rng = np.random.RandomState(17)
    grid = pgrid(rand_cells(rng, 120, 130), max_x=4.0, max_y=4.0)
    og = oracle_grid(oracle, grid)
    cloud, init = disk_cloud(rng, 77, 2.0), np.array([0.2, 0.1, 0.5])
    lin, ang = 2 * RES, 0.2
    fe = oracle.frontend2d(og, cloud, init, False, lin, ang, rt_mode=True)
    S = fe["num_scans"]
    rt = sm.RealTimeCorrelativeScanMatcher2D(
        sm.RealTimeCorrelativeScanMatcherOptions(lin, ang, 0.3, 0.2))
    for count in (1, 127, 129, 300):
        cand = np.stack([rng.randint(0, S, count), rng.randint(-9, 10, count),
                         rng.randint(-9, 10, count)], axis=1).astype(np.int32)
        want = oracle.rt2d_score_candidates(og, fe["discrete_scans"], 2, (S - 1) // 2, fe["step"],
                                            0.3, 0.2, cand)
        got = rt.ScoreCandidates(grid, fe["discrete_scans"], (S - 1) // 2, fe["step"], cand)
        np.testing.assert_array_equal(bits(got), bits(want))


# ==== regressions ==============================================================================
def overshooting_tsd_value(oracle, truncation):
    """The saturated tsd value (32767 or 1) whose decoding lies past +-truncation, so that a
    weighted cell holding it scores below 0: found by scoring a one-cell grid in the oracle."""
    for v in (32767, 1):
        s = oracle.rt2d_scores_tsdf(np.array([[v]], np.uint16), np.array([[32767]], np.uint16),
                                    RES, RES, RES, truncation, 10.0, np.zeros((1, 3), np.float32),
                                    [0.5 * RES, 0.5 * RES, 0.0], 0.0, 0.0, 0.0, 0.0)
        if s[0] < 0:
            return v
    raise AssertionError("truncation %g decodes both ends within range" % truncation)


@pytest.mark.parametrize("form", ["tma", "gather"])
def test_far_points_are_not_clamped_into_the_grid(oracle, sm, form):
    """A 29999 x 8 grid (the widest the handle takes) and points 1-3 cells beyond its last
    column, lin = 2.  A point 2 or 3 cells beyond reads outside the grid at every offset; a
    clamp of the cell to +-30000 would make it read column 29998 at x offset -2.  That column
    is the grid's only high-probability one, so such a clamp changes the winner's score."""
    nx, ny = 29999, 8
    cells = np.full((ny, nx), 32767, np.uint16)
    cells[:, nx - 1] = 1
    grid = pgrid(cells, max_x=0.0, max_y=0.0)
    init = init_at(grid, nx + 2, 3)
    cloud = cloud_at_cells(grid, init, [(nx + d, iy) for d in (1, 2, 3) for iy in (2, 3, 4, 5)])
    clouds, inits = [cloud], [init]
    if form == "gather":     # a job whose reach exceeds the box sends the batch to gathers
        far = init_at(grid, nx - 100, 4)
        clouds.append(cloud_at_cells(grid, far, [(nx - 100 - 300, 4), (nx - 100, 4)]))
        inits.append(far)
    assert expected_form(grid, clouds, inits, 2) == form
    names, _ = match_batch(oracle, sm, grid, clouds, inits, 2, 0.0)
    assert KERNEL[form] in names
    check_2d(oracle, sm, grid, clouds, inits, 2, 0.0, form=form)


@pytest.mark.parametrize("patch", ["mid", "corner", "none"])
@pytest.mark.parametrize("w_t", [0.1, 1e4])
@pytest.mark.parametrize("truncation", [0.35, 0.27])
def test_tsdf_non_positive_scores(oracle, sm, truncation, w_t, patch):
    """TSDF scores below zero.  For truncations 0.35 and 0.27 the saturated tsd value (32767 or
    1) decodes to slightly more than the truncation in magnitude, so (T - |tsd|) / T < 0 in
    every cell that carries weight.  A patch of weight-0 cells scores exactly 0 for the
    candidate that reads only it: the first maximum is that candidate (mid-window or the
    window's first), not candidate 0 with a clamped score.  With w_t = 1e4 every off-centre
    weight underflows to 0, so those candidates score -0.0, which ties with +0.0 in generation
    order; the returned score keeps the winner's sign."""
    value = overshooting_tsd_value(oracle, truncation)
    nx = ny = 40
    lin_cells = 2
    tsd = np.full((ny, nx), value, np.uint16)
    wgt = np.full((ny, nx), 32767, np.uint16)
    grid = synthetic.TSDFGridSpec(tsd, wgt, RES, 1.0, 1.0, truncation, 10.0)
    init = init_at(grid, 20, 20)
    cloud = np.zeros((5, 3), np.float32)   # every rotated scan reads cell (20, 20) + offset
    if patch == "mid":
        wgt[20, 20] = 0
    elif patch == "corner":
        wgt[20 - lin_cells, 20 - lin_cells] = 0
    ang = 0.7
    scores, want = oracle_2d(oracle, grid, cloud, init, lin_cells * RES, ang, w_t, 0.0)
    assert (scores <= 0).all() and (scores < 0).any() if w_t < 1 else (scores <= 0).all()
    if patch == "mid" and w_t < 1:
        assert want["score"] == 0.0 and (want["best_x_offset"], want["best_y_offset"]) == (0, 0)
    if w_t > 1 and patch != "corner":
        assert bits(want["score"]) == 0x80000000
    names, _ = match_batch(oracle, sm, grid, [cloud], [init], lin_cells, ang, w_t, 0.0)
    assert KERNEL["tsdf"] in names
    check_2d(oracle, sm, grid, [cloud], [init], lin_cells, ang, w_t, 0.0)


@pytest.mark.parametrize("lin_cells", [0, 1])
def test_idle_lanes_stay_inside_the_staged_box(oracle, sm, lin_cells):
    """Jobs whose reach misses the grid are planned into the staged box at (0, 0).  Their
    points lie left of the grid (x index -30 .. -7), in rows past the box height of a grid
    taller than the box.  Lanes without a candidate (every lane r >= per_scan) gather at the
    last candidate's offsets, within lin of a point's cell, so outside the grid; without that
    an idle lane's x offset reaches +31 (lin 0) or +9 (lin 1), back into the grid, and its
    row index past the box.  Run only against builds where idle lanes keep a real offset."""
    ny, nx = 300, 256
    bw, bh = box_dims(nx, ny)
    assert (bw, bh) == (256, 200)
    rng = np.random.RandomState(18)
    grid = pgrid(rand_cells(rng, ny, nx))
    clouds, inits = [], []
    for ix, iy in [(-9, 250), (-8, 299), (-12, 210), (-20, 260), (-25, 201)]:
        if ix + 6 + lin_cells >= 0:
            continue
        init = init_at(grid, ix, iy)
        clouds.append(cloud_at_cells(grid, init, [(ix, iy), (ix - 1, iy + 1), (ix, iy - 2)]))
        inits.append(init)
        fits, w, h = job_fits(grid, clouds[-1], inits[-1], lin_cells)
        assert fits and (w, h) == (0, 0)    # the reach misses the grid
    # and one job inside the grid, staged where it reads
    inits.append(init_at(grid, 100, 100))
    clouds.append(disk_cloud(rng, 200, 2.0))
    assert len(clouds) >= 4
    check_2d(oracle, sm, grid, clouds, inits, lin_cells, 0.5, form="tma")


# ==== 3D ======================================================================================
def rand_hybrid(rng, res, lo, hi, fill=0.5):
    g = np.stack(np.meshgrid(*[np.arange(lo, hi + 1)] * 3, indexing="ij"), -1).reshape(-1, 3)
    keep = rng.uniform(size=len(g)) < fill
    idx = g[keep].astype(np.int32)
    val = rng.randint(1, 32768, size=len(idx)).astype(np.uint16)
    return synthetic.HybridGridSpec(res, idx, val)


def angular_step(res, cloud):
    """The 3D search's angular step (real_time...3d.cc:66-77) in float32."""
    res = np.float32(res)
    r = np.sqrt((cloud.astype(np.float32) ** 2).sum(1), dtype=np.float32)
    msr = max(np.float32(3) * res, r.max()) if len(r) else np.float32(3) * res
    return float(np.float32(1 - 1e-3) * np.arccos(np.float32(1) - (res * res) /
                                                 (np.float32(2) * (msr * msr))))


def check_3d(oracle, sm, spec, cloud, init, lin, ang, w_t=0.1, w_r=0.5, dg=None):
    og = oracle.HybridGrid(spec.resolution, spec.indices, spec.values)
    own = dg is None
    dg = sm.DeviceHybridGrid(spec) if own else dg
    rt = sm.RealTimeCorrelativeScanMatcher3D(
        sm.RealTimeCorrelativeScanMatcherOptions(lin, ang, w_t, w_r))
    try:
        scores, names = profiled(lambda: rt.Scores(init, cloud, dg))
        score, pose = rt.Match(init, cloud, dg)
    finally:
        if own:
            dg.close()
    assert "k_rt3_match" in names
    want_scores = oracle.rt3d_scores(og, cloud, init, lin, ang, w_t, w_r)
    want = oracle.rt3d_match(og, cloud, init, lin, ang, w_t, w_r)
    np.testing.assert_array_equal(bits(scores), bits(want_scores))
    assert bits(score) == bits(want["score"])
    np.testing.assert_array_equal(pose, want["pose"])
    assert rt.last_stats["candidates_scored"] == want["candidates_scored"] == len(scores)
    return scores, want


POSE_3D = [0.05, -0.1, 0.02, math.cos(0.15), 0.0, 0.0, math.sin(0.15)]


@pytest.mark.parametrize("L,A", [(0, 0), (1, 2), (2, 1), (3, 0)])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 700])
def test_3d_point_counts_and_windows(oracle, sm, n, L, A):
    """n around the 256-point chunk; T = 1, 27, 125, 343 translations (partial passes of the
    128-thread stride) and 1, 27, 125 rotations."""
    rng = np.random.RandomState(1000 + n + 10 * L + A)
    spec = rand_hybrid(rng, 0.1, -8, 8)
    cloud = (rng.uniform(-0.7, 0.7, (n, 3))).astype(np.float32)
    ang = A * angular_step(0.1, cloud)
    scores, _ = check_3d(oracle, sm, spec, cloud, POSE_3D, L * 0.1, ang)
    assert len(scores) == (2 * L + 1) ** 3 * (2 * A + 1) ** 3


@pytest.mark.parametrize("uniform", [False, True])
def test_3d_ties(oracle, sm, uniform):
    """An empty grid and a uniform grid: with zero weights every candidate scores the same and
    candidate 0 wins; with weights the zero translation and rotation wins."""
    rng = np.random.RandomState(21)
    if uniform:
        spec = rand_hybrid(rng, 0.1, -12, 12, fill=1.0)
        spec.values[:] = 20000
    else:
        spec = synthetic.HybridGridSpec(0.1, np.zeros((0, 3), np.int32), np.zeros(0, np.uint16))
    cloud = rng.uniform(-0.5, 0.5, (300, 3)).astype(np.float32)
    ang = angular_step(0.1, cloud)
    scores, want = check_3d(oracle, sm, spec, cloud, POSE_3D, 0.1, ang, 0.0, 0.0)
    assert len(set(bits(scores).tolist())) == 1 and want["best_index"] == 0
    scores, want = check_3d(oracle, sm, spec, cloud, POSE_3D, 0.1, ang, 0.1, 0.5)
    assert want["best_index"] == len(scores) // 2


def test_3d_points_outside_the_dense_box(oracle, sm):
    """Voxels in [-4, 4]^3 (negative indices included); points well past every face of the
    dense box, at negative and positive indices."""
    rng = np.random.RandomState(22)
    spec = rand_hybrid(rng, 0.1, -4, 4, fill=0.7)
    cloud = rng.uniform(-1.0, 1.0, (500, 3)).astype(np.float32)
    for axis in range(3):
        for sign in (-1, 1):
            p = rng.uniform(-0.3, 0.3, (20, 3))
            p[:, axis] = sign * rng.uniform(0.45, 0.9, 20)
            cloud = np.concatenate([cloud, p.astype(np.float32)])
    check_3d(oracle, sm, spec, cloud, [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0], 0.2,
             angular_step(0.1, cloud))


def test_3d_points_on_half_cells(oracle, sm):
    """Identity pose and no rotation: points exactly on half cells of both signs, which
    lroundf rounds away from zero (HybridGrid::GetCellIndex)."""
    rng = np.random.RandomState(23)
    res = 0.125
    spec = rand_hybrid(rng, res, -7, 7, fill=0.8)
    k = np.arange(-6, 6)
    g = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)
    cloud = ((g + 0.5) * res).astype(np.float32)
    assert np.all(cloud / np.float32(res) % 1 == 0.5)
    check_3d(oracle, sm, spec, cloud, [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0], res, 0.0)


def test_3d_grid_from_range_data_inserter(oracle, sm):
    """A grid written by RangeDataInserter3D on the device, grown by a second scan."""
    rng = np.random.RandomState(24)
    dg = sm.DeviceHybridGrid.empty(0.1)
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D())
    try:
        for origin in ([0.0, 0.0, 0.0], [3.0, -2.0, 0.5]):
            ret = (np.array(origin) + rng.uniform(-1.5, 1.5, (400, 3))).astype(np.float32)
            ins.Insert(np.array(origin, np.float32), ret, None, dg)
        lo, vals = dg.read()
        z, y, x = np.nonzero(vals)
        idx = (np.stack([x, y, z], 1) + lo).astype(np.int32)
        spec = synthetic.HybridGridSpec(0.1, idx, vals[z, y, x])
        assert (idx.max(0) - idx.min(0)).max() > 30      # grown past the first scan's box
        cloud = rng.uniform(-1.2, 1.2, (300, 3)).astype(np.float32)
        check_3d(oracle, sm, spec, cloud, POSE_3D, 0.1, angular_step(0.1, cloud), dg=dg)
    finally:
        ins.close()
        dg.close()


def test_3d_refusals(sm):
    """CSM_E_INVALID (status 1) for L or A above 64, T * R of 2^31 or more, and n = 0."""
    from cartographer_b200._lib import CsmError
    spec = synthetic.HybridGridSpec(0.1, np.zeros((1, 3), np.int32), np.full(1, 100, np.uint16))
    dg = sm.DeviceHybridGrid(spec)
    cloud = np.array([[1.0, 0.0, 0.0]], np.float32)
    step = angular_step(0.1, cloud)
    try:
        for lin, ang, c in [(6.5, 0.0, cloud), (0.0, 65 * step, cloud),
                            (2.0, 20 * step, cloud), (0.1, 0.0, cloud[:0])]:
            rt = sm.RealTimeCorrelativeScanMatcher3D(
                sm.RealTimeCorrelativeScanMatcherOptions(lin, ang, 0.1, 0.1))
            for call in (rt.Match, rt.Scores):
                with pytest.raises(CsmError) as err:
                    call(POSE_3D, c, dg)
                assert err.value.status == 1, (lin, ang, len(c))
    finally:
        dg.close()
