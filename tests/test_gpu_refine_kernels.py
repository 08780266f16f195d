"""The refinement kernels residual by residual at their edges, and the trust-region minimiser
branch by branch (refine2d.cu, refine3d.cu, trust_region.cuh).

Rows: every residual and Jacobian row of the evaluate hooks against the restatements
(oracle_ceres2d.cc, oracle_ceres3d.cc, tests/tsdf2d_oracle.py, tests/intensity3d_oracle.py) at
points built from the grid's own limits — cell centres and boundaries, one float ulp either
side, the rows and columns around every border, marker cells, the dense box's faces — at the
existing tolerances (residuals 1e-12, Jacobians 1e-10 in 2D and 1e-12 in 3D), exactly where the
value is a constant.  Solves: the cases of tests/refine_cases.py against the traced oracles;
the trace proves that the case reached the branch it names and that every deciding quantity
is 1e-6 (relative) away from its threshold, so a device that took another branch cannot give
the same counts and the same pose to 1e-7.  Batches: every job equals its single call bit for
bit.  Non-finite coordinates, poses and targets are refused with CSM_E_INVALID.

Every case asserts that it reached the edge it names.

Not reached, tried once with the traced oracles over the seeds of refine_cases.py:
MIN_TRUST_REGION_RADIUS and INVALID_STEPS.  The longest run of rejections found is 9 (the
radius is then 1e4 / 2^45, far above 1e-32; the parameter tolerance stops a solve long
before) — and that run comes from a solve caught in an exact 2-cycle, whose step quality is
exactly 0 because the candidate's cost equals the reference cost bit for bit; such solves are
decided by rounding and refine_cases.assert_margins refuses them as parity cases
(TSDF_DECIDED_BY_ROUNDING).  The damped matrix keeps a diagonal >= 1e-6 / radius, so its Cholesky
factorisation does not fail on finite input.  No case is contrived for them."""
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import intensity3d_oracle as iorc
from tests import refine_cases as RC
from tests import tsdf2d_oracle as T

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-7
F = np.float32
OPTS2D = dict(occupied_space_weight=20.0, translation_weight=10.0, rotation_weight=1.0)


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def ulps(v):
    """v, one float32 ulp below and one above."""
    v = np.asarray(v, F)
    return np.concatenate([v, np.nextafter(v, F(-np.inf)), np.nextafter(v, F(np.inf))])


def same_solution(pose, summary, want):
    assert np.allclose(pose, want["pose"], rtol=0, atol=POSE_TOL), (pose, want["pose"])
    assert summary["termination"] == want["termination"]
    assert summary["iterations"] == want["iterations"]
    assert summary["num_successful_steps"] == want["num_successful_steps"]
    assert summary["initial_cost"] == pytest.approx(want["initial_cost"], rel=1e-12, abs=1e-15)
    assert summary["final_cost"] == pytest.approx(want["final_cost"], rel=1e-9, abs=1e-15)


# ============================ rows: 2D ProbabilityGrid ========================================
edge_cells = RC.edge_cells


def axis_positions(n):
    """Cell coordinates -3 .. 2 and n-3 .. n+2 at the cell's boundary and its centre."""
    cells = sorted(set(range(-3, 3)) | set(range(n - 3, n + 3)))
    return np.array([c + f for c in cells for f in (0.0, 0.5)])


def edge_cloud(nx, ny, res, max_x, max_y):
    """Sensor-frame points (pose 0) whose cell coordinates are axis_positions on both axes,
    each with its float neighbours: index x <- world y, index y <- world x."""
    wx = ulps(max_x - axis_positions(ny) * res)
    wy = ulps(max_y - axis_positions(nx) * res)
    gx, gy = np.meshgrid(wx, wy, indexing="ij")
    return np.stack([gx.ravel(), gy.ravel(), np.zeros(gx.size)], 1).astype(F)


def patch_origin(cloud, pose, res, max_x, max_y):
    """(row, col) of BiCubic's floor, without the kPadding shift, and whether the shifted
    coordinate is integral — restated from PointResidual."""
    cs, sn = math.cos(pose[2]), math.sin(pose[2])
    px, py = cloud[:, 0].astype(np.float64), cloud[:, 1].astype(np.float64)
    wx = (cs * px + (-sn) * py) + pose[0] * 1.0
    wy = (sn * px + cs * py) + pose[1] * 1.0
    r = (max_x - wx) / res - 0.5 + float(RC.K_PADDING)
    c = (max_y - wy) / res - 0.5 + float(RC.K_PADDING)
    return (np.floor(r).astype(np.int64) - RC.K_PADDING, np.floor(c).astype(np.int64) - RC.K_PADDING,
            (r == np.floor(r)) | (c == np.floor(c)), r, c)


def check_rows2d(sm, oracle, dev, grid, cloud, pose, target=(0.2, -0.1), angle=0.25):
    m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(**OPTS2D))
    out = None
    for jac in (True, False):
        r, j = m.Evaluate(dev, cloud, pose, target, angle, jacobian=jac)
        rc, jc, valid = m.EvaluateChecked(dev, cloud, pose, target, angle, jacobian=jac)
        wr, wj = oracle.ceres2d_evaluate(grid, cloud, pose, target, angle, jacobian=jac)
        assert valid and np.array_equal(r, rc)
        assert np.allclose(r, wr, rtol=0, atol=1e-12)
        if jac:
            assert np.array_equal(j, jc)
            assert np.allclose(j, wj, rtol=0, atol=1e-10)
            out = (r, j)
    return out


@pytest.mark.parametrize("ny,nx", [(1, 1), (1, 9), (9, 1), (5, 7), (8, 8), (6, 9), (3, 250),
                                   (4, 257)])
@pytest.mark.parametrize("theta", [0.0, 0.3])
def test_rows2d_around_every_border(sm, oracle, ny, nx, theta):
    """nx = 7, 9, 250, 257: the handle's 16-byte row pitch differs from nx."""
    rng = np.random.RandomState(1000 * ny + nx)
    res, max_x, max_y = 0.05, 1.3, -0.7            # non-zero, non-square limits
    grid = oracle.Grid2D(edge_cells(rng, ny, nx), res, max_x, max_y)
    dev = sm.RealTimeGrid2D(grid)
    try:
        cloud = edge_cloud(nx, ny, res, max_x, max_y)
        if theta != 0.0:      # the sensor-frame points that the pose turns onto those edges
            cs, sn = math.cos(theta), math.sin(theta)
            x, y = cloud[:, 0].astype(np.float64), cloud[:, 1].astype(np.float64)
            cloud = np.stack([cs * x + sn * y, -sn * x + cs * y, np.zeros(len(x))], 1).astype(F)
        pose = np.array([0.0, 0.0, theta])
        row, col, integral, _, _ = patch_origin(cloud, pose, res, max_x, max_y)
        # the 4 x 4 patch (row-1 .. row+2) straddles each border and each corner
        for lo in (-2, -1, 0):
            assert (row == lo).any() and (col == lo).any()
            assert ((row == lo) & (col == lo)).any()
            assert ((row == ny - 2 - lo) & (col == nx - 2 - lo)).any()
            assert ((row == lo) & (col == nx - 2 - lo)).any()
        assert (row < -2).any() and (row > ny).any() and (col < -2).any() and (col > nx).any()
        if theta == 0.0:
            assert integral.sum() >= 100        # floor() of an integral shifted coordinate
        if nx not in (1, 8):
            assert (nx * 2 + 15) // 16 * 16 != nx * 2
        r, j = check_rows2d(sm, oracle, dev, grid, cloud, pose)
        # patches wholly outside the grid: exactly the max-cost residual and a zero row
        outside = (row + 2 < 0) | (row - 1 >= ny) | (col + 2 < 0) | (col - 1 >= nx)
        assert outside.sum() >= 100
        scaling = OPTS2D["occupied_space_weight"] / math.sqrt(float(len(cloud)))
        assert np.all(r[:-3][outside] == scaling * float(F(0.9)))
        assert np.all(j[:-3][outside] == 0.0)
    finally:
        dev.close()


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 511, 513])
def test_rows2d_point_counts(sm, oracle, n):
    """The prior rows are written by thread n of a launch of (n + 1 + 255) / 256 blocks: for
    n = 255 it is the last thread of block 0, for n = 256 the first of block 1."""
    rng = np.random.RandomState(n)
    grid = oracle.Grid2D(edge_cells(rng, 12, 9), 0.05, 0.3, 0.2)
    dev = sm.RealTimeGrid2D(grid)
    try:
        full = edge_cloud(9, 12, 0.05, 0.3, 0.2)
        cloud = full[rng.permutation(len(full))[:n]]
        assert len(cloud) == n and (n + 1 + 255) // 256 == (1 if n < 256 else 2 if n < 512 else 3)
        r, j = check_rows2d(sm, oracle, dev, grid, cloud, np.array([0.01, -0.02, 0.1]))
        assert r.shape == (n + 3,)
        assert np.array_equal(r[n:], [10.0 * (0.01 - 0.2), 10.0 * (-0.02 + 0.1), 1.0 * (0.1 - 0.25)])
        assert np.array_equal(j[n:], np.diag([10.0, 10.0, 1.0]))
    finally:
        dev.close()


def test_rows2d_points_closer_than_the_padding_quantum(sm, oracle):
    """Adding kPadding = 2^29 to the cell coordinate leaves 23 fraction bits: points closer
    than 2^-23 of a cell get the same residual."""
    rng = np.random.RandomState(5)
    grid = oracle.Grid2D(RC.noise_cells(rng, 8, 8), 0.05, 0.2, 0.2)
    dev = sm.RealTimeGrid2D(grid)
    try:
        a = F(1.234e-3)
        b = np.nextafter(a, F(1))
        cloud = np.array([[a, a, 0], [b, b, 0], [a, b, 0]], F)
        assert 0 < (float(b) - float(a)) / 0.05 < 2.0 ** -23
        _, _, _, r, c = patch_origin(cloud, np.zeros(3), 0.05, 0.2, 0.2)
        assert r[0] == r[1] == r[2] and c[0] == c[1] == c[2]
        res, jac = check_rows2d(sm, oracle, dev, grid, cloud, np.zeros(3))
        assert res[0] == res[1] == res[2] and res[0] != 0.0
        assert np.array_equal(jac[0][:2], jac[1][:2])
    finally:
        dev.close()


def test_rows2d_after_update_and_after_growth(sm, oracle):
    rng = np.random.RandomState(9)
    res, max_x, max_y = 0.05, 0.4, 0.3
    first, second = edge_cells(rng, 10, 7), edge_cells(rng, 10, 7)
    dev = sm.RealTimeGrid2D(oracle.Grid2D(first, res, max_x, max_y))
    try:
        dev.update(second)
        assert not np.array_equal(first, second)
        check_rows2d(sm, oracle, dev, oracle.Grid2D(second, res, max_x, max_y),
                     edge_cloud(7, 10, res, max_x, max_y), np.array([0.0, 0.0, 0.2]))
    finally:
        dev.close()
    # a handle ProbabilityGridRangeDataInserter2D grew: its arrays were reallocated
    dev = sm.RealTimeGrid2D.empty(res, 0.5, 0.5, num_x=20, num_y=20)
    ins = sm.ProbabilityGridRangeDataInserter2D()
    try:
        a = np.linspace(-math.pi, math.pi, 90, endpoint=False)
        hits = np.stack([3.0 * np.cos(a), 2.0 * np.sin(a), np.zeros(90)], 1).astype(F)
        ins.Insert([0.1, 0.05, 0.0], hits, dev)
        st = dev.read()
        assert st.cells.shape[0] > 20 and st.cells.shape[1] > 20      # grown
        assert (st.cells != 0).sum() > 200
        grid = oracle.Grid2D(st.cells, st.resolution, st.max_x, st.max_y)
        ny, nx = st.cells.shape
        check_rows2d(sm, oracle, dev, grid, edge_cloud(nx, ny, res, st.max_x, st.max_y),
                     np.array([0.0, 0.0, -0.4]))
        check_rows2d(sm, oracle, dev, grid, hits, np.array([0.1, 0.05, 0.01]))
    finally:
        ins.close()
        dev.close()


# ============================ rows: TSDF2D ====================================================
def tsdf_pair(sm, tsd, wgt, res, max_x, max_y, truncation, max_weight=10.0):
    g = T.TSDF2D(tsd.shape[1], tsd.shape[0], res, max_x, max_y, truncation, max_weight, tsd, wgt)
    return g, sm.RealTimeGrid2D(sm.TSDF2DSpec(g.tsd_cells, g.weight_cells, res, max_x, max_y,
                                              g.truncation_distance, g.max_weight))


def check_rows_tsdf(sm, g, dev, cloud, pose, target=(0.2, -0.1), angle=0.25):
    m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(**OPTS2D))
    out = None
    for jac in (True, False):
        r, j, valid = m.EvaluateChecked(dev, cloud, pose, target, angle, jacobian=jac)
        wr, wj, wvalid = T.evaluate(g, cloud, pose, target, angle, jacobian=jac)
        assert valid == wvalid
        if not valid:
            return None
        assert np.allclose(r, wr, rtol=1e-12, atol=1e-12 * np.abs(wr).max())
        if jac:
            assert np.allclose(j, wj, rtol=1e-10, atol=1e-10 * np.abs(wj).max())
            out = (r, j)
    return out


@pytest.mark.parametrize("truncation", [0.3, 0.35, 0.27])
@pytest.mark.parametrize("ny,nx", [(6, 7), (9, 12)])
def test_rows_tsdf_centres_corners_and_markers(sm, truncation, ny, nx):
    rng = np.random.RandomState(int(truncation * 100) + nx)
    res, max_x, max_y = 0.05, 0.45, -0.2
    tsd, wgt = edge_cells(rng, ny, nx), edge_cells(rng, ny, nx)
    tsd[1, 1] = wgt[1, 2] = 32767                     # the saturated value
    g, dev = tsdf_pair(sm, tsd, wgt, res, max_x, max_y, truncation)
    try:
        # the saturated value decodes at or past the truncation for 0.35 and 0.27
        top = float(g.conv.value_to_cost(np.array([32767]))[0])
        assert (top > float(F(truncation))) == (truncation != 0.3) and (tsd == 32767).any()
        cloud = edge_cloud(nx, ny, res, max_x, max_y)
        pose = np.zeros(3)
        x, y = cloud[:, 0].astype(np.float64), cloud[:, 1].astype(np.float64)
        lx, ly, _, _, ix, iy = T._corners(g, x, y)
        cx, cy = g.cell_index(cloud[:, 0], cloud[:, 1])
        fx, fy = g.cell_center(cx, cy)
        # points exactly on a cell centre, and points whose centre is above them (lx > x)
        assert ((fx.astype(np.float64) == x) & (fy.astype(np.float64) == y)).sum() >= 10
        assert (fx.astype(np.float64) > x).sum() >= 100 and (fy.astype(np.float64) > y).sum() >= 100
        # each single corner without weight while the other three have it
        w = [g.get_weight(ix, iy), g.get_weight(ix - 1, iy), g.get_weight(ix, iy - 1),
             g.get_weight(ix - 1, iy - 1)]
        for k in range(4):
            others = np.all([w[m] != 0 for m in range(4) if m != k], axis=0)
            assert ((w[k] == 0) & others).any(), k
        assert np.all([wk != 0 for wk in w], axis=0).sum() >= 20
        # corners outside the limits and marker bits in both cell arrays
        assert ((ix - 1 < 0) | (iy - 1 < 0) | (ix >= nx) | (iy >= ny)).any()
        assert (tsd >= 32768).any() and (wgt >= 32768).any()
        r, j = check_rows_tsdf(sm, g, dev, cloud, pose)
        assert np.abs(r[:-3]).max() > 0
        check_rows_tsdf(sm, g, dev, cloud, np.array([0.003, -0.002, 0.3]))
    finally:
        dev.close()


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 511, 513])
def test_rows_tsdf_point_counts(sm, n):
    rng = np.random.RandomState(n)
    tsd, wgt = RC.noise_cells(rng, 12, 9), RC.noise_cells(rng, 12, 9)
    g, dev = tsdf_pair(sm, tsd, wgt, 0.05, 0.3, 0.2, 0.3)
    try:
        full = edge_cloud(9, 12, 0.05, 0.3, 0.2)
        inside = (np.abs(full[:, 0] - 0.0) < 0.25) & (np.abs(full[:, 1] + 0.02) < 0.18)
        cloud = np.concatenate([full[inside], full[~inside]])[:n]   # the first point sees weight
        assert len(cloud) == n
        r, j = check_rows_tsdf(sm, g, dev, cloud, np.array([0.01, -0.02, 0.1]))
        assert r.shape == (n + 3,)
        assert np.array_equal(j[n:], np.diag([10.0, 10.0, 1.0]))
        # no point sees weight: valid == 0
        far = cloud + np.array([50.0, 50.0, 0.0], F)
        assert check_rows_tsdf(sm, g, dev, far, np.zeros(3)) is None
    finally:
        dev.close()


# ============================ rows: 3D ========================================================
def hybrid_pair(sm, oracle, res, idx, val):
    spec = synthetic.HybridGridSpec(res, np.asarray(idx, np.int32), np.asarray(val, np.uint16))
    return oracle.HybridGrid(res, spec.indices, spec.values), sm.DeviceHybridGrid(spec)


def voxel_edge_axis(res, lo, hi):
    """p with p / res at k +- 0.5 for the voxels around both faces of [lo, hi] and around 0,
    at negative coordinates too, with the float neighbours; and the voxel centres."""
    ks = sorted(set(range(lo - 2, lo + 2)) | set(range(hi - 1, hi + 3)) | {-2, -1, 0, 1})
    half = np.array([(k + s) * res for k in ks for s in (-0.5, 0.0, 0.5)])
    return ulps(half)


def cell_of(p, res):
    return iorc.cell_index(res, p)


@pytest.mark.parametrize("size,res", [(1, 0.1), (4, 0.1), (3, 0.25)])
def test_rows3d_voxel_edges_and_box_faces(sm, oracle, size, res):
    rng = np.random.RandomState(size)
    lo, hi = -1, size - 2                      # the box spans negative and positive indices
    ax = np.arange(lo, hi + 1)
    idx = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    val = edge_cells(rng, 1, len(idx)).reshape(-1)
    val[val == 0] = 32768                      # a stored voxel is never 0: marked unknown instead
    grid, dev = hybrid_pair(sm, oracle, res, idx, val)
    try:
        a = voxel_edge_axis(F(res), lo, hi)
        rng.shuffle(a)
        a = a[:18]
        gx, gy, gz = np.meshgrid(a, a, a, indexing="ij")
        cloud = np.stack([gx.ravel(), gy.ravel(), gz.ravel()], 1).astype(F)
        q = cloud[:, 0] / F(res)
        frac = np.abs(q.astype(np.float64) - np.trunc(q.astype(np.float64)))
        assert (frac == 0.5).sum() >= 100      # lroundf decides: halves away from zero
        c = cell_of(cloud, F(res))
        assert (c[:, 0] == lo - 1).any() and (c[:, 0] == hi + 1).any()   # one voxel outside
        assert (c == lo).all(1).any() or size == 1
        assert (val >= 32768).any()
        m = sm.CeresScanMatcher3D()
        for pose in ([0, 0, 0, 1, 0, 0, 0], [0.01, -0.02, 0.015, 0.99, 0.05, -0.08, 0.06],
                     [0.0, 0.0, 0.0, -0.7, 0.1, 0.2, -0.65]):      # non-unit, and negative w
            assert pose[3] == 1 or abs(np.linalg.norm(pose[3:]) - 1.0) > 1e-3
            for jac in (True, False):
                r, j = m.Evaluate([(cloud, dev)], pose, [0.1, 0.0, 0.0], [1, 0, 0, 0], jacobian=jac)
                wr, wj = oracle.ceres3d_evaluate([(cloud, grid)], pose, [0.1, 0.0, 0.0],
                                                 [1, 0, 0, 0], jacobian=jac)
                assert np.allclose(r, wr, rtol=0, atol=1e-12)
                if jac:
                    assert np.allclose(j, wj, rtol=0, atol=1e-12)
        # two voxels outside the box on every axis: exactly 1 - min_probability, a zero row
        far = cloud + F(10.0)
        r, j = m.Evaluate([(far, dev)], [0, 0, 0, 1, 0, 0, 0], [0, 0, 0], [1, 0, 0, 0])
        scaling = 5.0 / math.sqrt(float(len(far)))
        assert np.all(r[:-6] == scaling * (1.0 - float(F(0.1)))) and np.all(j[:-6] == 0.0)
    finally:
        dev.close()


@pytest.mark.parametrize("n_hi,n_lo", [(1, 0), (1, 257), (257, 1), (255, 256), (31, 33), (513, 511)])
def test_rows3d_point_counts_one_and_two_clouds(sm, oracle, n_hi, n_lo):
    res, idx, val, _, _, tgt, init = RC.problem3d(7)
    rng = np.random.RandomState(n_hi + n_lo)
    grid, dev = hybrid_pair(sm, oracle, res, idx, val)
    try:
        hi = rng.uniform(-0.6, 0.6, (n_hi, 3)).astype(F)
        pairs_d, pairs_o = [(hi, dev)], [(hi, grid)]
        if n_lo:
            lo = rng.uniform(-0.6, 0.6, (n_lo, 3)).astype(F)
            pairs_d.append((lo, dev))
            pairs_o.append((lo, grid))
        m = sm.CeresScanMatcher3D()
        for jac in (True, False):
            r, j = m.Evaluate(pairs_d, init, tgt, [1, 0, 0, 0], jacobian=jac)
            wr, wj = oracle.ceres3d_evaluate(pairs_o, init, tgt, [1, 0, 0, 0], jacobian=jac)
            assert r.shape == (n_hi + n_lo + 6,)
            assert np.allclose(r, wr, rtol=0, atol=1e-12)
            if jac:
                assert np.allclose(j, wj, rtol=0, atol=1e-12)
    finally:
        dev.close()


# ============================ rows: intensity =================================================
def test_rows_intensity_threshold_and_boxes(sm, oracle):
    res, idx, val, _, _, tgt, init = RC.problem3d(11, size=6)
    rng = np.random.RandomState(3)
    grid, dev = hybrid_pair(sm, oracle, res, idx, val)
    # the intensity box is shifted against the probability box; one voxel has count 0
    iidx = idx + np.array([2, 0, -1], np.int32)
    sums = rng.uniform(10, 900, len(iidx)).astype(F)
    counts = rng.randint(1, 9, len(iidx)).astype(np.int32)
    counts[5] = 0
    igrid = iorc.IntensityHybridGrid(res, iidx, sums, counts)
    dint = sm.DeviceIntensityGrid(sm.IntensityGridSpec(res, iidx, sums, counts))
    try:
        n = 300
        cloud = rng.uniform(-0.45, 0.65, (n, 3)).astype(F)
        cloud[0] = (iidx[5] * F(res)).astype(F)          # on the count-0 voxel
        threshold = F(100.0)
        inten = rng.uniform(20, 99, n).astype(F)
        inten[1], inten[2], inten[3] = threshold, np.nextafter(threshold, F(0)), np.nextafter(threshold, F(1e9))
        c = cell_of(cloud, F(res))
        in_p = np.all((c >= idx.min(0)) & (c <= idx.max(0)), axis=1)
        in_i = np.all((c >= iidx.min(0)) & (c <= iidx.max(0)), axis=1)
        assert (in_p & ~in_i).sum() >= 5 and (in_i & ~in_p).sum() >= 5
        assert igrid.get_intensity(*iidx[5]) == 0.0
        pose = [0, 0, 0, 1, 0, 0, 0]
        io = (0.5, 0.3, float(threshold))       # the rows are uncorrected by the Huber loss
        m = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
            intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(*io)))
        for jac in (False, True):
            r, j = m.Evaluate([(cloud, dev, dint, inten)], pose, tgt, [1, 0, 0, 0], jacobian=jac)
            wr, wj = iorc.evaluate([(cloud, grid, igrid, inten)], pose, tgt, [1, 0, 0, 0],
                                   [io], jacobian=jac)
            assert np.allclose(r, wr, rtol=0, atol=1e-12)
            if jac:
                assert np.allclose(j, wj, rtol=0, atol=1e-12)
        # intensity == threshold and one float below are residuals; one float above is
        # skipped: exactly 0 and a zero row
        assert r[n + 1] != 0.0 and r[n + 2] != 0.0 and r[n + 3] == 0.0
        assert np.all(j[n + 3] == 0.0)
    finally:
        dint.close()
        dev.close()


# ============================ solves ==========================================================
@pytest.mark.parametrize("name,seed,opts,branches", RC.SOLVES_2D, ids=[c[0] for c in RC.SOLVES_2D])
def test_solve2d_branches(sm, oracle, name, seed, opts, branches):
    cells, res, mx, my, cloud, tgt, init = RC.problem2d(seed)
    grid = oracle.Grid2D(cells, res, mx, my)
    want = oracle.ceres2d_match(grid, cloud, tgt, init, trace=True, **opts)
    RC.assert_reaches(want, branches)
    dev = sm.RealTimeGrid2D(grid)
    try:
        pose, s = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(**opts)).Match(tgt, init, cloud, dev)
        same_solution(pose, s, want)
    finally:
        dev.close()


def test_solve2d_gradient_tolerance_before_the_first_step(sm, oracle):
    """Every point a grid-width outside and the pose on its target: the gradient is exactly 0."""
    cells, res, mx, my, _, _, _ = RC.problem2d(1)
    grid = oracle.Grid2D(cells, res, mx, my)
    init = np.array([0.3, -0.2, 0.1])
    dev = sm.RealTimeGrid2D(grid)
    try:
        for n in (1, 257):
            cloud = RC.far_cloud2d(n)
            want = oracle.ceres2d_match(grid, cloud, init[:2], init, trace=True)
            RC.assert_reaches(want, ["gradient_at_start"])
            pose, s = sm.CeresScanMatcher2D().Match(init[:2], init, cloud, dev)
            same_solution(pose, s, want)
            assert np.array_equal(pose, init) and s["final_cost"] == s["initial_cost"]
    finally:
        dev.close()


@pytest.mark.parametrize("case", RC.SOLVES_TSDF, ids=[c[0] for c in RC.SOLVES_TSDF])
def test_solve_tsdf_branches(sm, case):
    g, p, want = RC.tsdf_want(case)
    RC.assert_reaches(want, case[5])
    _, dev = tsdf_pair(sm, p[0], p[1], p[2], p[3], p[4], p[5], p[6])
    try:
        m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(
            occupied_space_weight=20.0, translation_weight=1e-2, rotation_weight=1e-2,
            use_nonmonotonic_steps=case[3], max_num_iterations=case[4]))
        pose, s = m.Match(p[8], p[9], p[7], dev)
        same_solution(pose, s, want)
    finally:
        dev.close()


def test_solve_tsdf_trial_point_without_weight_and_parameter_tolerance(sm):
    """n = 1 on an island of weight: trial steps that leave it cost DBL_MAX and are rejected
    (as opposed to W == 0 at the start, which fails the solve); and stiff priors stop on the
    parameter tolerance."""
    from tests.test_tsdf2d_oracle_cpu import _island
    g, cloud = _island()
    dev = sm.RealTimeGrid2D(sm.TSDF2DSpec(g.tsd_cells, g.weight_cells, g.resolution, g.max_x,
                                          g.max_y, g.truncation_distance, g.max_weight))
    try:
        reached = 0
        for dx in np.linspace(-0.04, 0.04, 9):
            init = np.array([dx, 0.5 * dx, 0.0])
            trace = []
            want = T.match(g, cloud, init[:2], init, 20.0, 1e-3, 1e-3, True, 10, trace=trace)
            want["trace"] = trace
            if not RC.BRANCHES["trial_failure"](want):
                continue
            RC.assert_margins(want)
            reached += 1
            m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(20.0, 1e-3, 1e-3, True, 10))
            pose, s = m.Match(init[:2], init, cloud, dev)
            same_solution(pose, s, want)
        assert reached >= 1
        init = np.array([0.01, 0.005, 0.0])
        trace = []
        want = T.match(g, cloud, init[:2], init, 20.0, 1e6, 1e6, True, 50, trace=trace)
        want["trace"] = trace
        RC.assert_reaches(want, ["parameter_tolerance"])
        m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(20.0, 1e6, 1e6, True, 50))
        same_solution(*m.Match(init[:2], init, cloud, dev), want)
    finally:
        dev.close()


@pytest.mark.parametrize("case", RC.SOLVES_3D, ids=[c[0] for c in RC.SOLVES_3D])
def test_solve3d_branches(sm, oracle, case):
    (res, idx, val, hi, low, tgt, init), want = RC.want3d(oracle, case)
    RC.assert_reaches(want, case[5])
    _, dev = hybrid_pair(sm, oracle, res, idx, val)
    try:
        m = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
            use_nonmonotonic_steps=case[3], max_num_iterations=case[4], **RC.WEAK_PRIOR_3D))
        pairs = [(hi, dev)] + ([(low, dev)] if low is not None else [])
        pose, s = m.Match(tgt, init, pairs)
        same_solution(pose, s, want)
    finally:
        dev.close()


@pytest.mark.parametrize("case", RC.SOLVES_INTENSITY, ids=[c[0] for c in RC.SOLVES_INTENSITY])
def test_solve_intensity_branches(sm, oracle, case):
    name, seed, weight, huber, prior, nonmono, iters, branches = case
    (res, idx, val, hi, tgt, init, sums, counts, inten), want = RC.want_intensity(oracle, case)
    RC.assert_reaches(want, branches)
    # which branch of HuberLoss the block takes at the start: s_b against huber_scale^2
    igrid = iorc.IntensityHybridGrid(res, idx, sums, counts)
    r, _ = iorc.evaluate([(hi, oracle.HybridGrid(res, idx, val), igrid, inten)], init, tgt,
                         init[3:], [(weight, huber, RC.INTENSITY_THRESHOLD)], jacobian=False)
    s_b = float(np.sum(r[len(hi):2 * len(hi)] ** 2))
    assert (inten > RC.INTENSITY_THRESHOLD).any() and (inten < RC.INTENSITY_THRESHOLD).any()
    if huber == 0.05:
        assert s_b > 100 * huber * huber
    if huber == 50.0:
        assert s_b < 0.2 * huber * huber
    _, dev = hybrid_pair(sm, oracle, res, idx, val)
    dint = sm.DeviceIntensityGrid(sm.IntensityGridSpec(res, idx, sums, counts))
    try:
        m = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
            translation_weight=prior, rotation_weight=prior, use_nonmonotonic_steps=nonmono,
            max_num_iterations=iters,
            intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(
                weight, huber, RC.INTENSITY_THRESHOLD)))
        same_solution(*m.Match(tgt, init, [(hi, dev, dint, inten)]), want)
    finally:
        dint.close()
        dev.close()


# ============================ batches =========================================================
def test_batch2d_sizes_and_the_job_table_offset(sm, oracle):
    """One job; 2000 jobs of n = 1 .. 40 on one grid (more CTAs than SMs); very different n in
    one launch; a float count whose bytes are a multiple of 256, where the job table starts
    right after the clouds.  Every job equals its single call bit for bit."""
    cells, res, mx, my, _, _, _ = RC.problem2d(3)
    tsd, wgt = RC.problem_tsdf(3)[:2]
    pdev = sm.RealTimeGrid2D(oracle.Grid2D(cells, res, mx, my))
    _, tdev = tsdf_pair(sm, tsd, wgt, res, mx, my, 0.3)
    m = sm.CeresScanMatcher2D(sm.CeresScanMatcherOptions2D(max_num_iterations=12, **RC.WEAK_PRIOR))
    rng = np.random.RandomState(2)

    def job(n, dev):
        cloud = np.concatenate([rng.uniform(-0.6, 0.6, (n, 2)), np.zeros((n, 1))], 1).astype(F)
        init = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(-1, 1)])
        return dev, cloud, init

    def run(jobs):
        return m.MatchBatch([j[2][:2] * 0.5 for j in jobs], [j[2] for j in jobs],
                            [j[1] for j in jobs], [j[0] for j in jobs])
    try:
        many = [job(1 + k % 40, pdev) for k in range(2000)]
        assert len(many) > 132 * 8
        poses, sums = run(many)
        check = list(range(0, 2000, 97)) + [1999]
        mixed = [job(n, d) for n, d in ((1, pdev), (4096, tdev), (2, tdev), (513, pdev), (255, pdev),
                                        (256, tdev), (257, pdev))]
        aligned = [job(64, pdev), job(64, tdev)]              # 2 * 64 * 3 floats = 1536 bytes
        assert sum(len(j[1]) for j in aligned) * 12 % 256 == 0
        mp, ms = run(mixed)
        ap, as_ = run(aligned)
        singles = 0
        for jobs, ps, ss, which in ((many, poses, sums, check), (mixed, mp, ms, range(len(mixed))),
                                    (aligned, ap, as_, range(2))):
            for k in which:
                p1, s1 = run([jobs[k]])
                assert np.array_equal(ps[k], p1[0]) and ss[k] == s1[0], k
                singles += 1
        assert singles >= 30
        assert len({s["iterations"] for s in sums}) > 3       # the jobs are not all alike
    finally:
        pdev.close()
        tdev.close()


def test_batch3d_one_and_two_clouds_mixed(sm, oracle):
    res, idx, val, _, _, _, _ = RC.problem3d(3)
    _, dev = hybrid_pair(sm, oracle, res, idx, val)
    isums = np.random.RandomState(1).uniform(10, 90, len(idx)).astype(F)
    dint = sm.DeviceIntensityGrid(sm.IntensityGridSpec(res, idx, isums, np.ones(len(idx), np.int32)))
    rng = np.random.RandomState(8)
    io = sm.IntensityCostFunctionOptions(0.5, 0.3, 100.0)
    m = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
        max_num_iterations=12, intensity_cost_function_options_0=io, **RC.WEAK_PRIOR_3D))

    def job(n_hi, n_lo, intensity=False):
        hi = rng.uniform(-0.35, 0.35, (n_hi, 3)).astype(F)
        pairs = [(hi, dev, dint, rng.uniform(10, 120, n_hi).astype(F)) if intensity else (hi, dev)]
        if n_lo:
            pairs.append((rng.uniform(-0.35, 0.35, (n_lo, 3)).astype(F), dev))
        a = rng.uniform(-0.3, 0.3)
        init = np.array([*rng.uniform(-0.1, 0.1, 3), math.cos(a / 2), 0.0, math.sin(a / 2), 0.0])
        return init, pairs
    try:
        plain = [job(*n) for n in ((1, 0), (1, 257), (257, 1), (64, 0), (2048, 3), (33, 31))]
        plain += [job(1 + k % 40, k % 3) for k in range(300)]
        with_i = [job(1, 0, True), job(40, 257), job(257, 1, True), job(64, 64, True)]
        assert {len(p[1]) for p in plain} == {1, 2}
        for jobs in (plain, with_i, plain[:1]):
            poses, sums = m.MatchBatch([j[0][:3] for j in jobs], [j[0] for j in jobs],
                                       [j[1] for j in jobs])
            for k in (range(len(jobs)) if len(jobs) < 10 else list(range(8)) + list(range(8, 306, 37))):
                p1, s1 = m.Match(jobs[k][0][:3], jobs[k][0], jobs[k][1])
                assert np.array_equal(poses[k], p1) and sums[k] == s1, k
    finally:
        dint.close()
        dev.close()


# ============================ non-finite input ================================================
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_input_is_refused(sm, oracle, bad):
    """A NaN coordinate would reach static_cast<int>(floor(r)), lround and lroundf: every
    csm_ceres_* entry point returns CSM_E_INVALID for a non-finite point, pose or target."""
    from cartographer_b200._lib import CsmError
    cells, res, mx, my, cloud, tgt, init = RC.problem2d(3)
    pdev = sm.RealTimeGrid2D(oracle.Grid2D(cells, res, mx, my))
    tsd, wgt = RC.problem_tsdf(3)[:2]
    _, tdev = tsdf_pair(sm, tsd, wgt, res, mx, my, 0.3)
    r3, idx, val, hi, _, tgt3, init3 = RC.problem3d(3)
    _, hdev = hybrid_pair(sm, oracle, r3, idx, val)
    dint = sm.DeviceIntensityGrid(sm.IntensityGridSpec(r3, idx, np.ones(len(idx), F),
                                                       np.ones(len(idx), np.int32)))
    m2 = sm.CeresScanMatcher2D()
    m3 = sm.CeresScanMatcher3D(sm.CeresScanMatcherOptions3D(
        intensity_cost_function_options_0=sm.IntensityCostFunctionOptions(0.5, 0.3, 100.0)))

    def poked(a, k):
        a = np.array(a, dtype=np.asarray(a).dtype if hasattr(a, "dtype") else np.float64)
        a.reshape(-1)[k] = bad
        return a
    inten = np.full(len(hi), 50.0, F)
    try:
        for dev in (pdev, tdev):
            good = m2.Match(tgt, init, cloud, dev)
            for args in ((poked(tgt, 1), init, cloud), (tgt, poked(init, 2), cloud),
                         (tgt, init, poked(cloud, 3 * 17)), (tgt, init, poked(cloud, 3 * 59 + 2))):
                with pytest.raises(CsmError):
                    m2.Match(args[0], args[1], args[2], dev)
                with pytest.raises(CsmError):       # one bad job refuses the whole batch
                    m2.MatchBatch([tgt, args[0]], [init, args[1]], [cloud, args[2]], [dev, dev])
                with pytest.raises(CsmError):
                    m2.EvaluateChecked(dev, args[2], args[1], args[0], 0.0)
            with pytest.raises(CsmError):
                m2.EvaluateChecked(dev, cloud, init, tgt, bad)
            again = m2.Match(tgt, init, cloud, dev)          # the handle and lane still work
            assert np.array_equal(good[0], again[0]) and good[1] == again[1]
        with pytest.raises(CsmError):
            m2.Evaluate(pdev, poked(cloud, 0), init, tgt, 0.0)
        for pairs in ([(hi, hdev)], [(hi, hdev), (hi, hdev)], [(hi, hdev, dint, inten)]):
            good = m3.Match(tgt3, init3, pairs)
            bad_pairs = [(poked(hi, 3 * 5 + 1),) + tuple(pairs[-1][1:])] if len(pairs) == 1 else \
                [pairs[0], (poked(hi, 7), hdev)]
            for args in ((poked(tgt3, 2), init3, pairs), (tgt3, poked(init3, 4), pairs),
                         (tgt3, init3, bad_pairs)):
                with pytest.raises(CsmError):
                    m3.Match(*args)
                with pytest.raises(CsmError):
                    m3.Evaluate(args[2], args[1], args[0], [1, 0, 0, 0])
            again = m3.Match(tgt3, init3, pairs)
            assert np.array_equal(good[0], again[0]) and good[1] == again[1]
        with pytest.raises(CsmError):
            m3.Match(tgt3, init3, [(hi, hdev, dint, poked(inten, 9))])
    finally:
        for d in (pdev, tdev, hdev, dint):
            d.close()
