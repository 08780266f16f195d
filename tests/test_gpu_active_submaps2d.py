"""ActiveSubmaps2D on the device (csm_range_inserter2d_insert_submaps, scan_matching.py's
ActiveSubmaps2D and DeviceSubmap2D): after every scan, every active handle bit-equal to twin
handles fed by one single-grid Insert each and to the CPU lifecycle restatement
(tests/active_submaps2d_oracle.py); the one call's edges and refusals; ConstraintBuilder2D and
OverlappingSubmapsTrimmer2D on the finished submaps."""
import ctypes as C

import numpy as np
import pytest

from benchmarks import synthetic
from benchmarks.bench_insert2d import range_data, trajectory
from tests import active_submaps2d_oracle as A
from tests import insert2d_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


@pytest.fixture(scope="module")
def world():
    """bench_insert2d.py's world and trajectory: 1081-beam scans, 30 m range, misses at 5 m."""
    spec, occ = synthetic.make_grid2d(3, size_cells=1000)
    poses = trajectory(occ, spec, np.random.RandomState(11), 400)
    return spec, occ, poses


def _scan(world, k):
    spec, occ, poses = world
    origin, returns, misses = range_data(occ, spec, poses[k], seed=k)
    if k % 97 == 13:   # an accumulated multi-ring scan: 17 296 returns around the same origin
        rng = np.random.RandomState(k)
        extra = np.repeat(returns, -(-17296 // len(returns)), 0)[:17296].copy()
        extra[:, :2] += rng.uniform(-0.02, 0.02, (17296, 2)).astype(np.float32)
        returns = extra
    return origin, returns, misses


def _state(grid):
    st = grid.read()
    return st.cells, (st.resolution, st.max_x, st.max_y), st.known_cells_box


def assert_same(dev, other):
    a = _state(dev)
    if isinstance(other, O.Grid):
        b = (other.cells, other.limits[:3], other.known_box)
    else:
        b = _state(other)
    assert a[1] == b[1] and a[2] == b[2]
    np.testing.assert_array_equal(a[0], b[0])


# ---- the lifecycle ----
@pytest.mark.parametrize("free_space", [True, False])
def test_lifecycle_400_scans(sm, world, free_space):
    ins_opts = sm.ProbabilityGridRangeDataInserterOptions2D(0.55, 0.49, free_space)
    options = sm.SubmapsOptions2D(num_range_data=20,
                                  probability_grid_range_data_inserter_options=ins_opts)
    active = sm.ActiveSubmaps2D(options)
    oracle = A.ActiveSubmaps(20, 0.05, 0.55, 0.49, free_space)
    single = sm.ProbabilityGridRangeDataInserter2D(ins_opts)
    twins = {}   # id(submap) -> a twin handle fed by single-grid Insert calls
    finished = evicted = 0
    for k in range(400):
        origin, returns, misses = _scan(world, k)
        before = {id(s) for s in active.submaps()}
        submaps = active.InsertRangeData(origin, returns, misses)
        assert active.range_data_inserter.last_stats["host_syncs"] == 1
        event = oracle.insert_range_data(origin, returns, misses)
        evicted += event["evicted"] is not None
        for s in submaps:
            if id(s) not in twins:
                twins[id(s)] = sm.RealTimeGrid2D.empty(*sm.create_grid_limits(origin[:2], 0.05))
            if not s.insertion_finished or event["finished"] is not None:
                single.Insert(origin, returns, twins[id(s)], misses)
        for gone in before - {id(s) for s in submaps}:
            twins.pop(gone).close()
        assert [s.local_pose for s in submaps] == [o.local_pose for o in oracle.submaps]
        assert [s.num_range_data for s in submaps] == [o.num_range_data for o in oracle.submaps]
        assert [s.insertion_finished for s in submaps] == \
            [o.insertion_finished for o in oracle.submaps]
        for s, o in zip(submaps, oracle.submaps):
            if s.insertion_finished and event["finished"] is not None:
                finished += 1
                assert_same(s.grid, o.grid)                       # the crop
                crop = twins[id(s)].ComputeCroppedGrid()
                assert_same(s.grid, crop)
                crop.close()
            elif not s.insertion_finished:
                assert_same(s.grid, o.grid)
                assert_same(s.grid, twins[id(s)])
    assert finished >= 9 and evicted >= 9 and oracle._created >= 10
    single.close()


# ---- insert_submaps edges ----
def _pair(sm, free_space=True):
    opts = sm.ProbabilityGridRangeDataInserterOptions2D(0.55, 0.49, free_space)
    return sm.ProbabilityGridRangeDataInserter2D(opts), O.Inserter(0.55, 0.49, free_space)


def _check_call(sm, grids, oras, origin, returns, misses=None, free_space=True):
    """insert_submaps on `grids` against Insert on twins and the oracle on `oras`."""
    ins, ora_ins = _pair(sm, free_space)
    twins = []
    for o in oras:   # not from the handles: reading one would compute its stale known box
        res, max_x, max_y, _, _ = o.limits
        twins.append(sm.RealTimeGrid2D(synthetic.GridSpec(o.cells, res, max_x, max_y))
                     if o.known_box is not None else sm.RealTimeGrid2D.empty(*o.limits))
    ins.insert_submaps(grids, origin, returns, misses)
    assert ins.last_stats["host_syncs"] == 1
    for g, t, o in zip(grids, twins, oras):
        ins.Insert(origin, returns, t, misses)
        ora_ins.insert(origin, returns, o, misses)
        assert_same(g, o)
        assert_same(g, t)
        t.close()
    ins.close()


def _empties(sm, origins, resolutions):
    grids, oras = [], []
    for o, r in zip(origins, resolutions):
        ora = O.Grid.create_grid(o, r)
        grids.append(sm.RealTimeGrid2D.empty(*ora.limits))
        oras.append(ora)
    return grids, oras


@pytest.mark.parametrize("count", [1, 2, 3])
def test_one_two_three_handles(sm, world, count):
    origin, returns, misses = _scan(world, 5)
    grids, oras = _empties(sm, [origin[:2] + 0.3 * k for k in range(count)], [0.05] * count)
    for k in range(3):
        origin, returns, misses = _scan(world, 5 + k)
        _check_call(sm, grids, oras, origin, returns, misses)


def test_handles_of_different_resolutions(sm, world):
    origin, returns, misses = _scan(world, 40)
    grids, oras = _empties(sm, [origin[:2]] * 3, [0.05, 0.1, 0.025])
    for k in range(2):
        origin, returns, misses = _scan(world, 40 + k)
        _check_call(sm, grids, oras, origin, returns, misses)


def test_two_handles_made_from_cells(sm, world):
    """Both handles' known boxes are stale when the call starts: each needs its own staging."""
    spec, occ, _ = world
    grids, oras = [], []
    for (x0, y0, w, h) in [(300, 320, 160, 120), (500, 450, 90, 200)]:
        sub, _ = synthetic.crop_grid(spec, occ, x0, y0, w, h)
        cells = sub.cells.copy()
        cells[:7, :] = 0
        cells[:, -11:] = 0
        grids.append(sm.RealTimeGrid2D(synthetic.GridSpec(cells, sub.resolution, sub.max_x,
                                                          sub.max_y)))
        oras.append(O.Grid(sub.resolution, sub.max_x, sub.max_y, cells.shape[1], cells.shape[0],
                           cells))
    # a short scan near the first grid
    origin = np.float32([oras[0].limits[1] - 3.0, oras[0].limits[2] - 2.0, 0])
    returns = origin + np.float32([[0.4, 0.1, 0], [-0.2, 0.3, 0]])
    _check_call(sm, grids, oras, origin, returns, returns[:1] * np.float32([1, 1, 0]))
    boxes = [g.read().known_cells_box for g in grids]
    assert boxes[0] != boxes[1]


@pytest.mark.parametrize("side", range(4))
def test_one_handle_grows_the_other_not(sm, side):
    big, small = O.Grid.create_grid([0.0, 0.0], 0.05), O.Grid.create_grid([0.0, 0.0], 0.2)
    grids = [sm.RealTimeGrid2D.empty(*big.limits), sm.RealTimeGrid2D.empty(*small.limits)]
    far = [[4.0, 0.1], [0.1, 4.0], [-4.0, -0.1], [-0.1, -4.0]][side]
    returns = np.float32([far + [0.0], [0.3, 0.2, 0.0]])
    _check_call(sm, grids, [big, small], [0.0, 0.0, 0.0], returns)
    assert grids[0].shape[0] > 100 and grids[1].shape == (100, 100)


@pytest.mark.parametrize("free_space", [True, False])
def test_returns_only_misses_only_neither(sm, world, free_space):
    origin, returns, misses = _scan(world, 60)
    grids, oras = _empties(sm, [origin[:2], origin[:2] + 0.7], [0.05, 0.05])
    empty = np.zeros((0, 3), np.float32)
    _check_call(sm, grids, oras, origin, returns, None, free_space)
    _check_call(sm, grids, oras, origin, empty, misses, free_space)
    _check_call(sm, grids, oras, origin + np.float32([0.4, 0, 0]), empty, None, free_space)


def test_exact_corner_rays(sm):
    r = 0.05
    grids, oras = _empties(sm, [[0.0, 0.0], [0.025, -0.025]], [r, r])
    _, max_x, max_y, _, _ = oras[0].limits
    border = lambda k: float(np.float32(max_x - k * r))  # noqa: E731
    o = np.float32([border(50), border(50), 0])
    pts = [[o[0] + 0.5, o[1] + 0.5], [o[0] - 0.5, o[1] + 0.5], [o[0] + 0.75, o[1] - 0.75],
           [border(30), border(62)], [border(71), border(40)], [border(44), border(44)],
           [o[0], o[1] + 1.0], [o[0] + 0.8, o[1]], [o[0] + 0.01, o[1] + 0.01]]
    ret = np.float32([[x, y, 0] for x, y in pts])
    _check_call(sm, grids, oras, o, ret, ret[::-1] * np.float32([1.01, 0.99, 0]))


# ---- refusals ----
def test_refusals_leave_every_handle_unchanged(sm, world):
    origin, returns, misses = _scan(world, 80)
    ins, _ = _pair(sm)
    grids, _ = _empties(sm, [origin[:2], origin[:2] + 0.5], [0.05, 0.05])
    ins.insert_submaps(grids, origin, returns, misses)
    before = [_state(g) for g in grids]
    lib = sm.lib()
    f = lib.csm_range_inserter2d_insert_submaps
    p = lambda a: np.ascontiguousarray(a, np.float32).ctypes.data_as(C.POINTER(C.c_float))  # noqa
    o, r, m = (np.ascontiguousarray(a, np.float32) for a in (origin, returns, misses))
    hs = lambda *g: (C.c_void_p * len(g))(*g)  # noqa: E731

    def call(org, ret, mis, handles, count):
        return f(ins._h, p(org), p(ret), len(ret), p(mis), len(mis), handles, count, None)

    both = hs(grids[0]._h, grids[1]._h)
    assert call(o, r, m, None, 2) == 1
    assert call(o, r, m, hs(grids[0]._h, None), 2) == 1
    assert call(o, r, m, both, 0) == 1
    assert call(o, r, m, hs(grids[0]._h, grids[1]._h, grids[0]._h), 3) == 1
    tsdf, _ = synthetic.make_tsdf2d(3, size_cells=64)
    tg = sm.RealTimeGrid2D(tsdf)
    assert call(o, r, m, hs(grids[0]._h, tg._h), 2) == 1
    tg.close()
    # past 30000 cells at 1 cm, while it fits at 5 cm
    fine = sm.RealTimeGrid2D.empty(*O.Grid.create_grid(origin[:2], 0.01).limits)
    far = np.float32([origin + np.float32([200.0, 0, 0])])
    assert call(o, far, np.zeros((0, 3), np.float32), hs(grids[0]._h, fine._h), 2) == 1
    fine_before = _state(fine)
    for bad in (0, 1, 2):
        oo, rr, mm = o.copy(), r.copy(), m.copy()
        [oo, rr, mm][bad].reshape(-1)[4 if bad else 1] = np.nan
        assert call(oo, rr, mm, both, 2) == 1
    assert call(o, r, np.float32([[np.inf, 0, 0]]), both, 2) == 1
    for g, b in zip(grids, before):
        a = _state(g)
        assert a[1:] == b[1:]
        np.testing.assert_array_equal(a[0], b[0])
    a = _state(fine)
    assert a[1:] == fine_before[1:] and np.array_equal(a[0], fine_before[0])
    fine.close()
    ins.insert_submaps(grids, origin, returns, misses)   # still usable


@pytest.mark.skipif("__import__('cartographer_b200').scan_matching.device_count() < 2")
def test_handle_on_another_device_is_refused(sm, world):
    origin, returns, misses = _scan(world, 81)
    ins, _ = _pair(sm)
    lim = O.Grid.create_grid(origin[:2], 0.05).limits
    g0, g1 = sm.RealTimeGrid2D.empty(*lim), sm.RealTimeGrid2D.empty(*lim, device=1)
    from cartographer_b200._lib import CsmError
    with pytest.raises(CsmError):
        ins.insert_submaps([g0, g1], origin, returns, misses)
    assert g0.read().known_cells_box is None


# ---- loop closure and trimming on the finished submaps ----
def _bits(result):
    return [(c.submap_id, c.node_id, np.float32(c.score).tobytes(),
             np.array(c.zbar_ij, np.float64).tobytes()) for c in result]


def test_constraint_builder_and_trimmer_on_finished_submaps(sm, world):
    from cartographer_b200 import constraint_builder as cb
    from cartographer_b200 import pose_graph as pg
    from tests import trimmer2d_cases as K
    spec, occ, poses = world
    active = sm.ActiveSubmaps2D(sm.SubmapsOptions2D(num_range_data=10))
    submaps, graph = {}, K.FakePoseGraph()
    for k in range(45):
        origin, returns, misses = range_data(occ, spec, poses[k], seed=k)
        graph.nodes[(0, k)] = K.Node(time=k)
        for s in active.InsertRangeData(origin, returns, misses):
            sid = (0, next((i for i, t in submaps.items() if t is s), len(submaps)))
            submaps[sid[1]] = s
            graph.constraints.append(K.Constraint(sid, (0, k), "INTRA_SUBMAP"))
    finished = {i: s for i, s in submaps.items() if s.insertion_finished}
    assert len(finished) >= 2
    opts = cb.ConstraintBuilderOptions(
        sampling_ratio=1.0, max_constraint_distance=50.0, min_score=0.3,
        global_localization_min_score=0.3, linear_search_window=1.0,
        angular_search_window=0.3, branch_and_bound_depth=5, ceres_scan_matcher_options=None)
    device_views = {(0, i): s.constraint_builder_submap() for i, s in finished.items()}
    host_views = {sid: cb.Submap2D(v.grid.read(), v.local_pose) for sid, v in device_views.items()}
    results = []
    for views in (device_views, host_views):
        b = cb.ConstraintBuilder2D(opts)
        for n in range(0, 40, 4):
            cloud = synthetic.cast_scan(occ, spec, poses[n], beams=361, max_range=8.0, seed=500 + n)
            start = (poses[n][0] + 0.05, poses[n][1] - 0.06, poses[n][2] + 0.03)
            for sid in sorted(views):
                rel = cb._compose(cb._inverse(tuple(views[sid].local_pose)), start)
                b.MaybeAddConstraint(sid, views[sid], (0, n), cloud, rel)
            b.NotifyEndOfNode()
        results.append(_bits(b.WhenDone(lambda r: None)))
    assert results[0] == results[1] and len(results[0]) > 0
    # OverlappingSubmapsTrimmer2D over a pose graph whose submaps are these objects, against
    # the restatement's trimmer over their read-back grids
    for i, s in submaps.items():
        graph.submap_data[(0, i)] = K.SubmapData(submap=s, pose=list(s.local_pose))
    host = K.FakePoseGraph(nodes=graph.nodes, constraints=graph.constraints)
    for sid, d in graph.submap_data.items():
        st = d.submap.grid.read()
        grid = K.HostGrid(st.cells, st.known_cells_box, (st.max_x, st.max_y, st.resolution))
        host.submap_data[sid] = K.SubmapData(
            K.Submap(grid, list(d.submap.local_pose), d.submap.insertion_finished), d.pose)
    dev_trimmer = pg.OverlappingSubmapsTrimmer2D(1, 0.0, 0)
    dev_trimmer.Trim(graph)
    K.OracleTrimmer(1, 0.0, 0).Trim(host)
    assert graph.trimmed == host.trimmed and dev_trimmer.last_stats is not None
