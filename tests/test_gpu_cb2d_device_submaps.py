"""ConstraintBuilder2D on device-resident submaps: finished ProbabilityGrid submaps grown by
ProbabilityGridRangeDataInserter2D and cropped on the device, passed to the builder as
RealTimeGrid2D handles.  The constraints must equal, bit for bit and in the same order, those
of the same builder fed host submaps made from the cells read back, and those of the CPU
restatement (tests/insert2d_oracle.cc for the grid, the oracle matcher and CeresMatch2D for
the constraints)."""
import numpy as np
import pytest

from benchmarks import synthetic
from cartographer_b200 import constraint_builder as cb
from tests import insert2d_oracle as O
from tests.test_constraint_builder_cpu import OracleExecutor
from tests.test_gpu_insert2d import _world_scan

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


def _grow(sm, occ, spec, poses, seed, max_range=8.0):
    """One finished submap from the same 1081-beam scans on the device and in the restatement:
    (cropped RealTimeGrid2D, cropped restatement Grid)."""
    ins = sm.ProbabilityGridRangeDataInserter2D(sm.ProbabilityGridRangeDataInserterOptions2D())
    ora_ins = O.Inserter(0.55, 0.49, True)
    ora = O.Grid.create_grid(poses[0][:2], 0.05)
    dev = sm.RealTimeGrid2D.empty(*ora.limits)
    for k, pose in enumerate(poses):
        origin, returns, misses = _world_scan(occ, spec, pose, seed=seed + k, max_range=max_range)
        ins.Insert(origin, returns, dev, misses)
        ora_ins.insert(origin, returns, ora, misses)
    crop, ora_crop = dev.ComputeCroppedGrid(), ora.crop()
    for h in (dev, ins, ora, ora_ins):
        h.close()
    np.testing.assert_array_equal(crop.read().cells, ora_crop.cells)
    return crop, ora_crop


def _spec(ora_grid):
    res, max_x, max_y, _, _ = ora_grid.limits
    return synthetic.GridSpec(ora_grid.cells, res, max_x, max_y)


@pytest.fixture(scope="module")
def world(sm):
    """Three device submaps with their local poses, their restated twins, and four nodes
    (cloud, true pose) in a 30 m synthetic world."""
    spec, occ = synthetic.make_grid2d(21, size_cells=600)
    rng = np.random.RandomState(7)
    centres = [synthetic.random_free_pose(occ, spec, rng, margin_cells=80) for _ in range(3)]
    grown = []
    for s, c in enumerate(centres):
        scans = [c + np.array([0.15 * k, -0.1 * k, 0.05 * k]) for k in range(8)]
        grown.append(_grow(sm, occ, spec, scans, seed=100 * s))
    local_poses = [(float(c[0]), float(c[1]), 0.1 * s) for s, c in enumerate(centres)]
    nodes = []
    for n in range(4):
        pose = centres[n % 3] + np.array([0.4, -0.3, 0.05]) * (1 + n // 3)
        nodes.append((synthetic.cast_scan(occ, spec, pose, beams=361, max_range=8.0, seed=500 + n),
                      tuple(float(v) for v in pose)))
    yield grown, local_poses, nodes
    for crop, ora in grown:
        crop.close()
        ora.close()


def _options(refine, sm, **kw):
    base = dict(sampling_ratio=1.0, max_constraint_distance=50.0, min_score=0.3,
                global_localization_min_score=0.3, linear_search_window=1.0,
                angular_search_window=0.3, branch_and_bound_depth=5,
                ceres_scan_matcher_options=sm.CeresScanMatcherOptions2D() if refine else None)
    base.update(kw)
    return cb.ConstraintBuilderOptions(**base)


def _fill(builder, submaps, nodes, which=None, global_constraints=True):
    """Every node against every submap of `which` (all by default), from a start 8 cm and
    0.03 rad off its true pose; a global constraint per node."""
    ids = sorted(submaps) if which is None else which
    for n, (cloud, pose) in enumerate(nodes):
        start = (pose[0] + 0.05, pose[1] - 0.06, pose[2] + 0.03)
        for sid in ids:
            rel = cb._compose(cb._inverse(tuple(submaps[sid].local_pose)), start)
            builder.MaybeAddConstraint(sid, submaps[sid], (0, n), cloud, rel)
        if global_constraints:
            sid = ids[n % len(ids)]
            builder.MaybeAddGlobalConstraint(sid, submaps[sid], (0, n), cloud)
        builder.NotifyEndOfNode()


def _submaps(world, host):
    grown, local_poses, _ = world
    return {(0, s): cb.Submap2D(crop.read() if host else crop, local_poses[s])
            for s, (crop, _) in enumerate(grown)}


def _bits(result):
    return [(c.submap_id, c.node_id, np.float32(c.score).tobytes(),
             np.array(c.zbar_ij, np.float64).tobytes()) for c in result]


def _drain(opts, submaps, nodes, **kw):
    b = cb.ConstraintBuilder2D(opts)
    _fill(b, submaps, nodes, **kw)
    calls = []
    got = b.WhenDone(lambda r: calls.append(r))
    assert calls == [got]
    return b, got


# ---- 1. the same results as host submaps ----
@pytest.mark.parametrize("global_constraints", [False, True])
@pytest.mark.parametrize("refine", [False, True])
def test_same_constraints_as_host_submaps(sm, world, refine, global_constraints):
    opts = _options(refine, sm)
    nodes = world[2]
    dev, got = _drain(opts, _submaps(world, False), nodes, global_constraints=global_constraints)
    host, want = _drain(opts, _submaps(world, True), nodes,
                        global_constraints=global_constraints)
    assert len(want) >= 6
    assert _bits(got) == _bits(want)
    assert dev.executor.stats["candidates_scored"] == host.executor.stats["candidates_scored"]
    assert dev.executor.stats["refined"] == host.executor.stats["refined"]
    if refine:
        assert dev.executor.stats["refined"] > 0
        assert dev.executor.grids == {}    # the device submaps were not uploaded again
        assert set(host.executor.grids) == {c.submap_id for c in want}
    for b in (dev, host):
        for sid in list(b.executor.matchers):
            b.DeleteScanMatcher(sid)


# ---- 2. against the restatement ----
def _against_oracle(sm, submaps, oracle_submaps, nodes, opts, fill_kw):
    from oracle import pyoracle
    dev, got = _drain(opts, submaps, nodes, **fill_kw)
    ref = cb.ConstraintBuilder2D(opts, executor=OracleExecutor(opts))
    _fill(ref, oracle_submaps, nodes, **fill_kw)
    want = ref.WhenDone(lambda r: None)
    assert len(want) > 0
    # found flags: every queued pair has a record on both sides
    assert [bool(r["found"]) for r in dev.last_records] == \
        [bool(r["found"]) for r in ref.last_records]
    assert _bits(got) == _bits(want)    # scores and pose estimates, bit for bit
    # CeresScanMatcher2D on the device from the same estimates, against the restatement
    co = sm.CeresScanMatcherOptions2D()
    ropts = cb.ConstraintBuilderOptions(**dict(opts.__dict__, ceres_scan_matcher_options=co))
    _, refined = _drain(ropts, submaps, nodes, **fill_kw)
    assert [(c.submap_id, c.node_id, c.score) for c in refined] == \
        [(c.submap_id, c.node_id, c.score) for c in want]
    clouds = {n: cloud for n, (cloud, _) in enumerate(nodes)}
    worst = 0.0
    for c, w in zip(refined, want):
        lp = tuple(oracle_submaps[c.submap_id].local_pose)
        estimate = cb._compose(lp, w.zbar_ij)
        g = oracle_submaps[c.submap_id].grid
        og = pyoracle.Grid2D(g.cells, g.resolution, g.max_x, g.max_y)
        r = pyoracle.ceres2d_match(og, clouds[c.node_id[1]], estimate[:2], estimate,
                                   co.occupied_space_weight, co.translation_weight,
                                   co.rotation_weight, co.use_nonmonotonic_steps,
                                   co.max_num_iterations)
        worst = max(worst, float(np.abs(np.array(cb._compose(lp, c.zbar_ij)) - r["pose"]).max()))
    assert worst < 1e-7, worst     # DESIGN §6c
    return dev


def test_against_the_restatement(sm, world):
    grown, local_poses, nodes = world
    oracle_submaps = {(0, s): cb.Submap2D(_spec(ora), local_poses[s])
                      for s, (_, ora) in enumerate(grown)}
    dev = _against_oracle(sm, _submaps(world, False), oracle_submaps, nodes, _options(False, sm),
                          {})
    for sid in list(dev.executor.matchers):
        dev.DeleteScanMatcher(sid)


def test_config4_sized_submap_against_the_restatement(sm):
    """A submap of about 1000 x 1000 cells at 5 cm, depth 7, a 7 m / 30° window, 50 pairs."""
    spec, occ = synthetic.make_grid2d(4, size_cells=1000)
    rng = np.random.RandomState(4)
    poses = [synthetic.random_free_pose(occ, spec, rng, margin_cells=100) for _ in range(60)]
    crop, ora = _grow(sm, occ, spec, poses[:10], seed=4000, max_range=30.0)
    assert min(ora.limits[3:]) >= 900
    nodes = [(synthetic.cast_scan(occ, spec, p, beams=181, max_range=30.0, seed=4100 + n),
              tuple(float(v) for v in p)) for n, p in enumerate(poses[10:60])]
    opts = cb.ConstraintBuilderOptions(sampling_ratio=1.0, max_constraint_distance=100.0,
                                       min_score=0.4, linear_search_window=7.0,
                                       angular_search_window=np.radians(30.0),
                                       branch_and_bound_depth=7)
    local = (float(poses[0][0]), float(poses[0][1]), 0.0)
    dev = _against_oracle(sm, {(0, 0): cb.Submap2D(crop, local)},
                          {(0, 0): cb.Submap2D(_spec(ora), local)}, nodes, opts,
                          {"global_constraints": False})
    assert dev.executor.stats["searched"] == 50
    dev.DeleteScanMatcher((0, 0))
    crop.close()
    ora.close()


# ---- 3. mixed queues ----
def test_mixed_queue_equals_two_drains(sm, world):
    opts = _options(True, sm)
    nodes = world[2]
    mixed = dict(_submaps(world, False))
    mixed[(0, 1)] = _submaps(world, True)[(0, 1)]
    _, together = _drain(opts, mixed, nodes, global_constraints=False)
    _, dev_only = _drain(opts, mixed, nodes, which=[(0, 0), (0, 2)], global_constraints=False)
    _, host_only = _drain(opts, mixed, nodes, which=[(0, 1)], global_constraints=False)
    assert len(together) == len(dev_only) + len(host_only) > 0
    key = lambda b: (b[1], b[0])  # noqa: E731  (node, submap): the queue's order
    assert _bits(together) == sorted(_bits(dev_only) + _bits(host_only), key=key)


# ---- 4. handles the inserter did not make ----
def _same_as_host(sm, handle, host_grid, nodes, refine, **kw):
    opts = _options(refine, sm, **kw)
    _, got = _drain(opts, {(0, 0): cb.Submap2D(handle, (0.2, -0.1, 0.05))}, nodes)
    _, want = _drain(opts, {(0, 0): cb.Submap2D(host_grid, (0.2, -0.1, 0.05))}, nodes)
    assert _bits(got) == _bits(want)
    return got


@pytest.mark.parametrize("refine", [False, True])
def test_uncropped_handle_with_a_row_pitch(sm, refine):
    spec, occ = synthetic.make_grid2d(21, size_cells=600)
    # 203 cells a row in a row pitch of 208
    sub, sub_occ = synthetic.crop_grid(spec, occ, 150, 140, 203, 157)
    handle = sm.RealTimeGrid2D(sub)
    np.testing.assert_array_equal(handle.read().cells, sub.cells)
    rng = np.random.RandomState(3)
    nodes = []
    for n in range(3):   # scans taken inside the grid
        pose = synthetic.random_free_pose(sub_occ, sub, rng, margin_cells=30)
        nodes.append((synthetic.cast_scan(sub_occ, sub, pose, beams=361, max_range=5.0, seed=n),
                      tuple(float(v) for v in pose)))
    # a sparse corner of the world: its scans score about 0.2
    got = _same_as_host(sm, handle, sub, nodes, refine, min_score=0.1,
                        global_localization_min_score=0.1)
    assert len(got) > 0
    handle.close()


def test_one_cell_crop_of_an_empty_grid(sm, world):
    empty = sm.RealTimeGrid2D.empty(0.05, 2.5, 2.5)
    crop = empty.ComputeCroppedGrid()
    st = crop.read()
    assert st.cells.shape == (1, 1) and st.known_cells_box is None
    assert _same_as_host(sm, crop, st, world[2][:2], True) == []   # nothing above min_score
    empty.close()
    crop.close()


# ---- 5. lifetime ----
def test_lifetime(sm, world):
    opts = _options(True, sm)
    nodes = world[2]
    submaps = _submaps(world, False)
    before = {sid: s.grid.read().cells.copy() for sid, s in submaps.items()}
    b = cb.ConstraintBuilder2D(opts)
    _fill(b, submaps, nodes)
    first = b.WhenDone(lambda r: None)
    for sid in submaps:
        b.DeleteScanMatcher(sid)
    assert b.executor.matchers == {}
    for sid, s in submaps.items():   # the handles are untouched and still usable
        np.testing.assert_array_equal(s.grid.read().cells, before[sid])
    _fill(b, submaps, nodes)
    again = b.WhenDone(lambda r: None)
    assert set(b.executor.matchers) == set(submaps)   # rebuilt from the handles
    assert _bits(again) == _bits(first)

    # a handle of our own that is closed once its drain's callback has run
    grown, local_poses, _ = world
    extra = grown[0][0].ComputeCroppedGrid()      # a crop of a crop: the same cells
    b.MaybeAddConstraint((1, 0), cb.Submap2D(extra, local_poses[0]), (0, 9), nodes[0][0],
                         cb._compose(cb._inverse(local_poses[0]), nodes[0][1]))
    b.NotifyEndOfNode()
    b.WhenDone(lambda r: None)
    extra.close()      # its stack keeps its own levels; the builder never reads the handle again
    _fill(b, submaps, nodes)
    assert _bits(b.WhenDone(lambda r: None)) == _bits(first)
    for sid in list(b.executor.matchers):
        b.DeleteScanMatcher(sid)


# ---- 6. refusals on the device ----
def _refuses(sm, monkeypatch, builder, grid):
    def no_launch(*args, **kwargs):
        raise AssertionError("the library was called")
    with monkeypatch.context() as m:
        m.setattr(sm, "lib", no_launch)
        with pytest.raises(ValueError):
            builder.MaybeAddConstraint((0, 0), cb.Submap2D(grid), (0, 0), np.zeros((1, 3)),
                                       (0.0, 0.0, 0.0))
        with pytest.raises(ValueError):
            builder.MaybeAddGlobalConstraint((0, 0), cb.Submap2D(grid), (0, 0), np.zeros((1, 3)))
    assert builder._jobs == [] and builder._submaps == {}


def test_tsdf_handle_is_refused(sm, monkeypatch):
    tsdf = sm.RealTimeGrid2D.empty_tsdf(0.05, 2.5, 2.5, 0.3, 10.0)
    _refuses(sm, monkeypatch, cb.ConstraintBuilder2D(_options(False, sm)), tsdf)
    tsdf.close()


def test_multi_rank_builder_refuses_device_submaps(sm, world, monkeypatch):
    ctx = object.__new__(sm.MultiGpuContext)   # its world, without a communicator
    ctx.world_size, ctx.rank, ctx.device = 2, 0, 0
    _refuses(sm, monkeypatch, cb.ConstraintBuilder2D(_options(False, sm), context=ctx),
             world[0][0][0])


def test_handle_on_another_device_is_refused(sm, monkeypatch):
    if sm.device_count() < 2:
        pytest.skip("needs two devices")
    other = sm.RealTimeGrid2D.empty(0.05, 2.5, 2.5, device=1)
    _refuses(sm, monkeypatch, cb.ConstraintBuilder2D(_options(False, sm), device=0), other)
    other.close()
