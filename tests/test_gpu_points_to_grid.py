"""The map-writing stages on the device: csm_rt_grid2d_draw against the DrawProbabilityGrid
restatement (tests/probability_grid_draw_oracle.cc), the 2D stage's grid against the insert
restatement (tests/insert2d_oracle.cc) after every batch of seeded streams that grow it on every
side, its PNG pixels and PB bytes, the 3D stage's proto bytes against tests/insert3d_oracle.py and
tests/grid_proto_ref.py, refusals, and the stages' Flush chain and file names."""
import ctypes as C
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import grid_proto_ref as R
from tests import insert2d_oracle as I2
from tests import insert3d_oracle as I3
from tests import probability_grid_draw_oracle as O

pytestmark = pytest.mark.gpu

HIT, MISS = 0.55, 0.49                   # trajectory_builder_2d.lua's range_data_inserter
INSERT3D = dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
                intensity_threshold=40.0)   # trajectory_builder_3d.lua
CSM_E_INVALID, CSM_E_CAPACITY = 1, 3


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


@pytest.fixture(scope="module")
def pp():
    from cartographer_b200 import points_processing
    return points_processing


@pytest.fixture(scope="module")
def lib():
    from cartographer_b200._lib import lib as L
    return L()


class Files:
    """A file_writer_factory that keeps every file's bytes by name."""

    def __init__(self):
        self.data, self.closed = {}, []

    def __call__(self, name):
        files = self

        class Writer:
            def write(self, b):
                files.data[name] = files.data.get(name, b"") + bytes(b)

            def close(self):
                files.closed.append(name)
        self.data[name] = b""
        return Writer()


class Next:
    """A `next` stage that counts batches and answers Flush with `result`."""

    def __init__(self, pp, result=None):
        self.batches, self.flushes = 0, 0
        self.result = result or pp.FlushResult.kFinished

    def Process(self, batch):
        self.batches += 1

    def Flush(self):
        self.flushes += 1
        return self.result


@pytest.fixture(scope="module")
def world():
    spec, occ = synthetic.make_grid2d(21, size_cells=600)
    rng = np.random.RandomState(7)
    poses = [synthetic.random_free_pose(occ, spec, rng, margin_cells=40) for _ in range(500)]
    # the world centred on the origin, where CreateProbabilityGrid centres its 100 x 100 cells
    centre = np.array([spec.max_x - 0.5 * occ.shape[0] * spec.resolution,
                       spec.max_y - 0.5 * occ.shape[1] * spec.resolution])
    return spec, occ, poses, centre


def _batch(pp, world, k):
    """Batch k of the stream: a 1081-beam scan cast from pose k, in the map frame; beams that
    found nothing end at max_range and count as points, as the assets writer's batches do."""
    spec, occ, poses, centre = world
    pose = poses[k]
    pts = synthetic.cast_scan(occ, spec, pose, beams=1081, max_range=8.0, seed=k)
    c, s = math.cos(pose[2]), math.sin(pose[2])
    xy = np.stack([c * pts[:, 0] - s * pts[:, 1], s * pts[:, 0] + c * pts[:, 1]], 1) + \
        (pose[:2] - centre)
    z = np.full((len(xy), 1), 0.1 * (k % 3))
    origin = np.float32([pose[0] - centre[0], pose[1] - centre[1], 0.2])
    return pp.PointsBatch(np.concatenate([xy, z], 1), origin=origin, start_time=k)


def _oracle_grid(resolution):
    half = 0.5 * 100 * resolution
    return I2.Grid(resolution, half, half, 100, 100)


def _assert_grid(grid, ora):
    st = grid.read()
    res, max_x, max_y, nx, ny = ora.limits
    assert (st.resolution, st.max_x, st.max_y, st.cells.shape) == (res, max_x, max_y, (ny, nx))
    np.testing.assert_array_equal(st.cells, ora.cells)
    assert st.known_cells_box == ora.known_box
    return st


def _assert_drawn(grid, ora):
    pixels, offset = grid.draw()
    want, want_offset = O.draw(ora.cells, ora.known_box)
    assert offset == want_offset
    np.testing.assert_array_equal(pixels, want)
    return pixels


# ---- 2D: the stage's grid, image and proto along seeded streams ----
@pytest.mark.parametrize("free_space,batches", [(True, 200), (False, 50)],
                         ids=["free_space", "no_free_space"])
def test_stream_grid_image_and_proto(sm, pp, world, free_space, batches):
    opts = sm.ProbabilityGridRangeDataInserterOptions2D(HIT, MISS, free_space)
    files = Files()
    png = pp.ProbabilityGridPointsProcessor(0.05, opts, "map", "png", files)
    pb = pp.ProbabilityGridPointsProcessor(0.05, opts, "map", "pb", files)
    ora, ins = _oracle_grid(0.05), I2.Inserter(HIT, MISS, free_space)
    for k in range(batches):
        batch = _batch(pp, world, k)
        png.Process(batch)
        pb.Process(batch)
        ins.insert(batch.origin, batch.points, ora)
        assert png.inserter.last_stats["host_syncs"] == 1
        _assert_grid(png.grid, ora)
        if k % 25 == 0 or k == batches - 1:
            _assert_drawn(png.grid, ora)
    _, max_x, max_y, nx, ny = ora.limits
    assert nx >= 800                               # 100 cells doubled at least three times
    pixels = _assert_drawn(png.grid, ora)
    assert len(np.unique(pixels)) > 5
    assert png.Flush() == pp.FlushResult.kFinished and pb.Flush() == pp.FlushResult.kFinished
    np.testing.assert_array_equal(pp.decode_png(files.data["map.png"]), pp.cairo_to_rgb(pixels))
    assert files.data["map.pb"] == R.grid2d_message(ora.cells, 0.05, max_x, max_y, ora.known_box)
    assert sorted(files.closed) == ["map.pb", "map.png"]


def test_stream_reaching_30000_cells_is_refused(sm, pp, world):
    from cartographer_b200._lib import CsmError
    stage = pp.ProbabilityGridPointsProcessor(0.05, sm.ProbabilityGridRangeDataInserterOptions2D(),
                                              "map", "png", Files())
    ora, ins = _oracle_grid(0.05), I2.Inserter(HIT, MISS, True)
    for k in range(3):
        batch = _batch(pp, world, k)
        stage.Process(batch)
        ins.insert(batch.origin, batch.points, ora)
    before = _assert_grid(stage.grid, ora)
    far = pp.PointsBatch(np.float32([[900.0, 0.0, 0.0], [1.0, 1.0, 0.0]]))   # 1.5 km is 30000
    with pytest.raises(CsmError):
        stage.Process(far)
    after = _assert_grid(stage.grid, ora)
    assert after.cells.shape == before.cells.shape
    batch = _batch(pp, world, 3)                   # still usable
    stage.Process(batch)
    ins.insert(batch.origin, batch.points, ora)
    _assert_grid(stage.grid, ora)
    _assert_drawn(stage.grid, ora)


def test_pitched_handle(sm, pp, world):
    # 100 cells per row live in rows of 104; a handle made from 37 x 23 cells in rows of 40
    stage = pp.ProbabilityGridPointsProcessor(0.05, sm.ProbabilityGridRangeDataInserterOptions2D(),
                                              "map", "png", Files())
    ora, ins = _oracle_grid(0.05), I2.Inserter(HIT, MISS, True)
    pts = np.float32([[0.4 * math.cos(a), 0.9 * math.sin(a), 0.0]
                      for a in np.linspace(0, 6.0, 200)])
    batch = pp.PointsBatch(pts, origin=(0.1, -0.05, 0.0))
    stage.Process(batch)
    ins.insert(batch.origin, batch.points, ora)
    assert _assert_grid(stage.grid, ora).cells.shape == (100, 100)
    _assert_drawn(stage.grid, ora)
    rng = np.random.RandomState(3)
    cells = rng.randint(0, 32768, (23, 37)).astype(np.uint16)
    cells[rng.rand(23, 37) < 0.3] = 0
    cells[:2] = 0
    cells[:, -3:] = 0
    g = sm.RealTimeGrid2D(synthetic.GridSpec(cells, 0.05, 1.0, 2.0))
    pixels, offset = g.draw()
    ys, xs = np.nonzero(cells)
    want, want_offset = O.draw(cells, (xs.min(), ys.min(), xs.max(), ys.max()))
    assert offset == want_offset == (int(xs.min()), 2)
    np.testing.assert_array_equal(pixels, want)


def test_empty_stream_draws_one_unknown_pixel(sm, pp):
    files, nxt = Files(), Next(pp)
    stage = pp.ProbabilityGridPointsProcessor(0.05, sm.ProbabilityGridRangeDataInserterOptions2D(),
                                              "empty", "png", files, nxt)
    pixels, offset = stage.grid.draw()
    assert pixels.tolist() == [[0xFF808080]] and offset == (0, 0)
    assert stage.Flush() == pp.FlushResult.kFinished and nxt.flushes == 1
    assert pp.decode_png(files.data["empty.png"]).tolist() == [[[128, 128, 128]]]


def test_draw_leaves_the_handle_unchanged_with_at_most_two_syncs(sm, lib, world):
    spec, occ, _, _ = world
    sub, _ = synthetic.crop_grid(spec, occ, 200, 200, 161, 117)
    g = sm.RealTimeGrid2D(sub)                     # made from cells: its box is not known yet
    before = sm.RealTimeGrid2D(sub).read()
    w, h = C.c_int32(), C.c_int32()
    offset = np.zeros(2, np.int32)
    op = offset.ctypes.data_as(C.POINTER(C.c_int32))
    stats = sm.CsmStats()
    ys, xs = np.nonzero(sub.cells)
    want, want_offset = O.draw(sub.cells, (xs.min(), ys.min(), xs.max(), ys.max()))
    px = np.zeros(want.size, np.uint32)
    pp_ = px.ctypes.data_as(C.POINTER(C.c_uint32))
    assert lib.csm_rt_grid2d_draw(g._h, pp_, C.c_int64(px.size), C.byref(w), C.byref(h), op,
                                  C.byref(stats)) == 0
    assert stats.host_syncs == 2 and stats.device_ms >= 0
    assert (h.value, w.value) == want.shape and tuple(offset) == want_offset
    np.testing.assert_array_equal(px.reshape(want.shape), want)
    assert lib.csm_rt_grid2d_draw(g._h, None, C.c_int64(0), C.byref(w), C.byref(h), op,
                                  C.byref(stats)) == 0
    assert stats.host_syncs == 0
    assert lib.csm_rt_grid2d_draw(g._h, pp_, C.c_int64(px.size), C.byref(w), C.byref(h), op,
                                  C.byref(stats)) == 0
    assert stats.host_syncs == 1
    # a capacity one short: the size and offset, no pixel
    px[:] = 7
    assert lib.csm_rt_grid2d_draw(g._h, pp_, C.c_int64(px.size - 1), C.byref(w), C.byref(h), op,
                                  None) == CSM_E_CAPACITY
    assert (px == 7).all() and (h.value, w.value) == want.shape
    after = g.read()
    np.testing.assert_array_equal(after.cells, before.cells)
    assert (after.resolution, after.max_x, after.max_y, after.known_cells_box) == \
        (before.resolution, before.max_x, before.max_y, before.known_cells_box)
    tsdf, _ = synthetic.make_tsdf2d(3, size_cells=64)
    tg = sm.RealTimeGrid2D(tsdf)
    assert lib.csm_rt_grid2d_draw(tg._h, None, C.c_int64(0), C.byref(w), C.byref(h), op,
                                  None) == CSM_E_INVALID
    with pytest.raises(Exception):
        tg.draw()


# ---- 3D ----
def _ordered(ora):
    keep = ora.values != 0
    idx, val, _ = R.walk((ora.indices()[keep], ora.values[keep]))
    return idx, val


def test_hybrid_grid_stage_proto_and_refusal(sm, pp):
    from cartographer_b200._lib import CsmError
    rng = np.random.RandomState(5)
    occ, cell, origin = synthetic.make_building(5, size_m=40.0)
    files, nxt = Files(), Next(pp)
    stage = pp.HybridGridPointsProcessor(0.1, sm.RangeDataInserterOptions3D(**INSERT3D),
                                         "map_3d", files, nxt)
    ora, ins = I3.HybridGrid(0.1), I3.RangeDataInserter3D(**INSERT3D)
    for k in range(8):
        pose = synthetic.random_free_pose_3d(occ, cell, origin, rng)
        cloud = synthetic.cast_lidar_3d(occ, cell, origin, pose, rings=64, azimuths=1024,
                                        max_range=20.0, seed=k)
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T +
               pose[:3]).astype(np.float32)
        batch = pp.PointsBatch(pts, origin=pose[:3].astype(np.float32))
        stage.Process(batch)
        ins.insert(batch.origin, batch.points, None, ora)
    before = stage.grid.to_proto()
    idx, val = _ordered(ora)
    assert len(val) > 10000
    assert before == R.hybrid_grid_message(np.float32(0.1), idx, val)
    with pytest.raises(CsmError):                 # cell 9000 is outside [-8192, 8192)^3
        stage.Process(pp.PointsBatch(np.float32([[900.0, 0.0, 0.0]])))
    assert stage.grid.to_proto() == before and nxt.batches == 8
    assert stage.Flush() == pp.FlushResult.kFinished and nxt.flushes == 1
    assert list(files.data) == ["map_3d"] and files.data["map_3d"] == before


# ---- the stages' Flush chain ----
def test_flush_chain_and_file_names(sm, pp):
    for make, name, text in (
            (lambda f, n: pp.ProbabilityGridPointsProcessor(
                0.05, sm.ProbabilityGridRangeDataInserterOptions2D(), "a", "png", f, n), "a.png",
             "ProbabilityGrid generation"),
            (lambda f, n: pp.ProbabilityGridPointsProcessor(
                0.05, sm.ProbabilityGridRangeDataInserterOptions2D(), "b", "pb", f, n), "b.pb",
             "ProbabilityGrid generation"),
            (lambda f, n: pp.HybridGridPointsProcessor(
                0.1, sm.RangeDataInserterOptions3D(**INSERT3D), "c", f, n), "c",
             "Hybrid grid generation")):
        files, nxt = Files(), Next(pp)
        stage = make(files, nxt)
        assert list(files.data) == [name]          # made at construction, as FromDictionary does
        batch = pp.PointsBatch(np.float32([[1.0, 0.5, 0.2], [-0.7, 0.3, 0.1]]),
                               origin=(0.0, 0.0, 0.1))
        stage.Process(batch)
        assert nxt.batches == 1 and not stage.output
        assert stage.Flush() == pp.FlushResult.kFinished
        assert files.closed == [name] and len(files.data[name]) > 0
        files, nxt = Files(), Next(pp, pp.FlushResult.kRestartStream)
        stage = make(files, nxt)
        with pytest.raises(RuntimeError, match=text + " must be configured to occur after any "
                           "stages that require multiple passes."):
            stage.Flush()
        alone = make(Files(), None)
        alone.Process(batch)
        assert alone.output == [batch] and alone.Flush() == pp.FlushResult.kFinished
