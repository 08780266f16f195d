"""The device XRayPointsProcessor (csm_xray_*) against the CPU restatement (tests/xray_oracle.cc):
the voxels, the column sums (bit for bit) and counts, the shared box and every pixel must be
equal."""
import functools
import math

import numpy as np
import pytest

from benchmarks import synthetic
from tests import xray_oracle as O

pytestmark = pytest.mark.gpu

S = math.sqrt(0.5)
IDENTITY = (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)
# the assets writer's view transforms: pitch -pi/2 (looking down) and yaw -pi/2
XY_VIEW = (0.0, 0.0, 0.0, S, 0.0, -S, 0.0)
XZ_VIEW = (0.0, 0.0, 0.0, S, 0.0, 0.0, -S)


def _tilted():
    q = np.array([0.93, 0.12, -0.21, 0.27])
    q /= np.linalg.norm(q)
    return (1.3, -0.7, 0.45) + tuple(q)


TILTED = _tilted()
TRANSFORMS = {"identity": IDENTITY, "xy": XY_VIEW, "xz": XZ_VIEW, "tilted": TILTED}


@pytest.fixture(scope="module")
def P():
    from cartographer_b200 import points_processing
    return points_processing


@functools.lru_cache(maxsize=None)
def _scans(seed=3, num_scans=10):
    return synthetic.moving_box_scans(seed, num_scans)


def _batches(num, seed=11):
    """`num` seeded (points, colours) batches cycled over the moving-box scans; every fifth
    batch has no colours."""
    rng = np.random.RandomState(seed)
    out = []
    for k in range(num):
        _, p = _scans()[k % len(_scans())]
        c = None if k % 5 == 4 else rng.uniform(0, 1, (len(p), 3)).astype(np.float32)
        out.append((p, c))
    return out


def _assert_same(x, o, aggregations=(0,), draw=True):
    lo, hi, empty = x.bounding_box()
    olo, ohi, oempty = o.bounding_box()
    assert empty == oempty
    if not empty:
        np.testing.assert_array_equal(lo, olo)
        np.testing.assert_array_equal(hi, ohi)
    for a in aggregations:
        np.testing.assert_array_equal(x.voxels(a), o.voxels(a))
        yz, sums, counts = x.columns(a)
        oyz, osums, ocounts = o.columns(a)
        np.testing.assert_array_equal(yz, oyz)
        np.testing.assert_array_equal(sums.view(np.uint32), osums.view(np.uint32))
        np.testing.assert_array_equal(counts, ocounts)
        if not draw:
            continue
        px, st = x.draw(a)
        want = o.draw(a)
        if want is None:
            assert px is None
        else:
            assert st["host_syncs"] == 1
            np.testing.assert_array_equal(px, want)


@pytest.mark.parametrize("voxel_size", [0.01, 0.05, 0.1])
@pytest.mark.parametrize("view", list(TRANSFORMS))
def test_moving_box_inserts(P, view, voxel_size):
    x = P.XRay(voxel_size, TRANSFORMS[view])
    o = O.Processor(voxel_size, transform=TRANSFORMS[view])
    for k, (p, c) in enumerate(_batches(50)):
        st = x.insert([p], [c])
        assert st["host_syncs"] == 1
        assert o.insert(p, c)
        if k % 7 == 0 or k == 49:
            _assert_same(x, o)
    px, _ = x.draw()
    assert (px != 0xFFFFFFFF).sum() > 100 and len({int(v) for v in px.ravel()}) > 20


@pytest.mark.parametrize("factor", [0.5, 1.0, 2.0])
def test_saturation_factors(P, factor):
    x = P.XRay(0.05, TILTED, saturation_factor=factor)
    o = O.Processor(0.05, factor, TILTED)
    for p, c in _batches(10):
        x.insert([p], [c])
        assert o.insert(p, c)
    _assert_same(x, o)


def test_one_column_whose_sum_depends_on_order(P):
    rng = np.random.RandomState(5)
    n = 100000
    pts = np.zeros((n, 3), np.float32)
    pts[:, 0] = rng.randint(0, 300, n) * 0.1
    colors = (rng.uniform(0, 1, (n, 3)) * 10.0 ** rng.randint(-6, 3, (n, 1))).astype(np.float32)
    x = P.XRay(0.1)
    x.insert([pts[:n // 2], pts[n // 2:]], [colors[:n // 2], colors[n // 2:]])
    o = O.Processor(0.1)
    assert o.insert(pts, colors)
    _assert_same(x, o)
    perm = rng.permutation(n)
    shuffled = O.Processor(0.1)
    assert shuffled.insert(pts[perm], colors[perm])
    assert not np.array_equal(shuffled.columns()[1], o.columns()[1])


def test_batches_in_one_call_or_one_at_a_time(P):
    batches = _batches(12)
    one = P.XRay(0.05, XY_VIEW)
    st = one.insert([p for p, _ in batches], [c for _, c in batches])
    assert st["host_syncs"] == 1
    each = P.XRay(0.05, XY_VIEW)
    for p, c in batches:
        each.insert([p], [c])
    o = O.Processor(0.05, transform=XY_VIEW)
    for p, c in batches:
        assert o.insert(p, c)
    _assert_same(one, o)
    _assert_same(each, o)


def test_growth_across_calls(P):
    # 0.01 m cells over many small calls: the tables start at 4096 slots and grow many times
    x = P.XRay(0.01, TILTED)
    o = O.Processor(0.01, transform=TILTED)
    for p, c in _batches(10):
        for i in range(0, len(p), 512):
            cc = None if c is None else c[i:i + 512]
            x.insert([p[i:i + 512]], [cc])
            assert o.insert(p[i:i + 512], cc)
    assert len(o.voxels()) > 4 * 4096 and len(o.columns()[0]) > 4096
    _assert_same(x, o)


def test_cube_faces(P):
    from cartographer_b200._lib import CsmError
    inside = np.float32([[-8192, 0, 0], [8191, 0, 0], [0, -8192, 8191], [0, 8191, -8192],
                         [8191.49, -8192.5 + 0.01, 0]])
    x = P.XRay(1.0)
    o = O.Processor(1.0)
    x.insert([inside])
    assert o.insert(inside)
    for bad in ([8192, 0, 0], [0, -8193, 0], [0, 0, 8191.5], [-8192.5, 0, 0]):
        with pytest.raises(CsmError) as e:
            x.insert([np.float32([[1, 2, 3]]), np.float32([[4, 5, 6], bad])])
        assert e.value.status == 1
        assert not o.insert(np.float32([[1, 2, 3], [4, 5, 6], bad]))
    # a translation that carries a point across a face is refused too
    t = P.XRay(1.0, (0.6, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0))
    with pytest.raises(CsmError):
        t.insert([np.float32([[8191.0, 0, 0]])])
    assert t.bounding_box()[2]
    x.insert([np.float32([[3, 3, 3]])])
    assert o.insert(np.float32([[3, 3, 3]]))
    _assert_same(x, o, draw=False)              # the image would be 16384 x 16384


def test_refused_calls_change_nothing(P):
    from cartographer_b200._lib import CsmError
    x = P.XRay(0.05, XZ_VIEW, num_aggregations=2)
    o = O.Processor(0.05, transform=XZ_VIEW, num_aggregations=2)
    p, c = _batches(1)[0]
    x.insert([p], [c], aggregation=1)
    assert o.insert(p, c, aggregation=1)
    before = (x.bounding_box(), x.voxels(1), x.columns(1), x.draw(1)[0])
    nan_colour = c.copy()
    nan_colour[7, 1] = np.nan
    inf_point = p.copy()
    inf_point[3, 2] = np.inf
    far = p.copy()
    far[100] = [1e3, 0, 0]                           # 20000 cells at 0.05 m
    for args, kw in (([[p, p], [c, nan_colour]], {}), ([[inf_point]], {}),
                     ([[p, far]], {}), ([[p]], {"aggregation": 2}),
                     ([[p]], {"aggregation": -1})):
        with pytest.raises(CsmError) as e:
            x.insert(*args, **kw)
        assert e.value.status == 1
    after = (x.bounding_box(), x.voxels(1), x.columns(1), x.draw(1)[0])
    for a, b in zip(before[0], after[0]):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(before[1], after[1])
    for a, b in zip(before[2], after[2]):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(before[3], after[3])
    assert len(x.voxels(0)) == 0
    _assert_same(x, o, (0, 1))


def test_empty_calls_and_box(P):
    x = P.XRay(0.1)
    assert x.insert([])["host_syncs"] == 0
    assert x.insert([np.zeros((0, 3), np.float32)])["host_syncs"] == 0
    assert x.bounding_box()[2]
    px, st = x.draw()
    assert px is None and st["host_syncs"] == 0


def test_floors(P, tmp_path):
    scans = _scans()[:6]
    rng = np.random.RandomState(2)
    colors = [rng.uniform(0, 1, (len(p), 3)).astype(np.float32) for _, p in scans]
    # floor 0 spans times 0..2, floor 1 times 2..4 (batch 2 is in both), floor 2 no batch
    floors = [[(0, 2)], [(2, 3), (4, 4)], [(100, 200)]]
    files = {}

    class Writer:
        def __init__(self, name):
            self.name, self.data = name, b""

        def write(self, b):
            self.data += b

        def close(self):
            files[self.name] = self.data

    stage = P.XRayPointsProcessor(0.05, XY_VIEW, str(tmp_path / "xray"), floors=floors,
                                  file_writer_factory=Writer)
    assert stage.kConfigurationFileActionName == "write_xray_image"
    for t, ((_, p), c) in enumerate(zip(scans, colors)):
        stage.Process(P.PointsBatch(p, colors=c, start_time=t))
    assert stage.Flush() == P.FlushResult.kFinished
    assert len(stage.output) == 6
    o = O.Processor(0.05, transform=XY_VIEW, num_aggregations=3)
    for t, ((_, p), c) in enumerate(zip(scans, colors)):
        for i, spans in enumerate(floors):
            if any(a <= t <= b for a, b in spans):
                assert o.insert(p, c, aggregation=i)
    assert sorted(files) == [str(tmp_path / ("xray%d.png" % i)) for i in range(3)]
    for i in range(3):
        want = o.draw(i)
        got = P.decode_png(files[str(tmp_path / ("xray%d.png" % i))])
        np.testing.assert_array_equal(got, P.cairo_to_rgb(want))
    assert (o.draw(2) == 0xFFFFFFFF).all() and o.draw(2).shape == o.draw(0).shape
    _assert_same(stage.xray, o, (0, 1, 2))


def test_processor_writes_one_png_and_flushes_next(P, tmp_path):
    class Next:
        def __init__(self, result):
            self.result, self.batches = result, []

        def Process(self, b):
            self.batches.append(b)

        def Flush(self):
            return self.result

    nxt = Next(P.FlushResult.kFinished)
    stage = P.XRayPointsProcessor(0.1, IDENTITY, str(tmp_path / "single"), next=nxt)
    p, c = _batches(1)[0]
    stage.Process(P.PointsBatch(p, colors=c))
    assert stage.Flush() == P.FlushResult.kFinished and len(nxt.batches) == 1
    o = O.Processor(0.1)
    assert o.insert(p, c)
    with open(tmp_path / "single.png", "rb") as f:
        np.testing.assert_array_equal(P.decode_png(f.read()), P.cairo_to_rgb(o.draw()))
    again = P.XRayPointsProcessor(0.1, IDENTITY, str(tmp_path / "again"),
                                  next=Next(P.FlushResult.kRestartStream))
    again.Process(P.PointsBatch(p))
    with pytest.raises(RuntimeError, match="X-Ray generation must be configured"):
        again.Flush()
    empty = P.XRayPointsProcessor(0.1, IDENTITY, str(tmp_path / "empty"))
    with pytest.warns(UserWarning):
        empty.Flush()
    assert not (tmp_path / "empty.png").exists()


def test_two_handles_side_by_side(P):
    a, b = P.XRay(0.05, XY_VIEW), P.XRay(0.1, TILTED, saturation_factor=2.0)
    oa, ob = O.Processor(0.05, transform=XY_VIEW), O.Processor(0.1, 2.0, TILTED)
    for p, c in _batches(8):
        b.insert([p], [c])
        a.insert([p], [c])
        assert oa.insert(p, c) and ob.insert(p, c)
    _assert_same(a, oa)
    _assert_same(b, ob)


def test_config5_size(P):
    """200 batches of 65,536 points (64 rings x 1024 azimuths), in calls of 20 batches."""
    base = synthetic.moving_box_scans(5, 4, rings=64, azimuths=1024, max_range=8.0)
    rng = np.random.RandomState(9)
    x = P.XRay(0.05, XY_VIEW)
    o = O.Processor(0.05, transform=XY_VIEW)
    batches = []
    for k in range(200):
        p = np.resize(base[k % len(base)][1], (65536, 3))
        batches.append((p, rng.uniform(0, 1, (65536, 3)).astype(np.float32)))
    for i in range(0, 200, 20):
        g = batches[i:i + 20]
        st = x.insert([p for p, _ in g], [c for _, c in g])
        assert st["host_syncs"] == 1
    for p, c in batches:
        assert o.insert(p, c)
    _assert_same(x, o)
