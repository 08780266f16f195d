"""The 3D map-writing kernels (csrc/insert3d.cu, csrc/grid3d.cu) at the edges where they go
wrong, against the existing references after every call:
  * tests/insert3d_oracle.py for occupancy values, intensity sums, counts and means, bit for bit;
  * the single-grid call (csm_range_inserter3d_insert) on the host-transformed scan, for the
    boxes the one-call submap insert (csm_range_inserter3d_insert_submaps) grows;
  * tests/hybrid_grid_walk.cc for the voxel order, tests/grid_proto_ref.py for the proto,
    tests/submap_texture_oracle.py for the texture and the list-built matcher for the from-grid
    matcher's levels;
  * numpy for the non-zero box, which the walk's voxels must span exactly, and
    tests/map_writing3d_refs.py (float64) for the range filter's and GetCellIndex's decisions.
Launch shapes (partial warps, single lanes, whole warps dropped), ties at max_range and at half
cells, contention on one cell and the update marker, miss samples of every sign, intensity runs
at the sort's key-width edges and non-finite intensities, the 2^14 cube's faces and growth slack
clamped there, and the non-zero box and voxel walk at block, tile and cube edges."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from benchmarks import synthetic
from tests import grid_proto_ref as R
from tests import insert3d_oracle as O
from tests import map_writing3d_refs as M
from tests import submap_texture_oracle as T
from tests import worlds3d
from tests.test_gpu_active_submaps3d import RefSubmap, assert_same, host_transform
from tests.test_gpu_insert3d import assert_grid_equal

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LUA = dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
           intensity_threshold=40.0)   # trajectory_builder_3d.lua submaps.range_data_inserter
IDENT = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
NAN_BITS = np.uint32(0x7fc00000)


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("map_writing3d") / "libsubmap_insert3d_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                           os.path.join(ROOT, "tests", "submap_insert3d_oracle.cc"), "-o", so])
    return C.CDLL(so)


def _pair(sm, **opts):
    o = dict(LUA, **opts)
    return sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**o)), O.RangeDataInserter3D(**o)


def _triple(sm, **opts):
    """(device, CPU) inserters, and a second device inserter with the same options for the
    single-grid calls of the reference submaps."""
    o = dict(LUA, **opts)
    return _pair(sm, **opts), sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**o))


def _fbits(a):
    """float32 bit patterns with every NaN mapped to one pattern: the device's float adds give
    the canonical NaN, the host's keep an operand's payload; both are NaN."""
    a = np.asarray(a, np.float32)
    return np.where(np.isnan(a), NAN_BITS, a.view(np.uint32))


def assert_igrid_equal(dev, ora):
    """Counts, and sums and means bit for bit (NaNs as one pattern)."""
    lo, mean, sums, counts = dev.read()
    dims = mean.shape[::-1]
    idx = O.unpack(ora.keys[ora.counts != 0]) - lo
    assert np.all((idx >= 0) & (idx < np.asarray(dims))), "a voxel outside the box"
    np.testing.assert_array_equal(counts, ora.dense(lo, dims, 1))
    np.testing.assert_array_equal(_fbits(sums), _fbits(ora.dense(lo, dims, 0)))
    np.testing.assert_array_equal(_fbits(mean), _fbits(ora.dense_mean(lo, dims)))
    return lo, dims


def _snapshot(handles):
    return [x.copy() for h in handles for x in h.read()]


def _assert_unchanged(before, handles):
    for a, b in zip(before, _snapshot(handles)):
        np.testing.assert_array_equal(a, b)


def _values(dev, cells):
    """The handle's values at the cells (n x 3), 0 outside its box."""
    lo, vol = dev.read()
    c = np.asarray(cells, np.int64).reshape(-1, 3) - lo
    inside = np.all((c >= 0) & (c < np.asarray(vol.shape[::-1])), 1)
    out = np.zeros(len(c), vol.dtype)
    out[inside] = vol[c[inside, 2], c[inside, 1], c[inside, 0]]
    return out


def _box(dev):
    lo, vol = dev.read()[:2]
    return tuple(int(v) for v in lo), tuple(int(v) for v in vol.shape[::-1])


class Submaps:
    """One call of csm_range_inserter3d_insert_submaps over fresh handles, and the same scan
    through the single-grid call on the host-transformed data and through the CPU inserter
    (RefSubmap); every handle compared after every call."""

    def __init__(self, sm, poses, intensity, hi_res=0.1, lo_res=0.45):
        self.refs = [RefSubmap(sm, p, hi_res, lo_res, intensity=i)
                     for p, i in zip(poses, intensity)]
        self.grids = [(sm.DeviceHybridGrid.empty(hi_res), sm.DeviceHybridGrid.empty(lo_res),
                       sm.DeviceIntensityGrid.empty(hi_res) if i else None)
                      for i in intensity]

    def call(self, host, ins, single, origin, pts, inten, max_range):
        dev, ora = ins
        dev.insert_submaps([(r.pose, *g) for r, g in zip(self.refs, self.grids)], origin, pts,
                           inten, max_range)
        for r in self.refs:
            r.insert(host, (single, ora), origin, pts, inten, max_range)
        for g, r in zip(self.grids, self.refs):
            assert_same(g[0], r.hi, False)
            assert_same(g[1], r.lo, False)
            if r.ig is not None:
                a, b = g[2].read(), r.ig[0].read()
                for x, y in zip(a, b):
                    np.testing.assert_array_equal(x.view(np.uint32) if x.dtype == np.float32
                                                  else x,
                                                  y.view(np.uint32) if y.dtype == np.float32
                                                  else y)
                assert_igrid_equal(g[2], r.ig[1])


# ---- 1. launch shapes: partial warps, single lanes, dropped warps, one side of the origin ----
SUBMAP_POSES = [IDENT, [1.5, -0.5, 0.25, math.cos(0.2), 0.0, 0.0, math.sin(0.2)],
                [-2.0, 3.0, -0.75, *(np.array([0.99, 0.05, -0.03, 0.1]) /
                                     np.linalg.norm([0.99, 0.05, -0.03, 0.1]))]]


def _shaped_scan(rng, n, keep, side, origin, max_range):
    """n returns around side * (40, 30, 20), about 40 m from the origin: the kept ones as they
    are, the others pushed beyond max_range + 5 along their ray, all on the same side of 0."""
    centre = side * np.array([40.0, 30.0, 20.0])
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = centre + d * rng.uniform(0.2, 3.0, (n, 1))
    ray = p - origin
    dist = np.linalg.norm(ray, axis=1, keepdims=True)
    far = origin + ray / dist * rng.uniform(max_range + 5, max_range + 9, (n, 1))
    p = np.where(keep[:, None], p, far).astype(np.float32)
    assert (np.sign(p) == side).all()
    return p


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 4097, 65537])
def test_launch_shapes(sm, host, n):
    rng = np.random.RandomState(n)
    ins, single = _triple(sm)
    # (entries, the one without intensity): 1 entry with and without, 2 and 3 entries with it
    # off in the first, middle or last
    layouts = [(1, 0), (2, 0), (3, 1), (1, None), (2, 1), (3, 2)]
    for k, pattern in enumerate(M.KEEP_PATTERNS):
        side = 1 if k % 2 == 0 else -1
        num, off = layouts[k]
        origin = (side * np.array([10.0, 8.0, 5.0])).astype(np.float32)
        max_range = 50.0
        keep = M.lane_keep(pattern, n)
        pts = _shaped_scan(rng, n, keep, side, origin.astype(np.float64), max_range)
        # the float64 range sides: every return is decided and as the pattern says
        for pose in SUBMAP_POSES[:num]:
            np.testing.assert_array_equal(M.range_sides64(pose, origin, pts, max_range),
                                          np.where(keep, 1, -1))
        inten = rng.uniform(0, 60, n).astype(np.float32)
        s = Submaps(sm, SUBMAP_POSES[:num], [i != off for i in range(num)])
        s.call(host, ins, single, origin, pts, inten, max_range)
        # with no return kept the high-resolution handles keep the fresh box
        if not keep.any():
            for g in s.grids:
                assert _box(g[0]) == ((0, 0, 0), (1, 1, 1))


# ---- 2. the range filter and half-cell ties ----
def test_range_filter_ulps(sm, host):
    """Returns on the axes at max_range and one float32 ulp either side: sqrt(d * d) == |d|
    exactly, so the filter keeps exactly the ones not beyond."""
    max_range = np.float32(5.0)
    ins, single = _triple(sm, num_free_space_voxels=0)
    for v, kept in zip(M.ulp_neighbours(max_range), (True, True, False)):
        pts = []
        for a in range(3):
            for sgn in (-1, 1):
                p = np.zeros(3, np.float32)
                p[a] = sgn * v
                pts.append(p)
        pts = np.asarray(pts, np.float32)
        s = Submaps(sm, [IDENT], [True])
        s.call(host, ins, single, np.zeros(3, np.float32), pts, np.full(6, 5.0, np.float32),
               float(max_range))
        hit = _values(s.grids[0][0], O.cell_index(0.1, pts)) != 0
        assert hit.tolist() == [kept] * 6


# identity rotation: the submap transform is one float32 add of the inverse translation, so
# returns can be placed exactly on half cells of the submap frame
TIE_POSES = {"identity": IDENT, "translated": [2.0, -3.0, 1.5, 1.0, 0.0, 0.0, 0.0]}


def _single_cell(sm, ins, pose, res, point):
    """The one cell a lone return hits in a fresh submap's high-resolution handle (no misses)."""
    hi, lo = sm.DeviceHybridGrid.empty(res), sm.DeviceHybridGrid.empty(res)
    ins.insert_submaps([(pose, hi, lo, None)], np.zeros(3, np.float32), point[None], None, 1e9)
    box_lo, vol = hi.read()
    z, y, x = np.nonzero(vol)
    assert len(x) == 1
    cell = np.array([x[0], y[0], z[0]]) + box_lo
    hi.close()
    lo.close()
    return cell


@pytest.mark.parametrize("pose_name", sorted(TIE_POSES))
@pytest.mark.parametrize("res", [0.5, 0.1])
def test_half_cell_ties(sm, host, res, pose_name):
    """Returns whose submap-frame quotient is a half-integer, and one ulp either side, at both
    signs on each axis.  Each return is inserted on its own, so the one cell it hits is the cell
    the device's GetCellIndex gives it: that equals the host's cell always, and the float64 cell
    wherever the quotient's rounding cannot move it (every return at resolution 0.5)."""
    pose = TIE_POSES[pose_name]
    t = np.float32(pose[:3])
    q = np.array([0.5, 1.5, 2.5, 7.5, 63.5, 64.5, 100.5])
    base = (q * float(np.float32(res))).astype(np.float32)
    vals = np.concatenate([np.concatenate(M.ulp_neighbours(b)) for b in (base, -base)])
    # the submap-frame values, one axis at a time, the others at 0
    sub = np.zeros((3 * len(vals), 3), np.float32)
    for a in range(3):
        sub[a * len(vals):(a + 1) * len(vals), a] = vals
    # the local-frame returns whose transform (p - t in float32) gives these values back exactly
    pts = (sub + t).astype(np.float32)
    exact = np.all((pts - t).astype(np.float32) == sub, axis=1)
    sub, pts = sub[exact], pts[exact]
    assert len(pts) >= 3 * len(vals) // 2
    _, p32, kept = host_transform(host, pose, np.zeros(3, np.float32), pts, 1e9)
    np.testing.assert_array_equal(p32, sub)
    assert kept.all()
    cells, decided = M.cell_sides64(sub, res)
    host_cells = O.cell_index(res, p32)
    np.testing.assert_array_equal(cells[decided], host_cells[decided])
    assert decided.sum() >= len(pts) // 4 and (res != 0.5 or decided.all())
    ins, single = _triple(sm, num_free_space_voxels=0)
    for j in range(len(pts)):
        got = _single_cell(sm, ins[0], pose, res, pts[j])
        np.testing.assert_array_equal(got, host_cells[j], err_msg=str(sub[j]))
        if decided[j]:
            np.testing.assert_array_equal(got, cells[j], err_msg=str(sub[j]))
    # all of them in one call, against the single-grid call and the CPU inserter
    s = Submaps(sm, [pose], [False], hi_res=res, lo_res=res)
    s.call(host, ins, single, np.zeros(3, np.float32), pts, None, 1e9)


def test_rotated_range_and_cells_float64(sm, host):
    """Under a tilted submap pose, returns near max_range and near half cells: the host
    transform the device agrees with (rigid3f.h) decides as float64 does wherever float64 is
    decided, and the one-call insert equals the single-grid one."""
    rng = np.random.RandomState(9)
    pose = SUBMAP_POSES[2]
    max_range = 6.0
    origin = np.float32([0.3, -0.2, 0.1])
    d = rng.normal(size=(3000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = max_range * (1 + rng.choice([-1e-2, -1e-6, 0.0, 1e-6, 1e-2], 3000))
    s_frame_origin, _ = M.submap_frame64(pose, origin)
    # points placed in the submap frame, mapped back to the local frame
    sub = s_frame_origin + d * r[:, None]
    pts = (sub @ M.rotation64(pose[3:]).T + np.asarray(pose[:3])).astype(np.float32)
    side = M.range_sides64(pose, origin, pts, max_range)
    o32, p32, kept = host_transform(host, pose, origin, pts, max_range)
    assert (side != 0).sum() > 1000 and (side == 0).any()
    np.testing.assert_array_equal(kept[side != 0], side[side != 0] == 1)
    p64, scale = M.submap_frame64(pose, pts)
    cells, decided = M.cell_sides64(p64, 0.1, scale)
    np.testing.assert_array_equal(cells[decided], O.cell_index(0.1, p32)[decided])
    ins, single = _triple(sm)
    s = Submaps(sm, [pose, IDENT], [True, False])
    s.call(host, ins, single, origin, pts, rng.uniform(0, 60, len(pts)).astype(np.float32),
           max_range)


# ---- 3. contention and the update marker ----
def test_one_cell_2e17_returns(sm, host):
    """2^17 returns in one voxel: one hit, one touched-list entry, and an intensity run whose
    float32 sum depends on the order of the adds."""
    rng = np.random.RandomState(17)
    n = 1 << 17
    pts = (np.float32([2.03, -1.02, 0.51]) + rng.uniform(-0.004, 0.004, (n, 3))).astype(np.float32)
    inten = (rng.uniform(0, 40, n) * rng.choice([1e-3, 1.0, 1e3], n) / 1e3).astype(np.float32)
    inten = np.minimum(inten, np.float32(40.0))
    # the order matters to this run's float32 sum (cumsum adds one at a time)
    a = np.cumsum(inten, dtype=np.float32)[-1]
    b = np.cumsum(inten[rng.permutation(n)], dtype=np.float32)[-1]
    assert a != b
    ins, single = _triple(sm, num_free_space_voxels=5)
    g = (sm.DeviceHybridGrid.empty(0.1), O.HybridGrid(0.1))
    ig = (sm.DeviceIntensityGrid.empty(0.1), O.IntensityHybridGrid(0.1))
    origin = np.float32([0.0, 0.0, 0.0])
    for _ in range(2):
        ins[0].Insert(origin, pts, inten, g[0], ig[0])
        ins[1].insert(origin, pts, inten, g[1], ig[1])
        assert_grid_equal(*g)
        assert_igrid_equal(*ig)
    assert len(np.unique(O.cell_index(0.1, pts), axis=0)) == 1
    s = Submaps(sm, [IDENT, SUBMAP_POSES[1]], [True, True])
    s.call(host, ins, single, origin, pts, inten, 20.0)


@pytest.mark.parametrize("hit_first", [True, False])
def test_rays_cross_a_hit_cell(sm, hit_first):
    """Rays whose miss samples all cross cell (3, 0, 0), which another return hits: the hit
    table wins in either index order; the next insert misses it, the marker cleared once."""
    ins = _pair(sm, num_free_space_voxels=1000)
    g = (sm.DeviceHybridGrid.empty(1.0), O.HybridGrid(1.0))
    rays = np.array([[9, a, b] for a in range(-2, 3) for b in range(-2, 3)], np.float32)
    rays = np.repeat(rays, 100, axis=0)
    hit = np.float32([[3, 0, 0]])
    for k in range(3):
        if k == 0:
            pts = np.concatenate([hit, rays] if hit_first else [rays, hit])
        else:   # hit in the first insert, only missed in the next ones
            pts = rays
        ins[0].Insert([0, 0, 0], pts, None, g[0])
        ins[1].insert([0, 0, 0], pts, None, g[1])
        assert_grid_equal(*g)
        lo, vol = g[0].read()
        v = int(vol[-lo[2], -lo[1], 3 - lo[0]])
        assert v < 32768   # no marker left behind
        if k == 0:
            assert v == int(ins[1].hit_table[0]) - 32768


def test_touched_list_fills_its_capacity(sm):
    """Every cell of a 3 x 3 x 3 handle touched (touched == Volume() == list_cap), and n
    distinct hits without misses (touched == n == list_cap)."""
    idx = np.array([[-1, -1, -1], [1, 1, 1]], np.int32)
    val = np.uint16([0, 0])
    for nfsv in (1, 0):
        ins = _pair(sm, num_free_space_voxels=nfsv)
        g = (sm.DeviceHybridGrid(synthetic.HybridGridSpec(1.0, idx, val)),
             O.HybridGrid(1.0, idx, val))
        cells = np.array([[x, y, z] for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)],
                         np.float32)
        for k in range(3):
            pts = cells[np.random.RandomState(k).permutation(27)]
            ins[0].Insert([0, 0, 0], pts, None, g[0])
            ins[1].insert([0, 0, 0], pts, None, g[1])
            assert _box(g[0]) == ((-1, -1, -1), (3, 3, 3))   # no growth: Volume() is 27
            assert_grid_equal(*g)
            assert (g[0].read()[1] != 0).all()


class _ChunkedInserter(O.RangeDataInserter3D):
    """The CPU inserter with the miss samples built in chunks of returns (the same samples in
    the same order, within a test's memory)."""

    def miss_cells(self, origin_cell, hit_cells):
        parts = [super(_ChunkedInserter, self).miss_cells(origin_cell, hit_cells[i:i + 4096])
                 for i in range(0, len(hit_cells), 4096)]
        return np.concatenate(parts) if parts else np.zeros((0, 3), np.int64)


@pytest.mark.parametrize("nfsv", [0, 1, 40, 1000])
def test_free_space_voxels(sm, nfsv):
    """num_free_space_voxels 0, 1, above the largest num_samples (40 > 37), and 1000 with
    65 536 returns: 65.5 M miss threads, more than one launch's grid, so the stride loop wraps."""
    rng = np.random.RandomState(nfsv)
    n = 65536 if nfsv == 1000 else 5000
    d = rng.normal(size=(n, 3))
    d /= np.abs(d).max(1, keepdims=True)
    r = rng.uniform(1, 37, (n, 1)) if nfsv != 1000 else rng.uniform(1, 6, (n, 1))
    pts = (d * r).astype(np.float32)
    if nfsv == 1000:   # the longest rays, along +x: 1200 samples
        pts[::997, 0] = np.float32(1200.0)
    opts = dict(LUA, num_free_space_voxels=nfsv)
    dev = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**opts))
    ora = _ChunkedInserter(**opts)
    g = (sm.DeviceHybridGrid.empty(1.0), O.HybridGrid(1.0))
    for origin in ([0.2, -0.3, 0.4], [-3.0, 2.0, 1.0]):
        dev.Insert(origin, pts, None, g[0])
        ora.insert(origin, pts, None, g[1])
        assert_grid_equal(*g)


# ---- 4. miss samples: every sign, not divisible, 0 / 1 / 2 / 16 000+ samples per axis ----
def _deltas():
    out = []
    for sx in (-1, 1):
        for sy in (-1, 1):
            for sz in (-1, 1):
                out.append([sx * 7, sy * 5, sz * 3])       # 7 samples, 5 / 7 and 3 / 7 steps
                out.append([sx * 2, sy * 1, sz * 1])
                out.append([sx * 1, sy * 1, 0])
    for a in range(3):
        for s in (-1, 1):
            for ns in (0, 1, 2):
                v = [0, 0, 0]
                v[a] = s * ns
                out.append(v)
    return np.array(out)


@pytest.mark.parametrize("nfsv", [3, 20000])
def test_miss_samples(sm, nfsv):
    ins = _pair(sm, num_free_space_voxels=nfsv)
    g = (sm.DeviceHybridGrid.empty(1.0), O.HybridGrid(1.0))
    origin = np.array([4, -6, 9])
    ins[0].Insert(origin.astype(np.float32), (origin + _deltas()).astype(np.float32), None, g[0])
    ins[1].insert(origin.astype(np.float32), (origin + _deltas()).astype(np.float32), None, g[1])
    assert_grid_equal(*g)
    # 16 001 samples along each axis, both signs, with non-divisible steps on the other axes
    for a in range(3):
        for s in (-1, 1):
            o = np.array([0, 0, 0])
            o[a] = -s * 8000
            dlt = np.array([7, -13, 5])
            dlt[a] = s * 16001
            h = sm.DeviceHybridGrid.empty(1.0), O.HybridGrid(1.0)
            flip = np.where(np.arange(3) == a, 1, -1)
            pts = (o + np.array([dlt, dlt * flip])).astype(np.float32)
            ins[0].Insert(o.astype(np.float32), pts, None, h[0])
            ins[1].insert(o.astype(np.float32), pts, None, h[1])
            assert_grid_equal(*h)
            h[0].close()


# ---- 5. intensities: key widths, long runs, first and last keys, non-finite values ----
# box shapes of volume 1, 2, 2^k and 2^k +- 1 (every extent inside the 2^14 cube)
INTENSITY_BOXES = {1: (1, 1, 1), 2: (2, 1, 1), 3: (3, 1, 1), 15: (15, 1, 1), 16: (4, 2, 2),
                   17: (17, 1, 1), 1023: (1023, 1, 1), 1024: (16, 8, 8), 1025: (25, 41, 1),
                   65535: (255, 257, 1), 65536: (64, 64, 16), (1 << 18) + 1: (65, 37, 109),
                   1 << 24: (256, 256, 256), (1 << 24) + 1: (97, 257, 673)}


@pytest.mark.parametrize("volume", sorted(INTENSITY_BOXES))
def test_intensity_box_volumes(sm, volume):
    """A handle made from a voxel list whose box holds `volume` voxels (the sort's key width is
    that of volume - 1), with runs at the first and the last key interleaved."""
    rng = np.random.RandomState(volume % 1000)
    shape = INTENSITY_BOXES[volume]
    assert int(np.prod(shape)) == volume
    lo = np.array([-3, 5, -2])
    hi = lo + np.array(shape) - 1
    idx = np.array([lo, hi][:1 if volume == 1 else 2], np.int32)
    sums, counts = np.float32([1.5, 2.25])[:len(idx)], np.int32([1, 3])[:len(idx)]
    dev = sm.DeviceIntensityGrid(sm.IntensityGridSpec(1.0, idx, sums, counts))
    ora = O.IntensityHybridGrid(1.0, idx, sums, counts)
    ins = _pair(sm)
    g = (sm.DeviceHybridGrid.empty(1.0), O.HybridGrid(1.0))
    m = 600
    cells = np.where((np.arange(m) % 2 == 0)[:, None], lo, hi).astype(np.float64)
    inside = lo + np.floor(rng.uniform(0, 1, (m, 3)) * np.array(shape)).astype(np.int64)
    cells[::3] = inside[::3]
    pts = cells.astype(np.float32)
    inten = rng.uniform(0, 40, m).astype(np.float32)
    for k in range(2):
        ins[0].Insert([lo[0], lo[1], lo[2]], pts, inten, g[0], dev)
        ins[1].insert(np.float32(lo), pts, inten, g[1], ora)
        got_lo, dims = assert_igrid_equal(dev, ora)
        assert tuple(got_lo) == tuple(lo) and tuple(dims) == tuple(shape)   # no growth
        assert int(np.prod(dims)) == volume


def test_intensity_values_at_the_edges(sm, host):
    """NaN, +-inf, -0.0, exactly the threshold and one ulp above it, into a handle made from a
    voxel list (its first insert), through both entry points."""
    thr = np.float32(40.0)
    above = M.ulp_neighbours(thr)[2]
    cases = [  # (cell, intensities added there in return order)
        ([0, 0, 0], [np.nan, 1.0, 2.0]),
        ([1, 0, 0], [np.inf, 3.0]),         # +inf is above the threshold: not added
        ([2, 0, 0], [-np.inf, np.inf]),     # NaN is not above it: added
        ([3, 0, 0], [-np.inf, -1.0]),
        ([4, 0, 0], [-0.0, -0.0]),
        ([5, 0, 0], [thr, thr]),
        ([6, 0, 0], [above, 1.0]),
        ([7, 0, 0], [above]),
        ([8, 0, 0], [1.0, np.nan]),
    ]
    pts, inten = [], []
    for cell, vals in cases:
        for v in vals:
            pts.append(cell)
            inten.append(v)
    pts = np.asarray(pts, np.float32)
    inten = np.asarray(inten, np.float32)
    order = np.random.RandomState(1).permutation(len(pts))   # interleave the voxels' returns
    pts, inten = pts[order], inten[order]
    idx = np.array([[4, 0, 0], [0, 0, 0], [9, 1, 1]], np.int32)
    sums, counts = np.float32([-0.0, 0.5, 0.0]), np.int32([1, 1, 0])
    ins, single = _triple(sm, num_free_space_voxels=1)
    dev = sm.DeviceIntensityGrid(sm.IntensityGridSpec(1.0, idx, sums, counts))
    ora = O.IntensityHybridGrid(1.0, idx, sums, counts)
    g = (sm.DeviceHybridGrid.empty(1.0), O.HybridGrid(1.0))
    for _ in range(2):
        ins[0].Insert([0, 0, 0], pts, inten, g[0], dev)
        ins[1].insert(np.float32([0, 0, 0]), pts, inten, g[1], ora)
        assert_igrid_equal(dev, ora)
    lo, mean, s, c = dev.read()
    at = lambda a, x: a[-lo[2], -lo[1], x - lo[0]]  # noqa: E731
    assert np.signbit(at(s, 4)) and at(c, 4) == 5 and np.signbit(at(mean, 4))
    assert at(c, 5) == 4 and at(c, 7) == 0 and at(c, 6) == 2
    assert np.isnan(at(s, 0)) and np.isnan(at(s, 8)) and at(c, 0) == 7 and at(c, 8) == 4
    assert at(s, 1) == 6.0 and at(c, 1) == 2 and at(s, 2) == -np.inf and at(s, 3) == -np.inf
    # the same scan through the one-call insert, into a handle made from the same list
    s = Submaps(sm, [IDENT], [True], hi_res=1.0, lo_res=1.0)
    s.grids[0] = (s.grids[0][0], s.grids[0][1],
                  sm.DeviceIntensityGrid(sm.IntensityGridSpec(1.0, idx, sums, counts)))
    s.refs[0].ig = (sm.DeviceIntensityGrid(sm.IntensityGridSpec(1.0, idx, sums, counts)),
                    O.IntensityHybridGrid(1.0, idx, sums, counts))
    for _ in range(2):
        s.call(host, ins, single, np.float32([0, 0, 0]), pts, inten, 1e9)


# ---- 6. the 2^14 cube's faces ----
def _face_values():
    """(value, accepted) along one axis at resolution 1: q = p."""
    up = M.ulp_neighbours(np.float32(8191.5))
    dn = M.ulp_neighbours(np.float32(-8192.5))
    return [(up[0], True), (up[1], False), (up[2], False),
            (dn[2], True), (dn[1], False), (dn[0], False)]


@pytest.mark.parametrize("what", ["return", "origin"])
def test_cube_faces(sm, host, what):
    """A return or the origin with q at +-(8192 - 0.5) and one ulp either side, on each axis,
    through both entry points: accepted ones land in the face cell, refused ones change no
    handle.  Other returns keep the face return's other axes inside the box."""
    from cartographer_b200._lib import CsmError
    ins, single = _triple(sm, num_free_space_voxels=3)
    for a in range(3):
        for v, ok in _face_values():
            inside = np.float32(8180.0 if v > 0 else -8180.0)
            base = np.zeros(3, np.float32)
            base[a] = inside
            face = base.copy()
            face[a] = v
            others = np.array([base + np.float32(3) * (np.arange(3) != a),
                               base - np.float32(3) * (np.arange(3) != a)], np.float32)
            if what == "return":
                origin, pts = base, np.concatenate([others, face[None]])
            else:
                origin, pts = face, others
            g = (sm.DeviceHybridGrid.empty(1.0), O.HybridGrid(1.0))
            ig = (sm.DeviceIntensityGrid.empty(1.0), O.IntensityHybridGrid(1.0))
            inten = np.full(len(pts), 5.0, np.float32)
            s = Submaps(sm, [IDENT], [True], hi_res=1.0, lo_res=2.0)

            def single_grid(o, p, i):
                ins[0].Insert(o, p, i, g[0], ig[0])
                ins[1].insert(o, p, i, g[1], ig[1])
                assert_grid_equal(*g)
                assert_igrid_equal(*ig)

            # a first insert that succeeds, so that a refusal has contents to keep
            single_grid(base, others, inten[:2])
            s.call(host, ins, single, base, others, inten[:2], 1e9)
            handles = [g[0], ig[0], *s.grids[0]]
            before = _snapshot(handles)
            if ok:
                single_grid(origin, pts, inten)
                c = O.cell_index(1.0, face)[0]
                assert c[a] == (8191 if v > 0 else -8192)
                s.call(host, ins, single, origin, pts, inten, 1e9)
                continue
            with pytest.raises(CsmError) as e:
                ins[0].Insert(origin, pts, inten, g[0], ig[0])
            assert e.value.status == 1
            with pytest.raises(CsmError) as e:
                ins[0].insert_submaps([(IDENT, *s.grids[0])], origin, pts, inten, 1e9)
            assert e.value.status == 1
            _assert_unchanged(before, handles)


def test_growth_clamped_on_all_six_faces(sm, host):
    """One call grows two submaps' handles, one against the three low faces and one against the
    three high faces of the cube: the slack is clamped there, and the boxes equal the
    single-grid call's and the slack box of the tight box."""
    rng = np.random.RandomState(6)
    pts = rng.randint(-7, 8, (500, 3)).astype(np.float32)
    pts[:2] = [[-7, -7, -7], [7, 7, 7]]
    poses = [[8185.0, 8185.0, 8185.0, 1.0, 0.0, 0.0, 0.0],
             [-8184.0, -8184.0, -8184.0, 1.0, 0.0, 0.0, 0.0]]
    ins, single = _triple(sm)
    s = Submaps(sm, poses, [True, True], hi_res=1.0, lo_res=1.0)
    origin = np.float32([0.0, 0.0, 0.0])
    s.call(host, ins, single, origin, pts, rng.uniform(0, 60, 500).astype(np.float32), 1e9)
    for (hi, lo, ig), pose in zip(s.grids, poses):
        cells = np.concatenate([pts, origin[None]]) - np.float32(pose[:3])
        tlo, thi = cells.min(0).astype(np.int64), cells.max(0).astype(np.int64)
        for h in (hi, lo):
            blo, dims = M.slack_box(tlo, thi)
            got = _box(h)
            assert got == (tuple(blo), tuple(dims))
            assert (blo >= -8192).all() and (blo + dims <= 8192).all()
            assert (blo == -8192).all() or (blo + dims == 8192).all()   # clamped on three faces


# ---- 7. the non-zero box and the voxel walk ----
def _handle(sm, idx, val, res=0.1):
    return sm.DeviceHybridGrid(synthetic.HybridGridSpec(
        res, np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(val, np.uint16)))


def _box_case(lo, hi, nonzero):
    """Zero voxels at the box's corners lo / hi (unless a non-zero cell is there), and the
    listed non-zero cells: every voxel listed once."""
    nonzero = np.asarray(nonzero, np.int64).reshape(-1, 3)
    zeros = [c for c in (lo, hi) if not (nonzero == np.asarray(c)).all(1).any()]
    idx = np.concatenate([np.reshape(zeros, (-1, 3)), nonzero]).astype(np.int32)
    val = np.concatenate([np.zeros(len(zeros)),
                          1000 + np.arange(len(nonzero)) * 7 % 30000]).astype(np.uint16)
    assert len(np.unique(idx, axis=0)) == len(idx)
    return idx, val


def _walk_cases():
    cases = {}
    lo, hi = np.array([-70, -3, 5]), np.array([229, 60, 40])   # 300 x 64 x 36: partial blocks
    for k in range(8):
        corner = np.where([(k >> a) & 1 for a in range(3)], hi, lo)
        cases["corner%d" % k] = _box_case(lo, hi, [corner])
    for a in range(3):
        for s, end in (("lo", lo), ("hi", hi)):
            face = []
            for u in (0, 7, 13):
                c = lo + (hi - lo) * np.array([u, 13 - u, u % 5]) // 13
                c[a] = end[a]
                face.append(c)
            cases["face%d_%s" % (a, s)] = _box_case(lo, hi, face)
    cases["last_x_column"] = _box_case(lo, hi, [[hi[0], y, z] for y, z in
                                                ((lo[1], lo[2]), (7, 20), (hi[1], hi[2]))])
    # more y * z rows (300 * 250) than one launch's gridDim.y (at most 65 535)
    rlo, rhi = np.array([0, -150, -125]), np.array([3, 149, 124])
    cases["rows_beyond_grid"] = _box_case(rlo, rhi, [[1, 149, 124], [3, -150, 124],
                                                     [0, 0, -125]])
    # 64-multiples at negative coordinates, and the cube's faces
    cases["straddle_neg64"] = _box_case([-130, -65, -64], [-60, -1, 64],
                                        [[-129, -65, -64], [-128, -64, -1], [-65, -1, 0],
                                         [-64, -2, 63], [-63, -64, 64]])
    cases["cube_faces"] = _box_case([-8192, -5, -3], [8191, 5, 3],
                                    [[-8192, -5, -3], [8191, 5, 3], [-8129, 0, 0],
                                     [8128, 1, 1]])
    # the last cell of thread 255's row in tile 0 and tile 127 of a 64^3 block
    tlo = np.array([-128, -64, 0])
    cases["tile_last_cell"] = _box_case(tlo - 5, tlo + 70, [tlo + [31, 7, 7]])
    cases["block_last_cell"] = _box_case(tlo - 5, tlo + 70, [tlo + [63, 63, 63]])
    # rows of one 8^3 block whose (y, z) order and (z, y) order differ: z is the outer one
    cases["rows_in_one_block"] = _box_case(tlo - 5, tlo + 70,
                                           [tlo + [2, y, z] for y, z in
                                            ((1, 0), (0, 1), (7, 2), (2, 7), (3, 3))])
    cases["all_zero"] = _box_case(lo, hi, np.zeros((0, 3)))
    return cases


WALK_CASES = _walk_cases()


def _nonzero_box(idx, val):
    nz = idx[val != 0]
    if len(nz) == 0:
        return None
    return nz.min(0), nz.max(0)


@pytest.mark.parametrize("case", sorted(WALK_CASES))
def test_nonzero_box_and_voxel_walk(sm, case):
    idx, val = WALK_CASES[case]
    g = _handle(sm, idx, val)
    before = g.read()
    keep = val != 0
    want_idx, want_val, _ = R.walk((idx[keep], val[keep]))
    got_idx, got_val = g.voxels()
    np.testing.assert_array_equal(got_idx, want_idx)
    np.testing.assert_array_equal(got_val, want_val)
    assert g.to_proto() == R.hybrid_grid_message(g.resolution, want_idx, want_val)
    box = _nonzero_box(idx, val)
    if box is not None:   # the walk's voxels span exactly the numpy non-zero box
        np.testing.assert_array_equal(got_idx.min(0), box[0])
        np.testing.assert_array_equal(got_idx.max(0), box[1])
    pose = (0.3, -0.2, 0.1, 1.0, 0.0, 0.0, 0.0)
    msg = g.to_texture(pose)
    want = T.texture3d(want_idx, want_val, g.resolution, pose)
    got = T.parse(msg)
    assert got["cells"] == want["cells"]
    assert (got["width"], got["height"]) == (want["width"], want["height"])
    # the from-grid matcher's level boxes and grid size follow the non-zero box
    od = worlds3d.fast_options(depth=3, frd=2)
    o = sm.FastCorrelativeScanMatcherOptions3D(
        od["branch_and_bound_depth"], od["full_resolution_depth"], od["min_rotational_score"],
        od["min_low_resolution_score"], od["linear_xy_search_window"],
        od["linear_z_search_window"], od["angular_search_window"])
    lo_g = _handle(sm, idx, val, 0.45)
    spec = synthetic.HybridGridSpec(0.1, idx[keep], val[keep])
    lspec = synthetic.HybridGridSpec(0.45, idx[keep], val[keep])
    hist = np.zeros(10, np.float32)
    a = sm.FastCorrelativeScanMatcher3D.from_device_grids(g, lo_g, hist, o)
    b = sm.FastCorrelativeScanMatcher3D(spec, lspec, hist, o)
    for d in range(3):
        la, va = a.precomputation_grid(d)
        lb, vb = b.precomputation_grid(d)
        np.testing.assert_array_equal(la, lb)
        np.testing.assert_array_equal(va, vb)
    node = sm.TrajectoryNodeData3D(worlds3d.random_cloud(np.random.RandomState(2), 30, 0.4),
                                   worlds3d.random_cloud(np.random.RandomState(3), 10, 0.4), hist)
    q = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    if box is None or (box[1] - box[0]).max() < 1024:   # a lattice the engine can hold
        ta, tb = a.score_top(True, q, q, node, 0.0), b.score_top(True, q, q, node, 0.0)
        assert (ta["nxc"], ta["nzc"]) == (tb["nxc"], tb["nzc"])
    after = g.read()
    np.testing.assert_array_equal(before[0], after[0])
    np.testing.assert_array_equal(before[1], after[1])
    for h in (a, b, g, lo_g):
        h.close()


@pytest.mark.parametrize("side", ["low", "high"])
def test_grid_size_at_powers_of_two(sm, side):
    """A non-zero box whose extent sits just inside and just outside 256 cells from 0 (grid size
    512 or 1024), with zero voxels beyond it: the from-grid matcher's derived grid size equals
    the list-built one.  (64 and 128 are test_gpu_matcher3d_from_grid.py's.)"""
    k = 3
    edge = 64 << (k - 1)
    hist = np.zeros(10, np.float32)
    od = worlds3d.fast_options(depth=5, frd=3)
    o = sm.FastCorrelativeScanMatcherOptions3D(
        od["branch_and_bound_depth"], od["full_resolution_depth"], od["min_rotational_score"],
        od["min_low_resolution_score"], od["linear_xy_search_window"],
        od["linear_z_search_window"], od["angular_search_window"])
    node = sm.TrajectoryNodeData3D(worlds3d.random_cloud(np.random.RandomState(k), 30, 0.4),
                                   worlds3d.random_cloud(np.random.RandomState(k), 10, 0.4), hist)
    q = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    nxc = []
    for far in ((-edge, -edge - 1) if side == "low" else (edge - 1, edge)):
        zero = far - 5 if side == "low" else far + 5
        idx = np.array([[0, 0, 0], [far, 1, 0], [zero, 0, 0]], np.int32)
        val = np.uint16([20000, 25000, 0])
        hi, lo = _handle(sm, idx, val), _handle(sm, idx, val, 0.45)
        a = sm.FastCorrelativeScanMatcher3D.from_device_grids(hi, lo, hist, o)
        b = sm.FastCorrelativeScanMatcher3D(synthetic.HybridGridSpec(0.1, idx[:2], val[:2]),
                                            synthetic.HybridGridSpec(0.45, idx[:2], val[:2]),
                                            hist, o)
        ta, tb = a.score_top(True, q, q, node, 0.0), b.score_top(True, q, q, node, 0.0)
        assert (ta["nxc"], ta["nzc"]) == (tb["nxc"], tb["nzc"])
        for d in range(5):
            la, va = a.precomputation_grid(d)
            lb, vb = b.precomputation_grid(d)
            np.testing.assert_array_equal(la, lb)
            np.testing.assert_array_equal(va, vb)
        nxc.append(ta["nxc"])
        for h in (a, b, hi, lo):
            h.close()
    assert nxc[1] > nxc[0], "the grid size did not follow the non-zero box"
