"""The 2D map-writing kernels (csrc/insert2d.cu, csrc/insert_tsdf2d.cu, csrc/grid2d.cu) at the
edges where they go wrong: launch shapes, slot ranges, grid-stride wrap, many handles, shared
16-bit cells, TSDF claims and numerics, growth at the 30 000-cell guard.

After every call every cell, the limits and the known box equal the sequential restatements
(tests/insert2d_oracle.cc, tests/insert_tsdf2d_oracle.cc) bit for bit, no cell carries the
update marker, and wherever tests/map_writing2d_refs.py decides them, the cells equal its exact
or float64 reference too."""
import math
import time

import numpy as np
import pytest

from benchmarks import synthetic
from tests import insert2d_oracle as O
from tests import insert_tsdf2d_oracle as T
from tests import map_writing2d_refs as R

pytestmark = pytest.mark.gpu

F = np.float32
S = R.SUBPIXEL


@pytest.fixture(scope="module")
def sm():
    from cartographer_b200 import scan_matching
    return scan_matching


# ---- ProbabilityGrid helpers ----
class Twin:
    """A device handle, its restatement, and the state the float64 reference expects."""

    def __init__(self, sm, limits, cells=None):
        res, max_x, max_y, nx, ny = limits
        if cells is None:
            self.dev = sm.RealTimeGrid2D.empty(res, max_x, max_y, nx, ny)
            self.ora = O.Grid(res, max_x, max_y, nx, ny)
            self.want = (self.ora.limits, np.zeros((ny, nx), np.uint16), None, True)
        else:
            self.dev = sm.RealTimeGrid2D(synthetic.GridSpec(cells, res, max_x, max_y))
            self.ora = O.Grid(res, max_x, max_y, nx, ny, cells)
            self.want = (self.ora.limits, cells.copy(), R.nonzero_box(cells), True)

    def expect(self, origin, returns, misses, tables, free_space):
        L, cells, box, _ = self.want
        self.want = R.expected_probability_grid(L, cells, box, origin, returns, misses, tables,
                                                free_space)

    def check(self, float64=True):
        st = self.dev.read()
        res, max_x, max_y, nx, ny = self.ora.limits
        assert (st.resolution, st.max_x, st.max_y) == (res, max_x, max_y)
        assert st.cells.shape == (ny, nx)
        assert not (st.cells & 0x8000).any(), "a cell still carries the update marker"
        np.testing.assert_array_equal(st.cells, self.ora.cells)
        assert st.known_cells_box == self.ora.known_box
        if float64 and self.want is not None and self.want[3]:
            assert self.ora.limits == self.want[0]
            np.testing.assert_array_equal(st.cells, self.want[1])
            assert st.known_cells_box == self.want[2]
        return st


def _inserters(sm, free_space=True, hit=0.55, miss=0.49):
    dev = sm.ProbabilityGridRangeDataInserter2D(
        sm.ProbabilityGridRangeDataInserterOptions2D(hit, miss, free_space))
    ora = O.Inserter(hit, miss, free_space)
    return dev, ora, ora.tables()


def _insert(ins, twins, origin, returns, misses, float64=True, one_call=True):
    """One insert_submaps call (or single Insert calls) on the devices, single inserts on the
    restatements, and the float64 expectation."""
    dev, ora, tables = ins
    free_space = dev.options.insert_free_space
    if one_call:
        dev.insert_submaps([t.dev for t in twins], origin, returns, misses)
        assert dev.last_stats["host_syncs"] == 1
    else:
        for t in twins:
            dev.Insert(origin, returns, t.dev, misses)
    for t in twins:
        ora.insert(origin, returns, t.ora, misses)
        if float64:
            t.expect(origin, returns, misses, tables, free_space)
        else:
            t.want = None


def _limits(origin, resolution, nx=100, ny=100, shift=(0.0, 0.0)):
    """CreateGrid's limits around `origin` (nx x ny), moved by `shift` cells, so that the origin
    is off the cell corners when the shift is fractional."""
    r = float(F(resolution))
    o = np.asarray(origin, F).astype(np.float64)
    return (r, o[0] + (0.5 * ny + shift[0]) * r, o[1] + (0.5 * nx + shift[1]) * r, nx, ny)


def _cloud(rng, origin, n, spread):
    return np.column_stack([origin[0] + rng.uniform(-spread, spread, n),
                            origin[1] + rng.uniform(-spread, spread, n),
                            np.zeros(n)]).astype(F)


# ---- launch shapes ----
SIZES = (1, 31, 32, 33, 255, 256, 257, 4097, 65537)


@pytest.mark.parametrize("pattern", R.LANE_PATTERNS)
@pytest.mark.parametrize("n", SIZES)
def test_launch_shapes(sm, n, pattern):
    """The one point that extends every handle's touched box sits at the lane or block edge the
    pattern names; free space, misses and handle counts vary with the case."""
    case = SIZES.index(n) * 4 + R.LANE_PATTERNS.index(pattern)
    free_space = case % 2 == 0
    with_misses = (case // 2) % 2 == 1
    H = 1 + case % 3
    rng = np.random.RandomState(case)
    origin = np.float32([1.2137, -0.4211, 0])
    twins = [Twin(sm, _limits(origin, (0.05, 0.1, 0.04)[h], shift=(0.3117 * h + 0.1731, 0.2349)))
             for h in range(H)]
    ins = _inserters(sm, free_space)
    ret = _cloud(rng, origin, n, 0.4)
    k = R.extreme_index(pattern, n)
    far = np.float32([[origin[0] - 1.3, origin[1] + 1.1, 0], [origin[0] + 1.7, origin[1] - 0.9, 0]])
    ret[k] = far[case % 2]
    mis = _cloud(rng, origin, n, 1.0) if with_misses else None
    if with_misses:
        mis[k] = far[1 - case % 2] * np.float32([1.01, 1.01, 0])
    _insert(ins, twins, origin, ret, mis, float64=n <= 4097)
    for t in twins:
        assert n > 4097 or t.want[3]
        t.check()
    # the box lies strictly inside the grid: an idle lane's identity would show as index 0
    for t in twins:
        box = t.dev.read().known_cells_box
        assert box[0] > 0 and box[1] > 0


# ---- many handles ----
def _mixed_twins(sm, rng, H, origin):
    """Handle 0 is the largest; the others mix resolutions, origins, nx not a multiple of 8,
    handles made from cells (whose known box is computed lazily) and handles that grow."""
    twins = [Twin(sm, _limits(origin, 0.05, 200, 200, shift=(0.3013, 0.7071)))]
    for h in range(1, H):
        res = (0.05, 0.1, 0.03, 0.07)[h % 4]
        nx, ny = 37 + (h * 7) % 50, 41 + (h * 11) % 40
        lim = _limits(origin + rng.uniform(-0.5, 0.5, 3).astype(F), res, nx, ny,
                      shift=(rng.rand(), rng.rand()))
        if h % 3 == 1:
            cells = np.zeros((ny, nx), np.uint16)
            y0, x0 = rng.randint(0, ny - 3), rng.randint(0, nx - 3)
            cells[y0:y0 + 3, x0:x0 + 3] = rng.randint(1, 32768, size=(3, 3))
            twins.append(Twin(sm, lim, cells))
        else:
            twins.append(Twin(sm, lim))
    return twins


@pytest.mark.parametrize("H", [1, 2, 31, 32, 33, 257])
def test_many_handles_equal_single_calls(sm, H):
    rng = np.random.RandomState(100 + H)
    origin = np.float32([0.4137, 0.2211, 0])
    twins = _mixed_twins(sm, rng, H, origin)
    shapes = [t.dev.shape for t in twins]
    singles = _mixed_twins(sm, np.random.RandomState(100 + H), H, origin)
    ins = _inserters(sm)
    for k in range(2):
        ret = _cloud(rng, origin, 300, 1.2 + 2.0 * k)   # the second scan grows the small ones
        mis = _cloud(rng, origin, 50, 2.5 + 2.0 * k)
        _insert(ins, twins, origin, ret, mis, float64=H <= 33)
        assert H > 33 or all(t.want[3] for t in twins)
        _insert(ins, singles, origin, ret, mis, float64=False, one_call=False)
        for a, b in zip(twins, singles):
            sa, sb = a.check(), b.check(float64=False)
            np.testing.assert_array_equal(sa.cells, sb.cells)
            assert sa.known_cells_box == sb.known_cells_box
    grew = [t.dev.shape != s for t, s in zip(twins, shapes)]
    assert H == 1 or (any(grew) and not all(grew))


def test_gridDim_y_limit_and_one_past_it(sm):
    """65 535 small handles in one call (the blockIdx.y limit), then 65 536, which is refused
    before anything changes."""
    H = 65535
    origin = np.float32([0.0137, 0.0211, 0])
    kinds = [_limits(origin, (0.05, 0.1, 0.07)[k % 3], 8 + k, 9 + k, shift=(0.1013 * k, 0.3071))
             for k in range(5)]
    t0 = time.perf_counter()
    devs = [sm.RealTimeGrid2D.empty(*kinds[h % 5][:3], kinds[h % 5][3], kinds[h % 5][4])
            for h in range(H + 1)]
    t1 = time.perf_counter()
    oras = [O.Grid(*kinds[k]) for k in range(5)]
    ins = _inserters(sm)
    rng = np.random.RandomState(7)
    ret = _cloud(rng, origin, 5, 0.15)
    mis = _cloud(rng, origin, 3, 0.2)
    ins[0].insert_submaps(devs[:H], origin, ret, mis)
    t2 = time.perf_counter()
    for o in oras:
        ins[1].insert(origin, ret, o, mis)
    want = [(o.limits, o.cells, o.known_box) for o in oras]
    for h in range(H):
        st = devs[h].read()
        L, cells, box = want[h % 5]
        assert (st.resolution, st.max_x, st.max_y) == L[:3]
        np.testing.assert_array_equal(st.cells, cells)
        assert st.known_cells_box == box
    before = devs[H].read()
    from cartographer_b200._lib import CsmError
    with pytest.raises(CsmError) as e:
        ins[0].insert_submaps(devs, origin, ret, mis)
    assert e.value.status == 1
    for h in list(range(0, H, 997)) + [H - 1]:
        st = devs[h].read()
        np.testing.assert_array_equal(st.cells, want[h % 5][1])
    st = devs[H].read()
    np.testing.assert_array_equal(st.cells, before.cells)
    assert st.known_cells_box is None
    print(f"\n65535 handles: creation {t1 - t0:.1f} s, one insert_submaps call {t2 - t1:.2f} s, "
          f"device {ins[0].last_stats['device_ms']:.1f} ms")
    for d in devs:
        d.close()


# ---- slot ranges ----
def _corner_rays(origin_cell_xy, limits, far):
    """Points whose rays from an origin near a pixel corner cross it in far less than a cell:
    3 pixels each, the exact corner (2 pixels), zero length (1) and axis-parallel rays ending
    on borders.  Subpixel offsets grow with the coordinates' float32 ulp."""
    res, max_x, max_y, nx, ny = limits
    sres = res / S
    X, Y = origin_cell_xy   # the pixel corner (X s, Y s) in superscaled units
    step = 3 if not far else 4   # subpixels; at 600 m a float32 ulp is about 1.2 subpixels

    def point(sx, sy):   # a float32 point at superscaled index (sx, sy) + 1/2
        return (F(max_x - (sy + 1.0) * sres), F(max_y - (sx + 1.0) * sres))
    o = point(X - step, Y - step)
    pts = []
    for a in range(1, 6):
        for b in range(1, 6):
            if a != b:
                pts.append(point(X + step * a // 2, Y + step * b // 2))   # 3 pixels
    pts.append(point(X + step, Y + step))    # through the corner
    pts.append(point(X - step, Y - step))    # zero length
    pts.append(point(X - step, Y + 2 * S))   # axis-parallel, ending near a border
    pts.append(point(X - step, Y + S))
    return np.float32([o[0], o[1], 0]), np.float32([[p[0], p[1], 0] for p in pts])


@pytest.mark.parametrize("far", [False, True])
def test_tightest_reservation(sm, far):
    """65 537 rays of about 3 pixels each against a reservation of 3 R + 1 + ΣL1 / res."""
    base = np.float32([600.3, -599.7]) if far else np.float32([0.3, 0.2])
    lim = _limits(base, 0.05, 100, 100, shift=(0.5, 0.5))
    twin = Twin(sm, lim)
    ins = _inserters(sm)
    origin, pts = _corner_rays((52 * S, 47 * S), lim, far)
    reps = -(-65537 // len(pts))
    ret = np.tile(pts, (reps, 1))[:65537]
    o, ends, decided = R.superscaled_ends(lim, origin, ret)
    total = R.exact_slot_total(o, ends)
    cap = R.slot_reservation(R.l1_sum(origin, ret), lim[0], len(ret))
    assert 2.9 * len(ret) < total <= cap < 3.2 * len(ret)
    _insert(ins, [twin], origin, ret, None)
    twin.check()
    assert decided or far
    # the same rays as misses only: every ray's pixels are misses
    twin2 = Twin(sm, lim)
    _insert(ins, [twin2], origin, np.zeros((0, 3), F), ret)
    twin2.check()


def test_grid_stride_wrap(sm):
    """Rays of about 300 m at 0.05 m: more than 2^24 slots in one handle, so the miss and
    finish kernels' grid-stride loops run a second pass; once alone, once beside a handle that
    does not wrap."""
    base = _device_mib()
    rng = np.random.RandomState(9)
    origin = np.float32([0.0137, 0.0211, 0])
    a = rng.uniform(0, 2 * np.pi, 3000)
    r = rng.uniform(280.0, 300.0, 3000)
    ret = np.column_stack([origin[0] + r * np.cos(a), origin[1] + r * np.sin(a),
                           np.zeros(3000)]).astype(F)
    lim = _limits(origin, 0.05)
    cap = R.slot_reservation(R.l1_sum(origin, ret), lim[0], 3000)
    assert cap > 1 << 24
    ins = _inserters(sm)
    for second in (False, True):
        twins = [Twin(sm, lim)] + ([Twin(sm, _limits(origin, 1.0, 37, 45, (0.3, 0.6)))]
                                   if second else [])
        _insert(ins, twins, origin, ret, None, float64=False)
        ms = ins[0].last_stats["device_ms"]
        print(f"\nwrap, {len(twins)} handle(s): {cap} slots reserved, device {ms:.1f} ms, "
              f"{_device_mib() - base:.0f} MiB more device memory in use than before the test")
        for t in twins:
            t.check(float64=False)
        # The time is the only observable of a stride that revisits slots: the update markers
        # make a second visit change no cell.  A stride of one block (every slot visited by
        # thousands of threads) took 2.8 s of device time on an H100; the bound is generous
        # against the milliseconds a correct launch takes, so a shared GPU does not trip it.
        assert ms < 1000.0, ms
        for t in twins:
            t.dev.close()
            t.ora.close()


def _device_mib():
    """Device memory in use on the current device, in MiB: the difference of two readings is
    what the test allocated, as long as nothing else on the device changes meanwhile."""
    import torch
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2 ** 20


# ---- per-cell interactions ----
def test_cells_shared_by_rays_returns_and_words(sm):
    lim = (0.05, 1.0, 2.0, 45, 37)   # pitch 48 > nx
    res, max_x, max_y, nx, ny = lim
    ins = _inserters(sm, hit=0.7, miss=0.4)

    def centre(x, y):   # near the centre of cell (x, y), off the subpixel borders
        return [F(max_x - (y + 0.5) * res + 0.00137), F(max_y - (x + 0.5) * res + 0.00211)]
    origin = np.float32(centre(20, 18) + [0]) + np.float32([0.0037, 0.0011, 0])
    ret = np.float32([
        centre(25, 18) + [0],     # a return's cell on the next ray's mask
        centre(30, 18) + [0],
        centre(10, 5) + [0], centre(10, 5) + [0],   # two returns in one cell
        centre(12, 30) + [0],     # hit at x = 12 (even) ...
        centre(44, 2) + [0], centre(44, 36) + [0],   # the last column
    ])
    mis = np.float32([centre(13, 31) + [0], centre(13, 30) + [0]])   # ... miss at x = 13
    for order in (1, -1):
        twin = Twin(sm, lim)
        _insert(ins, [twin], origin, ret[::order], mis)
        assert twin.want[3]
        st = twin.check()
        assert st.cells[18, 25] == ins[2][0][0] & 0x7fff   # hit wins over the later mask
        assert st.cells[30, 12] == ins[2][0][0] & 0x7fff
        assert st.cells[30, 13] == ins[2][1][0] & 0x7fff
        assert st.cells[2, 44] == ins[2][0][0] & 0x7fff
    # both halves of one word touched in one insert, over a known grid
    cells = np.full((ny, nx), 1000, np.uint16)
    twin = Twin(sm, lim, cells)
    for k in range(3):
        _insert(ins, [twin], origin, ret, mis)
        twin.check()


# ---- growth ----
def test_growth_to_the_guard_and_one_cell_past_it(sm):
    base = _device_mib()
    from cartographer_b200._lib import CsmError
    origin = np.float32([0.0137, 0.0211, 0])
    lim = _limits(origin, 0.05)
    ins = _inserters(sm)
    twin = Twin(sm, lim)
    # 600 m out: 100 -> 25 600 cells in one call, returns beyond 16 m where the padding is
    # absorbed in float32
    ret = np.float32([[origin[0] - 600.0, origin[1] + 3.0, 0], [40.0, -48.0, 0],
                      [origin[0] + 17.0, origin[1] - 33.0, 0]])
    grown = R.grow_as_needed(lim, origin, ret)
    assert grown[0][3] == 25600
    _insert(ins, [twin], origin, ret, None, float64=False)
    st = twin.check(float64=False)
    assert st.cells.shape == (25600, 25600)
    print(f"\n25600^2 grid: {_device_mib() - base:.0f} MiB more device memory in use than "
          "before the test")
    L = twin.ora.limits
    assert L == grown[0]
    before = (st.cells, st.known_cells_box)
    del st
    # one cell past the grown border: refused, and so for every handle of the call
    small = Twin(sm, lim)
    far = np.float32([[F(L[1] + 0.5 * L[0]), origin[1], 0]])
    assert R.grow_as_needed(L, origin, far) is None
    with pytest.raises(CsmError) as e:
        ins[0].insert_submaps([small.dev, twin.dev], origin, far)
    assert e.value.status == 1
    st = twin.dev.read()
    np.testing.assert_array_equal(st.cells, before[0])
    assert st.known_cells_box == before[1]
    small.check()
    del st, before
    # an origin on the grown grid's lower border, then the crop
    res, max_x, max_y, nx, ny = L
    o2 = np.float32([F(max_x - ny * res + 1e-3), F(max_y - nx * res + 2e-3), 0])
    _insert(ins, [twin], o2, ret + np.float32([0.1, 0.1, 0]), None, float64=False)
    st = twin.check(float64=False)
    crop = twin.dev.ComputeCroppedGrid()
    cst = crop.read()
    box = R.nonzero_box(st.cells)
    assert box == st.known_cells_box
    np.testing.assert_array_equal(cst.cells, twin.ora.crop().cells)
    assert cst.cells.shape == (box[3] - box[1] + 1, box[2] - box[0] + 1)
    np.testing.assert_array_equal(cst.cells, st.cells[box[1]:box[3] + 1, box[0]:box[2] + 1])
    crop.close()
    twin.dev.close()
    twin.ora.close()


def test_guard_at_15000_cells(sm):
    """7 500 cells double to 15 000; the next doubling would reach 30 000 and is refused."""
    from cartographer_b200._lib import CsmError
    origin = np.float32([0.0137, 0.0211, 0])
    lim = _limits(origin, 0.05, 7500, 7500)
    ins = _inserters(sm)
    twin = Twin(sm, lim)
    ret = np.float32([[origin[0] + 200.0, origin[1], 0]])
    _insert(ins, [twin], origin, ret, None, float64=False)
    st = twin.check(float64=False)
    assert st.cells.shape == (15000, 15000)
    L = twin.ora.limits
    far = np.float32([[F(L[1] + 0.5 * L[0]), origin[1], 0]])
    with pytest.raises(CsmError):
        ins[0].Insert(origin, far, twin.dev)
    assert twin.dev.read().cells.shape == (15000, 15000)
    twin.dev.close()
    twin.ora.close()


# ---- TSDF ----
def _tsdf_opts(sm, **kw):
    base = dict(truncation_distance=0.3, maximum_weight=10.0, update_free_space=False,
                project_sdf_distance_to_scan_normal=False, update_weight_range_exponent=0,
                update_weight_angle_scan_normal_to_ray_kernel_bandwidth=0.0,
                update_weight_distance_cell_to_hit_kernel_bandwidth=0.0)
    base.update(kw)
    opts = sm.TSDFRangeDataInserterOptions2D(**base)
    return sm.TSDFRangeDataInserter2D(opts), T.TsdfInserter(opts), opts


def _tsdf_twin(sm, limits, truncation, max_weight, tsd=None, weight=None):
    res, max_x, max_y, nx, ny = limits
    if tsd is None:
        return (sm.RealTimeGrid2D.empty_tsdf(res, max_x, max_y, truncation, max_weight, nx, ny),
                T.TsdfGrid(res, max_x, max_y, nx, ny, truncation, max_weight))
    spec = sm.TSDF2DSpec(tsd, weight, res, max_x, max_y, truncation, max_weight)
    return (sm.RealTimeGrid2D(spec),
            T.TsdfGrid(res, max_x, max_y, nx, ny, truncation, max_weight, tsd, weight))


def _tsdf_insert(ins, twin, origin, returns):
    """One insert on both sides; where the restatement refuses, the device must refuse too.
    Then every cell, the limits and the box, and no update marker."""
    from cartographer_b200._lib import CsmError
    dev_ins, ora_ins, _ = ins
    dev, ora = twin
    if ora_ins.insert(origin, returns, ora):
        dev_ins.Insert(origin, returns, dev)
        assert dev_ins.last_stats["host_syncs"] == 1
        accepted = True
    else:
        with pytest.raises(CsmError):
            dev_ins.Insert(origin, returns, dev)
        accepted = False
    st = dev.read()
    res, max_x, max_y, nx, ny = ora.limits
    assert (st.resolution, st.max_x, st.max_y) == (res, max_x, max_y)
    tsd, weight = ora.arrays()
    np.testing.assert_array_equal(st.cells, tsd)
    np.testing.assert_array_equal(st.weight_cells, weight)
    assert st.known_cells_box == ora.known_box
    assert not (st.cells & 0x8000).any() and not (st.weight_cells & 0x8000).any()
    return accepted, st


def _check_float64(st, want, min_decided=1):
    decided = 0
    for (x, y), (tv, wv, ok) in want.items():
        if ok:
            assert (int(st.cells[y, x]), int(st.weight_cells[y, x])) == (tv, wv), (x, y)
            decided += 1
    assert decided >= min_decided
    return decided


@pytest.mark.parametrize("num_rays", [1, 255, 256, 257, 65537])
def test_tsdf_ray_counts(sm, num_rays):
    rng = np.random.RandomState(num_rays)
    origin = np.float32([0.2137, 0.1211, 0])
    lim = _limits(origin, 0.05, 200, 200, shift=(0.3731, 0.4117))
    ins = _tsdf_opts(sm, update_weight_distance_cell_to_hit_kernel_bandwidth=0.1 * (num_rays % 2))
    twin = _tsdf_twin(sm, lim, 0.3, 10.0)
    a = rng.uniform(0, 2 * np.pi, num_rays)
    r = rng.uniform(0.35, 3.5, num_rays)
    ret = np.column_stack([origin[0] + r * np.cos(a), origin[1] + r * np.sin(a),
                           np.zeros(num_rays)]).astype(F)
    accepted, st = _tsdf_insert(ins, twin, origin, ret)
    assert accepted
    if num_rays <= 257:
        want = R.tsdf_expected(twin[1].limits, origin, ret, 0.3, 10.0,
                               sigma=ins[2].update_weight_distance_cell_to_hit_kernel_bandwidth)
        _check_float64(st, want)


def _return_with_count(limits, origin, direction, count, truncation):
    """A return along an axis whose free-space ray (origin to band end) has exactly `count`
    slots: along an axis the count grows by one pixel per cell of range."""
    res = limits[0]
    for k in range(int(4 * count * 8)):
        r = truncation + k * res / 8
        p = np.float32([origin[0] + direction[0] * r, origin[1] + direction[1] * r, 0])
        ray = R._tsdf_ray64(limits, origin, p, F(truncation), True)
        c = R.count_bound(ray[1], ray[2])
        if c == count:
            return p
        assert c < count
    raise AssertionError(count)


@pytest.mark.parametrize("count", [255, 256, 257, 511, 512, 513])
def test_tsdf_slot_totals_straddle_multiples_of_256(sm, count):
    """Free-space rays along the four axes whose |dx| + |dy| + 1 slot counts add up to exactly
    255, 256, 257, 511, 512 and 513: the slot kernels' last block is full, one slot short of it
    or one slot into the next."""
    origin = np.float32([0.2137, 0.1211, 0])
    lim = _limits(origin, 0.05, 200, 200, shift=(0.3731, 0.4117))
    ins = _tsdf_opts(sm, truncation_distance=0.3, update_free_space=True)
    twin = _tsdf_twin(sm, lim, 0.3, 10.0)
    parts = -(-count // 50)
    counts = [count // parts + (i < count % parts) for i in range(parts)]
    axes = ((1, 0), (0, 1), (-1, 0), (0, -1))
    ret = np.float32([_return_with_count(lim, origin, axes[i % 4], c, 0.3)
                      for i, c in enumerate(counts)])
    o, e = [], []
    for p in ret:
        _, b, end = R._tsdf_ray64(lim, origin, p, F(0.3), True)
        o.append(b)
        e.append(end)
    assert sum(R.count_bound(b, end) for b, end in zip(o, e)) == count
    accepted, st = _tsdf_insert(ins, twin, origin, ret)
    assert accepted and st.cells.shape == (200, 200)
    _check_float64(st, R.tsdf_expected(twin[1].limits, origin, ret, 0.3, 10.0, free_space=True))


def _axis_claims_float64(limits, origin, ret, truncation, sigma):
    """Each cell's winner among rays along the four axes, in float64: the first ray in input
    order whose weight is non-zero.  {(x, y): (tsd value, weight value)} for the decided cells,
    and how many decided cells had a zero-weight first claim."""
    out, skipped = {}, 0
    t = float(F(truncation))
    rays = {}
    for k, p in enumerate(ret):
        ray = R._tsdf_ray64(limits, origin, p, F(truncation), False)
        if ray is not None:
            rays[k] = ray
    cells = {}
    for k, (rng, b, e) in rays.items():
        for c in R.geometric_mask(b, e):
            cells.setdefault(c, []).append(k)
    least = 2.0 ** -149
    for c, ks in cells.items():
        zero_first = False
        for k in ks:
            rng = rays[k][0]
            ut, uw, err = R.tsdf_pair64(limits, origin, rng, c[0], c[1], t, 1.0, sigma)
            w_hi = R._gaussian64(max(abs(ut) - err, 0.0), sigma)
            w_lo = R._gaussian64(min(abs(ut) + err, t), sigma)
            if w_hi < least / 4:
                zero_first = True
                continue
            if w_lo > 2.0 ** -100:
                tv, tdist, tres = R.tsdf_value64(ut, -t, t)
                wv, wdist, wres = R.tsdf_value64(uw, 0.0, 10.0)
                w_rel = R.F32_ERROR_ULPS * 2.0 ** -24 * 2 + (abs(ut) + err) * err / sigma ** 2
                if tdist > err * tres and wdist > w_rel * uw * wres:
                    out[c] = (tv, wv)
                    skipped += zero_first
            break
    return out, skipped


def test_tsdf_claims_across_radix_passes(sm):
    """2^17 returns along the four axes at different ranges: thousands of pairs claim each cell
    near the origin, and the first claims of many cells have a weight of exactly 0.f (the
    distance kernel underflows), so a later pair must win."""
    origin = np.float32([0.2137, 0.1211, 0])
    lim = _limits(origin, 0.05, 200, 200, shift=(0.3731, 0.4117))
    sigma = 0.02
    ins = _tsdf_opts(sm, update_weight_distance_cell_to_hit_kernel_bandwidth=sigma)
    twin = _tsdf_twin(sm, lim, 0.3, 10.0)
    n = 1 << 17
    rng = np.random.RandomState(17)
    d = rng.randint(0, 4, n)
    r = F(0.3) + rng.randint(0, 40, n).astype(F) * F(0.0173)
    ux = np.float32([1, 0, -1, 0])[d]
    uy = np.float32([0, 1, 0, -1])[d]
    ret = np.column_stack([origin[0] + r * ux, origin[1] + r * uy, np.zeros(n)]).astype(F)
    accepted, st = _tsdf_insert(ins, twin, origin, ret)
    assert accepted
    want, skipped = _axis_claims_float64(twin[1].limits, origin, ret[:4096], 0.3, sigma)
    # the first 4096 rays decide the cells they claim only if no later ray comes first: compare
    # the cells whose every claiming ray is among them (every range occurs in the first 4096)
    assert skipped > 0
    checked = 0
    for (x, y), (tv, wv) in want.items():
        assert (int(st.cells[y, x]), int(st.weight_cells[y, x])) == (tv, wv), (x, y)
        checked += 1
    assert checked > 50


@pytest.mark.parametrize("nx,ny", [(128, 128), (712, 23), (24, 683)])
def test_tsdf_sort_key_width(sm, nx, ny):
    """pitch * ny = 2^14, 2^14 - 8 and 2^14 + 8, with claims on flat index 0 and on the last
    flat index, each by two rays with different updates and non-claiming slots between."""
    assert nx * ny in (1 << 14, (1 << 14) - 8, (1 << 14) + 8)
    res = 0.05
    # the origin inside the grid, near its middle
    max_x, max_y = 3.0 + 0.0137, 2.0 + 0.0211
    lim = (res, max_x, max_y, nx, ny)
    origin = np.float32([max_x - ny * res / 2 + 0.0137, max_y - nx * res / 2 + 0.0211, 0])
    # free space on: every cell between the origin and the band has ut = +t, where a kernel of
    # bandwidth t / 16 underflows to a weight of 0.f, so those slots claim nothing
    t, sigma = 0.04, 0.0025
    ins = _tsdf_opts(sm, update_weight_distance_cell_to_hit_kernel_bandwidth=sigma,
                     truncation_distance=t, update_free_space=True)
    tsd = np.zeros((ny, nx), np.uint16)
    twin = _tsdf_twin(sm, lim, t, 10.0, tsd, tsd.copy())

    def toward(x, y, before):   # a return whose band claims cell (x, y) at ut = -before
        cx, cy = max_x - res * (y + 0.5), max_y - res * (x + 0.5)
        v = np.array([cx - origin[0], cy - origin[1]])
        dist = np.hypot(*v)
        r = dist - before
        return np.float32([origin[0] + v[0] / dist * r, origin[1] + v[1] / dist * r, 0])
    # the bands end less than half a cell past the corner cells' centres, inside the grid
    ret = np.float32([toward(0, 0, 0.017), toward(nx - 1, ny - 1, 0.018),
                      toward(0, 0, 0.021), toward(nx - 1, ny - 1, 0.022)])
    accepted, st = _tsdf_insert(ins, twin, origin, ret)
    assert accepted and st.cells.shape == (ny, nx)
    assert st.weight_cells[0, 0] and st.weight_cells[ny - 1, nx - 1]
    # Only the restatement decides these cells: at a truncation of 0.04 m one tsd value step is
    # 1.2e-6 m, below the float32 error of a distance of metres, so the float64 reference
    # leaves every claimed cell undecided.


@pytest.mark.parametrize("truncation", [0.3, 0.02])
def test_tsdf_range_at_the_truncation(sm, truncation):
    """A range equal to the truncation is inserted, one ulp below it is skipped; at 0.02 m the
    whole band lies in the origin's cell and its neighbours."""
    origin = np.float32([0.0, 0.1211, 0])   # hit x - origin x is the range exactly
    lim = _limits(origin, 0.05, shift=(0.3731, 0.4117))
    t = F(truncation)
    for rx, kept in ((t, True), (np.nextafter(t, F(0)), False)):
        ins = _tsdf_opts(sm, truncation_distance=float(t))
        twin = _tsdf_twin(sm, lim, float(t), 10.0)
        ret = np.float32([[origin[0] + rx, origin[1], 0]])
        assert F(math.sqrt(float(F(F(ret[0, 0] - origin[0]) ** 2)))) == rx
        accepted, st = _tsdf_insert(ins, twin, origin, ret)
        assert accepted
        assert bool(st.weight_cells.any()) == kept
        if kept:
            _check_float64(st, R.tsdf_expected(twin[1].limits, origin, ret, float(t), 10.0))


def test_tsdf_weight_quantisation_tie_and_maximum(sm):
    """maximum_weight = 32766 / 4096 makes the weight resolution exactly 4096; range exponent
    13 at a range of exactly 2 m gives every update a weight of 2^-13, which quantises on an
    exact .5: RoundToInt (half away from zero) stores 2, round-half-even would store 1."""
    mw = 32766 / 4096
    assert float(F(mw)) == mw
    origin = np.float32([0.2137, 0.1211, 0])
    lim = _limits(origin, 0.05, shift=(0.3731, 0.4117))
    ins = _tsdf_opts(sm, maximum_weight=mw, update_weight_range_exponent=13)
    twin = _tsdf_twin(sm, lim, 0.3, mw)
    ret = np.float32([[origin[0] + 2.0, origin[1], 0], [origin[0], origin[1] - 2.0, 0]])
    accepted, st = _tsdf_insert(ins, twin, origin, ret)
    assert accepted
    w = st.weight_cells[st.weight_cells != 0]
    assert len(w) > 10 and (w == 2).all()
    # weights that reach and then pass maximum_weight = 3 exactly, one unit per insert
    ins = _tsdf_opts(sm, maximum_weight=3.0)
    twin = _tsdf_twin(sm, lim, 0.3, 3.0)
    ret = np.float32([[origin[0] + 1.0, origin[1] + 0.5, 0]])
    for k in range(1, 6):
        accepted, st = _tsdf_insert(ins, twin, origin, ret)
        w = st.weight_cells[st.weight_cells != 0]
        want, _, _ = R.tsdf_value64(float(min(k, 3)), 0.0, 3.0)
        assert (w == want).all()
    assert want == 32767


def _tsd_ties(limits, origin, x_row, truncation, start, want=3):
    """Returns along +x from an origin on the centre line of cell row x_row, whose update of
    some cell quantises on an exact .5 with an even integer part: [(return x, cell y, q)].
    Along the row every float32 step is exact or one rounding the model repeats (the range is
    |rx|, a centre's distance is |dx|), and the truncation makes the tsd resolution 2^16, so
    q = (ut + t) * 65536 exactly."""
    res, max_x, _, _, ny = limits
    t32 = F(truncation)
    ox = origin[0]
    out = []
    hx = F(start)
    for _ in range(20000):
        hx = np.nextafter(hx, F(np.inf))
        rng = abs(F(hx - ox))
        for y in range(ny):
            cx = F(max_x - res * (y + 0.5))
            if cx <= ox:   # behind the origin: on no ray
                continue
            ut = F(rng - abs(F(cx - ox)))
            if not -t32 < ut < t32:
                continue
            q = float(F(ut + t32)) * 65536
            if q - math.floor(q) == 0.5 and math.floor(q) % 2 == 0:
                out.append((hx, y, q))
                break
        if len(out) == want:
            return out
    raise AssertionError("no tie found")


def test_tsdf_tsd_quantisation_tie(sm):
    """A truncation of 16383 / 65536 makes the tsd resolution exactly 2^16; a host search finds
    returns whose update of one cell quantises on k + .5 with k even.  RoundToInt (half away
    from zero) stores k + 2; round-half-even would store k + 1."""
    t = 16383 / 65536
    lim = (0.05, 3.0137, 2.0211, 100, 100)
    res, max_x, max_y, nx, ny = lim
    x_row = 47
    origin = np.float32([max_x - res * 50.3, max_y - res * (x_row + 0.5), 0])
    ties = _tsd_ties(lim, origin, x_row, t, origin[0] + F(1.3))
    for hx, y, q in ties:
        ins = _tsdf_opts(sm, truncation_distance=t)
        twin = _tsdf_twin(sm, lim, t, 10.0)
        accepted, st = _tsdf_insert(ins, twin, origin, np.float32([[hx, origin[1], 0]]))
        assert accepted
        assert int(st.cells[y, x_row]) == math.floor(q) + 2, (hx, y, q)


def _contraction_cells(ut_cells, truncation, max_weight, rng, tries=20000):
    """For each update ut (weight 1), an old (tsd value, weight value) pair whose stored tsd
    value differs between the unfused float32 average and the average with multiply-adds
    (exact fmaf), whichever product of tsd * w + ut * uw the multiply-add takes."""
    ts, tb, ws, wb = R.tsdf_conversion(truncation, max_weight)
    out = []
    for ut in ut_cells:
        tv = rng.randint(1, 32768, tries)
        wv = rng.randint(1, 32768, tries)
        # a float64 screen of the fused decodes and either fused product; the exact model
        # confirms
        tsd_f = (tv * np.float64(ts) + np.float64(tb)).astype(F)
        w_f = (wv * np.float64(ws) + np.float64(wb)).astype(F)
        num_f = (tsd_f.astype(np.float64) * w_f + np.float64(ut)).astype(F)
        num_f2 = ((tsd_f * w_f).astype(F).astype(np.float64) + np.float64(ut)).astype(F)
        tsd_u = ((tv * ts).astype(F) + tb).astype(F)
        w_u = ((wv * ws).astype(F) + wb).astype(F)
        num_u = ((tsd_u * w_u).astype(F) + F(ut)).astype(F)
        unfused = (num_u / (w_u + F(1))).astype(F)
        cand = np.nonzero(((num_f / (w_f + F(1))).astype(F) != unfused) |
                          ((num_f2 / (w_f + F(1))).astype(F) != unfused))[0]
        found = None
        # keep a pair only where the answer holds for ut and its two ulp neighbours, so that it
        # does not depend on the last bit of the update
        near = (np.nextafter(F(ut), F(-1)), F(ut), np.nextafter(F(ut), F(1)))
        for i in cand:
            a = {R.tsdf_update32(int(tv[i]), int(wv[i]), u, 1.0, truncation, max_weight, False)
                 for u in near}
            b = {R.tsdf_update32(int(tv[i]), int(wv[i]), u, 1.0, truncation, max_weight, f)
                 for u in near for f in R.FUSIONS}
            if len(a) == 1 and not a & b:
                found = (int(tv[i]), int(wv[i]), a.pop())
                break
        out.append(found)
    return out


def test_tsdf_no_contraction(sm):
    """Cells whose stored tsd differs when the decodes and either product of the weighted
    average are contracted into multiply-adds: the device stores the unfused value."""
    res, trunc, mw = 0.05, 0.3, 10.0
    origin = np.float32([0.2137, 0.1211, 0])
    lim = _limits(origin, res, 60, 60, shift=(0.3731, 0.4117))
    _, max_x, max_y, nx, ny = lim
    ret = np.float32([[origin[0] + 0.8, origin[1] + 0.3, 0]])
    ray = R._tsdf_ray64(lim, origin, ret[0], F(trunc), False)
    cells = sorted(R.geometric_mask(ray[1], ray[2]))
    # the device's float32 update of each cell (unfused, as -fmad=false builds it)
    rng32 = F(math.sqrt(float(F(F(ret[0, 0] - origin[0]) ** 2 + F(ret[0, 1] - origin[1]) ** 2))))
    uts = []
    for x, y in cells:
        cx, cy = F(max_x - res * (y + 0.5)), F(max_y - res * (x + 0.5))
        dx, dy = F(cx - origin[0]), F(cy - origin[1])
        ut = F(rng32 - F(math.sqrt(float(F(F(dx * dx) + F(dy * dy))))))
        uts.append(F(min(max(ut, -F(trunc)), F(trunc))))
    found = _contraction_cells(uts, trunc, mw, np.random.RandomState(11))
    tsd = np.zeros((ny, nx), np.uint16)
    wgt = np.zeros((ny, nx), np.uint16)
    expect = {}
    for (x, y), f in zip(cells, found):
        if f is not None:
            tsd[y, x], wgt[y, x] = f[0], f[1]
            expect[(x, y)] = f[2]
    assert len(expect) >= 3
    ins = _tsdf_opts(sm)
    twin = _tsdf_twin(sm, lim, trunc, mw, tsd, wgt)
    accepted, st = _tsdf_insert(ins, twin, origin, ret)
    assert accepted
    for (x, y), (tv, wv) in expect.items():
        assert (int(st.cells[y, x]), int(st.weight_cells[y, x])) == (tv, wv), (x, y)


def test_tsdf_band_leaves_the_grid_by_less_than_a_cell(sm):
    """Returns above the origin's height grow the grid by their 3D-normalised truncation, less
    than the 2D band: on each of the four sides the band ends past the edge by less than a
    cell.  Negative subpixel indices use C division there, so only the restatement decides
    (including its refusals)."""
    origin = np.float32([0.2137, 0.1211, 0])
    lim = _limits(origin, 0.05)
    res, max_x, max_y, nx, ny = lim
    lo_x, lo_y = max_x - ny * res, max_y - nx * res
    for k, past in enumerate((0.004, 0.02, 0.049, 0.03)):
        for side in range(4):
            ins = _tsdf_opts(sm)
            twin = _tsdf_twin(sm, lim, 0.3, 10.0)
            edge = [(max_x, None), (lo_x, None), (None, max_y), (None, lo_y)][side]
            sign = [1, -1, 1, -1][side]
            if edge[0] is not None:   # band end at edge + sign * past along x
                p = [edge[0] + sign * (past - 0.3), origin[1] + 0.01 * k]
            else:
                p = [origin[0] + 0.01 * k, edge[1] + sign * (past - 0.3)]
            dist = math.hypot(p[0] - origin[0], p[1] - origin[1])
            ret = np.float32([[p[0], p[1], 1.5 * dist]])   # 3D: growth adds only ~0.55 t
            _tsdf_insert(ins, twin, origin, ret)
