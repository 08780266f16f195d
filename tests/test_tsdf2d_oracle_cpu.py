"""CPU checks of the TSDF2D refinement: the restatement (tests/tsdf2d_oracle.py) against the
reference's known answers, and the device kernel's TSDF instantiation run in the CPU
emulation harness (tests/emulation/refine2d_tsdf_emulation.cc) against the restatement."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from benchmarks import synthetic
from tests import tsdf2d_oracle as T

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emulation")
SO = os.path.join(HERE, "_build", "librefine2d_tsdf_emulation.so")


def _interpolation_fixture():
    # interpolated_tsdf_2d_test.cc: MapLimits(1., (5.5, 5.5), CellLimits(10, 10)), 1.0, 10.0
    return T.TSDF2D(10, 10, 1.0, 5.5, 5.5, 1.0, 10.0)


def _set(g, x, y, tsd, w):
    ix, iy = g.cell_index(x, y)
    g.set_cell(int(ix), int(iy), tsd, w)


def test_interpolates_grid_points():
    g = _interpolation_fixture()
    inner = [(1.0, 1.0), (2.0, 1.0), (1.0, 2.0), (2.0, 2.0)]
    for p in inner:
        _set(g, p[0], p[1], 0.1, 1.0)
    for x in range(4):
        _set(g, float(x), 0.0, 0.1, 1.0)
        _set(g, float(x), 3.0, 0.1, 1.0)
    for y in range(1, 3):
        _set(g, 0.0, float(y), 0.1, 1.0)
        _set(g, 3.0, float(y), 0.1, 1.0)
    for p in inner:
        ix, iy = g.cell_index(p[0], p[1])
        w, _, cost, _ = T.interpolate(g, p[0], p[1])
        assert abs(float(g.get_correspondence_cost(ix, iy)) - cost[0]) < 1e-4
        assert abs(float(g.get_weight(ix, iy)) - w[0]) < 1e-4
    # unknown cell
    w, _, cost, _ = T.interpolate(g, 3.0, 2.0)
    assert abs(float(g.conv.max_tsd) - cost[0]) < 1e-4
    ix, iy = g.cell_index(3.0, 2.0)
    assert abs(float(g.get_weight(ix, iy)) - w[0]) < 1e-4


def test_interpolates_within_cell():
    g = _interpolation_fixture()
    tsd = {(0, 0): 0.1, (0, 1): 0.2, (1, 0): 0.3, (1, 1): 0.4}
    wgt = {(0, 0): 1.0, (0, 1): 2.0, (1, 0): 3.0, (1, 1): 4.0}
    for (x, y), v in tsd.items():
        _set(g, float(x), float(y), v, wgt[(x, y)])
    step = g.resolution / 100.0
    x = 0.0 + step
    while x < 1.0:
        y = 0.0 + step
        while y < 1.0:
            want_c = (x * 0.3 + (1 - x) * 0.1) * (1 - y) + (x * 0.4 + (1 - x) * 0.2) * y
            want_w = (x * 3.0 + (1 - x) * 1.0) * (1 - y) + (x * 4.0 + (1 - x) * 2.0) * y
            w, _, cost, _ = T.interpolate(g, x, y)
            assert abs(cost[0] - want_c) < 1e-3
            assert abs(w[0] - want_w) < 1e-3
            y += g.resolution
        x += g.resolution


def test_set_cell_keeps_the_first_update():
    g = _interpolation_fixture()
    g.set_cell(2, 3, 0.5, 2.0)
    g.set_cell(2, 3, -0.5, 9.0)     # ignored until FinishUpdate
    assert g.tsd_cells[3, 2] >= T.UPDATE_MARKER
    g.finish_update()
    assert abs(float(g.get_correspondence_cost(2, 3)) - 0.5) < 1e-4
    assert abs(float(g.get_weight(2, 3)) - 2.0) < 1e-3
    assert float(g.get_weight(-1, 3)) == 0.0 and float(g.get_weight(2, 10)) == 0.0


def _world(seed=3, size_cells=200, beams=181, max_range=8.0):
    spec, occ = synthetic.make_tsdf2d(seed, size_cells=size_cells)
    rng = np.random.RandomState(seed)
    pose = synthetic.random_free_pose(occ, spec, rng, margin_cells=20)
    scan = synthetic.cast_scan(occ, spec, pose, beams=beams, max_range=max_range, seed=seed)
    return spec, T.TSDF2D.from_spec(spec), pose, scan


def test_match_empty_tsdf_is_invalid():
    g = T.TSDF2D(20, 20, 0.1, 1.0, 1.0, 0.3, 10.0)
    cloud = np.array([[0.1, 0.2, 0.0], [-0.3, 0.1, 0.0]], np.float32)
    _, _, valid = T.evaluate(g, cloud, [0.0, 0.0, 0.0], [0.0, 0.0], 0.0)
    assert not valid
    want = T.match(g, cloud, [0.0, 0.0], [0.05, -0.02, 0.1])
    assert want["termination"] == "EVALUATION_FAILED"
    assert np.array_equal(want["pose"], [0.05, -0.02, 0.1])
    assert want["iterations"] == 0


def test_tsdf_floorplan_is_a_signed_distance():
    spec, occ = synthetic.make_tsdf2d(5, size_cells=120)
    g = T.TSDF2D.from_spec(spec)
    iy, ix = np.nonzero(spec.weight_cells)
    cost = g.get_correspondence_cost(ix, iy)
    assert (cost[occ[iy, ix]] < 0).all() and (cost[~occ[iy, ix]] > 0).all()
    assert (np.abs(cost) <= spec.truncation_distance).all()
    assert (spec.tsd_cells[spec.weight_cells == 0] == 0).all()


def test_jacobian_matches_finite_differences():
    _, g, pose, scan = _world()
    x = pose + np.array([0.02, -0.015, 0.01])
    r, j, valid = T.evaluate(g, scan, x, x[:2], x[2])
    assert valid
    h = 1e-7
    fd = np.zeros_like(j)
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        rp, _, _ = T.evaluate(g, scan, x + e, x[:2], x[2], jacobian=False)
        rm, _, _ = T.evaluate(g, scan, x - e, x[:2], x[2], jacobian=False)
        fd[:, k] = (rp - rm) / (2 * h)
    # bilinear interpolation is piecewise: rows whose points cross a cell edge within +-h are
    # the only ones allowed to differ
    err = np.abs(fd - j).max(axis=1) / (1e-3 + np.abs(j).max(axis=1))
    assert (err < 1e-4).mean() > 0.97, np.sort(err)[-10:]
    assert np.abs(fd - j).sum() / np.abs(j).sum() < 1e-2


@pytest.mark.parametrize("nonmonotonic", [True, False])
def test_match_recovers_a_perturbed_pose(nonmonotonic):
    _, g, pose, scan = _world()
    init = pose + np.array([0.04, -0.03, 0.02])
    want = T.match(g, scan, init[:2], init, 1.0, 0.1, 0.1, nonmonotonic, 50)
    assert want["final_cost"] < 0.75 * want["initial_cost"]
    # the perturbation is 5 cm / 0.02 rad: the refinement must remove most of it
    assert np.hypot(*(want["pose"][:2] - pose[:2])) < 0.5 * np.hypot(0.04, 0.03), (want, pose)
    assert abs(want["pose"][2] - pose[2]) < 0.5 * 0.02


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "refine2d_tsdf_emulation.cc")
    csrc = os.path.join(HERE, "..", "..", "cartographer_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("refine2d.cu", "trust_region.cuh")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(map(os.path.getmtime, deps)):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                               "-pthread", "-w", "-x", "c++", src, "-o", SO])
    return C.CDLL(SO)


def _run(emu, g, xyz, target, init, opts):
    xyz = np.ascontiguousarray(xyz, np.float32)
    tsd = np.ascontiguousarray(g.tsd_cells, np.uint16)
    wgt = np.ascontiguousarray(g.weight_cells, np.uint16)
    gp = np.array([g.resolution, g.max_x, g.max_y, g.truncation_distance, g.max_weight])
    op, t = np.array(opts, np.float64), np.array(target, np.float64)
    ip, out = np.array(init, np.float64), np.zeros(8)

    def p(a, ty):
        return a.ctypes.data_as(C.POINTER(ty))
    emu.emu_ceres_match2d_tsdf(p(tsd, C.c_uint16), p(wgt, C.c_uint16), C.c_int(g.num_x),
                               C.c_int(g.num_y), p(gp, C.c_double), p(xyz, C.c_float),
                               C.c_int(len(xyz)), p(op, C.c_double), p(t, C.c_double),
                               p(ip, C.c_double), p(out, C.c_double))
    return out


def _check(out, want):
    assert np.allclose(out[:3], want["pose"], rtol=0, atol=1e-9), (out, want)
    assert out[3] == pytest.approx(want["initial_cost"], rel=1e-12)
    assert out[4] == pytest.approx(want["final_cost"], rel=1e-9)
    assert int(out[5]) == want["iterations"]
    assert int(out[6]) == want["num_successful_steps"]
    assert T.CERES_TERMINATION[int(out[7])] == want["termination"]


@pytest.mark.parametrize("nonmonotonic", [1, 0])
def test_emulated_tsdf_kernel_on_a_floorplan(emu, nonmonotonic):
    _, g, pose, scan = _world(beams=601)   # several strides of 256 threads, not a multiple of 32
    init = pose + np.array([0.04, -0.03, 0.02])
    opts = [20.0, 10.0, 1.0, nonmonotonic, 15]
    want = T.match(g, scan, init[:2], init, *opts[:3], bool(nonmonotonic), opts[4])
    _check(_run(emu, g, scan, init[:2], init, opts), want)


def test_emulated_tsdf_kernel_initial_failure(emu):
    _, g, pose, scan = _world()
    init = np.array([500.0, -500.0, 0.3])    # the whole scan far outside the grid: W == 0
    want = T.match(g, scan, init[:2], init)
    assert want["termination"] == "EVALUATION_FAILED"
    out = _run(emu, g, scan, init[:2], init, [20.0, 10.0, 1.0, 1, 10])
    _check(out, want)
    assert np.array_equal(out[:3], init)


def _island():
    """A 2 x 2-cell patch of weight in an otherwise unknown grid, and a one-point scan."""
    g = T.TSDF2D(12, 12, 0.1, 0.6, 0.6, 0.3, 10.0)
    # a shallow slope far from zero: the Gauss-Newton step overshoots the patch by metres
    vals = {(5, 5): 0.20, (6, 5): 0.22, (5, 6): 0.20, (6, 6): 0.22}
    for (ix, iy), tsd in vals.items():
        g.set_cell(ix, iy, tsd, 5.0)
    g.finish_update()
    return g, np.array([[0.0, 0.0, 0.0]], np.float32)


def test_emulated_tsdf_kernel_trial_step_failure(emu):
    """Weak priors and a steep cost: the first Gauss-Newton steps leave the patch of weight,
    the cost function fails there and the minimiser rejects those steps."""
    g, cloud = _island()
    found = None
    for dx in np.linspace(-0.04, 0.04, 9):
        init = np.array([0.0 + dx, 0.0 + 0.5 * dx, 0.0])
        want = T.match(g, cloud, init[:2], init, 20.0, 1e-3, 1e-3, True, 10)
        if want["trial_failures"] > 0:
            found = (init, want)
            break
    assert found is not None
    init, want = found
    _check(_run(emu, g, cloud, init[:2], init, [20.0, 1e-3, 1e-3, 1, 10]), want)
