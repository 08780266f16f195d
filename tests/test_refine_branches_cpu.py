"""The trust-region minimiser branch by branch, and the per-point edges, without a GPU.

On the case tables of tests/refine_cases.py, which tests/test_gpu_refine_kernels.py runs on the
device:
  * the traced oracles reach every branch a case names, every deciding quantity 1e-6 away
    from its threshold, and the margin check refuses a solve that rounding decides;
  * the device code of trust_region.cuh, refine2d.cu and refine3d.cu, run by the four SIMT
    harnesses of tests/emulation, gives the oracle's counts, termination and pose on those
    cases — rejections with a doubling decrease factor, rising accepted costs, the
    reference-cost switch, the lowest-cost iterate returned when it is not the last;
  * the emulated kernels on the per-point edges: a row pitch that differs from nx, unknown /
    saturated / update-marked cells in ProbabilityGrid, tsd and weight cells, scan points
    exactly on TSDF cell centres, 3D points with p / res at the halves.
Test infrastructure, not a fallback: the library has no CPU path."""
import ctypes as C

import numpy as np
import pytest

from tests import intensity3d_oracle as iorc
from tests import refine_cases as RC
from tests import tsdf2d_oracle as T
from tests.test_refine2d_emulation_cpu import _check as check2d
from tests.test_refine2d_emulation_cpu import _run as run2d
from tests.test_refine2d_emulation_cpu import emu as emu2d            # noqa: F401 (fixture)
from tests.test_refine3d_emulation_cpu import _check as check3d
from tests.test_refine3d_emulation_cpu import dense_box
from tests.test_refine3d_emulation_cpu import emu as emu3d            # noqa: F401 (fixture)
from tests.test_refine3d_emulation_cpu import run_emulation as run3d
from tests.test_refine3d_intensity_emulation_cpu import emu as emu_intensity   # noqa: F401
from tests.test_refine3d_intensity_emulation_cpu import run_match as run_intensity
from tests.test_tsdf2d_oracle_cpu import _check as check_tsdf
from tests.test_tsdf2d_oracle_cpu import _run as run_tsdf
from tests.test_tsdf2d_oracle_cpu import emu as emu_tsdf              # noqa: F401 (fixture)

F = np.float32


def _p(a, ty):
    return a.ctypes.data_as(C.POINTER(ty))


def _opts2d(o):
    return [o["occupied_space_weight"], o["translation_weight"], o["rotation_weight"],
            int(o["use_nonmonotonic_steps"]), o["max_num_iterations"]]


def pitched(cells, pitch, fill):
    """cells in rows of `pitch`, the padding holding `fill` (a value no cell should read)."""
    out = np.full((cells.shape[0], pitch), fill, np.uint16)
    out[:, :cells.shape[1]] = cells
    return np.ascontiguousarray(out)


# ---- the minimiser's branches -------------------------------------------------------------------
@pytest.mark.parametrize("name,seed,opts,branches", RC.SOLVES_2D, ids=[c[0] for c in RC.SOLVES_2D])
def test_2d_cases_reach_their_branches_and_the_emulated_kernel_follows(oracle, emu2d, name, seed,
                                                                       opts, branches):
    cells, res, mx, my, cloud, tgt, init = RC.problem2d(seed)
    grid = oracle.Grid2D(cells, res, mx, my)
    want = oracle.ceres2d_match(grid, cloud, tgt, init, trace=True, **opts)
    RC.assert_reaches(want, branches)
    plain = oracle.ceres2d_match(grid, cloud, tgt, init, **opts)      # the trace changes nothing
    assert np.array_equal(plain["pose"], want["pose"])
    assert {k: v for k, v in want.items() if k not in ("pose", "trace")} == \
        {k: v for k, v in plain.items() if k != "pose"}
    check2d(oracle, run2d(emu2d, grid, cloud, tgt, init, _opts2d(opts)), want)


def test_the_case_tables_cover_every_branch_in_every_instantiation():
    """Each branch of the minimiser's state machine is named by a case of each of the four
    tables (the trial failure is TSDF only and has its own test)."""
    shared = {"rejected", "two_rejections", "three_rejections", "accepted_rising",
              "reference_switch", "best_not_last", "max_iterations", "function_tolerance"}
    assert shared <= {b for c in RC.SOLVES_2D for b in c[3]}
    assert shared <= {b for c in RC.SOLVES_TSDF for b in c[5]}
    assert shared <= {b for c in RC.SOLVES_3D for b in c[5]}
    assert shared | {"parameter_tolerance"} <= {b for c in RC.SOLVES_INTENSITY for b in c[7]}


def test_a_solve_decided_by_rounding_is_refused_by_the_margin_check():
    """The TSDF solve that falls into an exact 2-cycle: its cost comparison in the step
    evaluator is closer than the margin, so it may not serve as a parity case."""
    _, _, want = RC.tsdf_want(RC.TSDF_DECIDED_BY_ROUNDING)
    closest = min(abs(t["candidate_cost"] - t["evaluator_minimum_cost"]) /
                  t["evaluator_minimum_cost"] for t in want["trace"] if t["outcome"] == "ACCEPTED")
    assert closest < 1e-12
    assert any(t["step_quality"] == 0.0 for t in want["trace"])      # cost == reference cost
    with pytest.raises(AssertionError):
        RC.assert_margins(want)


def test_2d_gradient_tolerance_before_the_first_step(oracle, emu2d):
    cells, res, mx, my, _, _, _ = RC.problem2d(1)
    grid = oracle.Grid2D(cells, res, mx, my)
    init = np.array([0.3, -0.2, 0.1])
    for n in (1, 257):
        cloud = RC.far_cloud2d(n)
        want = oracle.ceres2d_match(grid, cloud, init[:2], init, trace=True)
        RC.assert_reaches(want, ["gradient_at_start"])
        out = run2d(emu2d, grid, cloud, init[:2], init, [20.0, 10.0, 1.0, 1, 10])
        check2d(oracle, out, want)
        assert np.array_equal(out[:3], init)


@pytest.mark.parametrize("case", RC.SOLVES_TSDF, ids=[c[0] for c in RC.SOLVES_TSDF])
def test_tsdf_cases_reach_their_branches_and_the_emulated_kernel_follows(emu_tsdf, case):
    g, p, want = RC.tsdf_want(case)
    RC.assert_reaches(want, case[5])
    plain = T.match(g, p[7], p[8], p[9], 20.0, 1e-2, 1e-2, case[3], case[4])
    assert np.array_equal(plain["pose"], want["pose"]) and plain["iterations"] == want["iterations"]
    check_tsdf(run_tsdf(emu_tsdf, g, p[7], p[8], p[9], [20.0, 1e-2, 1e-2, int(case[3]), case[4]]),
               want)


@pytest.mark.parametrize("case", RC.SOLVES_3D, ids=[c[0] for c in RC.SOLVES_3D])
def test_3d_cases_reach_their_branches_and_the_emulated_kernel_follows(oracle, emu3d, case):
    (res, idx, val, hi, low, tgt, init), want = RC.want3d(oracle, case)
    RC.assert_reaches(want, case[5])
    spec = (res, idx, val)
    pairs = [(hi, spec)] + ([(low, spec)] if low is not None else [])
    out = run3d(emu3d, pairs, tgt, init,
                [RC.WEAK_PRIOR_3D["translation_weight"], RC.WEAK_PRIOR_3D["rotation_weight"],
                 int(case[3]), case[4], 5.0, 30.0])
    check3d(oracle, out, want)


@pytest.mark.parametrize("case", RC.SOLVES_INTENSITY, ids=[c[0] for c in RC.SOLVES_INTENSITY])
def test_intensity_cases_reach_their_branches_and_the_emulated_kernel_follows(oracle, emu_intensity,
                                                                              case):
    name, seed, weight, huber, prior, nonmono, iters, branches = case
    (res, idx, val, hi, tgt, init, sums, counts, inten), want = RC.want_intensity(oracle, case)
    RC.assert_reaches(want, branches)
    out = run_intensity(emu_intensity, [(hi, (res, idx, val), (res, idx, sums, counts), inten)],
                        tgt, init, [prior, prior, int(nonmono), iters, 5.0, 30.0],
                        [weight, huber, RC.INTENSITY_THRESHOLD])
    check3d(oracle, out, want)


# ---- the per-point edges in the emulated kernels ----------------------------------------------
def test_2d_marker_cells_border_patches_and_row_pitch_in_the_emulated_kernel(oracle, emu2d):
    """A solve on a grid with unknown, saturated and update-marked cells whose scan overlaps
    the border, the cells in rows of 16 for nx = 11: PaddedValue's mask, bounds and
    iy * pitch inside the solver kernel."""
    rng = np.random.RandomState(21)
    cells = RC.edge_cells(rng, 14, 11)
    grid = oracle.Grid2D(cells, 0.05, 0.35, 0.275)
    assert (cells >= 32768).sum() > 10 and (cells == 0).sum() > 5
    cloud = np.concatenate([rng.uniform(-0.45, 0.45, (257, 2)), np.zeros((257, 1))], 1).astype(F)
    outside = (np.abs(cloud[:, 0]) > 0.35) | (np.abs(cloud[:, 1]) > 0.275)
    assert 10 < outside.sum() < 200
    init = np.array([0.05, -0.04, 0.2])
    opts = dict(RC.WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=15)
    want = oracle.ceres2d_match(grid, cloud, init[:2], init, trace=True, **opts)
    RC.assert_margins(want)
    assert want["iterations"] >= 3
    check2d(oracle, run2d(emu2d, grid, cloud, init[:2], init, _opts2d(opts)), want)
    rows = pitched(cells, 16, 20000)
    op, t, ip, out = np.array(_opts2d(opts), np.float64), init[:2].copy(), init.copy(), np.zeros(8)
    emu2d.emu_ceres_match2d_pitched(
        _p(rows, C.c_uint16), C.c_int(11), C.c_int(14), C.c_int(16), C.c_double(0.05),
        C.c_double(0.35), C.c_double(0.275), _p(cloud, C.c_float), C.c_int(len(cloud)),
        _p(op, C.c_double), _p(t, C.c_double), _p(ip, C.c_double), _p(out, C.c_double))
    check2d(oracle, out, want)


def test_tsdf_markers_cell_centres_and_row_pitch_in_the_emulated_kernel(emu_tsdf):
    """Scan points exactly on cell centres at the initial pose (cos 0 and sin 0 are exact), tsd
    and weight cells with unknown, saturated and update-marked values, rows of 16 for nx = 9:
    TsdfCornersAt's `lx > x`, the masks of TsdfWeight / TsdfCost and iy * pitch."""
    rng = np.random.RandomState(33)
    ny, nx, res, max_x, max_y = 12, 9, 0.05, 0.3, 0.2
    tsd, wgt = RC.edge_cells(rng, ny, nx), RC.edge_cells(rng, ny, nx)
    g = T.TSDF2D(nx, ny, res, max_x, max_y, 0.3, 10.0, tsd, wgt)
    iy, ix = np.meshgrid(np.arange(ny), np.arange(nx), indexing="ij")
    cx, cy = g.cell_center(ix.ravel(), iy.ravel())
    cloud = np.stack([cx, cy, np.zeros(len(cx), F)], 1).astype(F)
    init = np.zeros(3)
    # reached: every point sits on its cell's centre, so `lx > x` is false and `lx >= x` true
    lx, ly, _, _, _, _ = T._corners(g, cloud[:, 0].astype(np.float64), cloud[:, 1].astype(np.float64))
    assert np.array_equal(lx, cx) and np.array_equal(ly, cy) and len(cloud) == 108
    assert ((tsd >= 32768) & (wgt != 0) & (wgt != 32768)).sum() > 5 and (wgt >= 32768).sum() > 5
    opts = [20.0, 1e-2, 1e-2, 1, 6]
    trace = []
    want = T.match(g, cloud, init[:2], init, *opts[:3], True, 6, trace=trace)
    want["trace"] = trace
    RC.assert_margins(want)
    assert want["termination"] != "EVALUATION_FAILED" and want["iterations"] >= 2
    check_tsdf(run_tsdf(emu_tsdf, g, cloud, init[:2], init, opts), want)
    gp = np.array([res, max_x, max_y, g.truncation_distance, g.max_weight])
    op, t, ip, out = np.array(opts, np.float64), np.zeros(2), np.zeros(3), np.zeros(8)
    emu_tsdf.emu_ceres_match2d_tsdf_pitched(
        _p(pitched(tsd, 16, 20000), C.c_uint16), _p(pitched(wgt, 16, 20000), C.c_uint16),
        C.c_int(nx), C.c_int(ny), C.c_int(16), _p(gp, C.c_double), _p(cloud, C.c_float),
        C.c_int(len(cloud)), _p(op, C.c_double), _p(t, C.c_double), _p(ip, C.c_double),
        _p(out, C.c_double))
    check_tsdf(out, want)


def test_3d_rows_at_the_voxel_halves_in_the_emulated_kernel(oracle, emu3d):
    """k_ceres_evaluate3d at p / res = +-0.5, +-1.5, +-2.5 with their float neighbours and on
    the faces of the dense box: CellOf's lroundf and the i + 1, j + 1, k + 1 reads, bit for bit
    against the oracle."""
    res, idx, val, _, _, _, _ = RC.problem3d(2, size=4)       # voxels -2 .. 1
    grid = oracle.HybridGrid(res, idx, val)
    r32 = F(res)
    half = np.array([(k + 0.5) * r32 for k in (-3, -2, -1, 0, 1, 2)], F)
    a = np.concatenate([half, np.nextafter(half, F(-9)), np.nextafter(half, F(9)),
                        np.array([-2, -1, 0, 1], F) * r32])
    gx, gy, gz = np.meshgrid(a, a, a, indexing="ij")
    cloud = np.stack([gx.ravel(), gy.ravel(), gz.ravel()], 1).astype(F)
    q = (cloud[:, 0] / r32).astype(np.float64)
    assert (np.abs(q - np.trunc(q)) == 0.5).sum() >= 1000
    c = iorc.cell_index(r32, cloud)
    assert (c.min(0) == -3).all() and (c.max(0) == 3).all()    # outside every face of the box
    vol, lo, n = dense_box(idx, val)
    volp = (C.POINTER(C.c_uint16) * 1)(_p(vol, C.c_uint16))
    xp = (C.POINTER(C.c_float) * 1)(_p(cloud, C.c_float))
    rs, npt = np.array([res], F), np.array([len(cloud)], np.int32)
    op, tt, tq = np.array([10.0, 1.0, 5.0, 30.0]), np.zeros(3), np.array([1.0, 0.0, 0.0, 0.0])
    for pose in (np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]),
                 np.array([0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0])):      # exact transforms
        for jac in (1, 0):
            got_r, got_j = np.zeros(len(cloud) + 6), np.zeros((len(cloud) + 6, 6))
            emu3d.emu_ceres_evaluate3d(C.c_int(1), volp, _p(lo, C.c_int32), _p(n, C.c_int32),
                                       _p(rs, C.c_float), xp, _p(npt, C.c_int32),
                                       _p(op, C.c_double), _p(tt, C.c_double), _p(tq, C.c_double),
                                       _p(pose, C.c_double), C.c_int(jac), _p(got_r, C.c_double),
                                       _p(got_j, C.c_double))
            want_r, want_j = oracle.ceres3d_evaluate([(cloud, grid)], pose, tt, tq,
                                                     jacobian=bool(jac))
            assert np.array_equal(got_r, want_r)
            if jac:
                assert np.array_equal(got_j, want_j)
