"""CPU check of the 3D refinement KERNEL's control flow (see test_refine2d_emulation_cpu.py):
the device code of cartographer_b200/csrc/refine3d.cu runs in tests/emulation's SIMT harness
and is compared with the oracle.  Test infrastructure, not a fallback."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from tests.test_oracle_golden_ceres3d import POINTS

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emulation")
SO = os.path.join(HERE, "_build", "librefine3d_emulation.so")


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "refine3d_emulation.cc")
    csrc = os.path.join(HERE, "..", "..", "cartographer_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("refine3d.cu", "trust_region.cuh",
                                                       "value_conversion.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(map(os.path.getmtime, deps)):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                               "-pthread", "-w", "-x", "c++", src, "-o", SO])
    return C.CDLL(SO)


def dense_box(indices, values):
    """The dense volume csm_grid3d_create builds: values[z, y, x] from the lowest index."""
    idx = np.asarray(indices, np.int32)
    lo, hi = idx.min(0), idx.max(0)
    n = hi - lo + 1
    vol = np.zeros((n[2], n[1], n[0]), np.uint16)
    for (x, y, z), v in zip(idx - lo, values):
        vol[z, y, x] = v
    return np.ascontiguousarray(vol), lo.astype(np.int32), n.astype(np.int32)


def hybrid(oracle, resolution, points):
    idx = np.array([oracle.hybrid_get_cell_index(resolution, p) for p in points], np.int32)
    val = np.full(len(idx), oracle.probability_to_value(1.0), np.uint16)
    return (resolution, idx, val), oracle.HybridGrid(resolution, idx, val)


def run_emulation(emu, pairs, target_t, init, opts):
    num = len(pairs)
    vols, los, ns, res, xs, npts = [], [], [], [], [], []
    for xyz, (r, idx, val) in pairs:
        v, lo, n = dense_box(idx, val)
        vols.append(v)
        los += list(lo)
        ns += list(n)
        res.append(r)
        xs.append(np.ascontiguousarray(xyz, np.float32))
        npts.append(len(xyz))

    def p(a, ty):
        return a.ctypes.data_as(C.POINTER(ty))
    volp = (C.POINTER(C.c_uint16) * num)(*[p(v, C.c_uint16) for v in vols])
    xp = (C.POINTER(C.c_float) * num)(*[p(x, C.c_float) for x in xs])
    lo, n = np.array(los, np.int32), np.array(ns, np.int32)
    rs, npt = np.array(res, np.float32), np.array(npts, np.int32)
    op, tt = np.array(opts, np.float64), np.array(target_t, np.float64)
    ip, out = np.array(init, np.float64), np.zeros(12)
    emu.emu_ceres_match3d(C.c_int(num), volp, p(lo, C.c_int32), p(n, C.c_int32), p(rs, C.c_float),
                          xp, p(npt, C.c_int32), p(op, C.c_double), p(tt, C.c_double),
                          p(ip, C.c_double), p(out, C.c_double))
    return out


def _check(oracle, out, want):
    assert np.allclose(out[:7], want["pose"], rtol=0, atol=1e-9)
    assert out[7] == pytest.approx(want["initial_cost"], rel=1e-12, abs=1e-15)
    assert out[8] == pytest.approx(want["final_cost"], rel=1e-9, abs=1e-15)
    assert int(out[9]) == want["iterations"]
    assert int(out[10]) == want["num_successful_steps"]
    assert oracle.CERES_TERMINATION[int(out[11])] == want["termination"]


@pytest.mark.parametrize("start", [(-1.0, 0.0, 0.0), (-0.9, -0.2, 0.2)])
def test_emulated_kernel_on_the_reference_fixture(oracle, emu, start):
    spec, grid = hybrid(oracle, 1.0, POINTS + np.array([-1, 0, 0], np.float32))
    init = [start[0], start[1], start[2], 1.0, 0.0, 0.0, 0.0]
    out = run_emulation(emu, [(POINTS, spec)], init[:3], init, [0.01, 0.1, 1, 10, 1.0, 1.0])
    _check(oracle, out, oracle.ceres3d_match(
        [(POINTS, grid)], init[:3], init, occupied_space_weights=[1.0], translation_weight=0.01,
        rotation_weight=0.1, use_nonmonotonic_steps=True, max_num_iterations=10))


@pytest.mark.parametrize("nonmonotonic", [1, 0])
def test_emulated_kernel_two_clouds_with_rotation(oracle, emu, nonmonotonic):
    """High- and low-resolution pairs, more points than threads, a rotated start."""
    spec, grid = hybrid(oracle, 1.0, POINTS + np.array([-1, 0, 0], np.float32))
    spec2, grid2 = hybrid(oracle, 2.0, POINTS + np.array([-1, 0, 0], np.float32))
    rng = np.random.RandomState(1)
    cloud = (POINTS[rng.randint(0, 7, 300)] + rng.uniform(-0.3, 0.3, (300, 3))).astype(np.float32)
    a = 0.05
    init = [-0.95, -0.05, 0.05, math.cos(a / 2), math.sin(a / 2), 0.0, 0.0]
    out = run_emulation(emu, [(cloud, spec), (POINTS, spec2)], init[:3], init,
                        [10.0, 1.0, nonmonotonic, 12, 5.0, 30.0])
    _check(oracle, out, oracle.ceres3d_match(
        [(cloud, grid), (POINTS, grid2)], init[:3], init, occupied_space_weights=[5.0, 30.0],
        translation_weight=10.0, rotation_weight=1.0,
        use_nonmonotonic_steps=bool(nonmonotonic), max_num_iterations=12))


def test_emulated_evaluate_kernel_rows(oracle, emu):
    """k_ceres_evaluate3d (the GPU tests' residual / Jacobian hook): row indexing over two
    clouds and the six prior rows, against the oracle — values must be identical."""
    spec, grid = hybrid(oracle, 1.0, POINTS + np.array([-1, 0, 0], np.float32))
    spec2, grid2 = hybrid(oracle, 2.0, POINTS + np.array([-1, 0, 0], np.float32))
    rng = np.random.RandomState(3)
    cloud = (POINTS[rng.randint(0, 7, 270)] + rng.uniform(-0.4, 0.4, (270, 3))).astype(np.float32)
    a = 0.07
    q = np.array([math.cos(a), math.sin(a) * 0.2, -math.sin(a) * 0.3, math.sin(a) * 0.933])
    pose = np.concatenate([[-0.95, 0.04, 0.06], q / np.linalg.norm(q)])
    tq = np.array([math.cos(0.02), 0.0, 0.0, math.sin(0.02)])
    pairs = [(cloud, spec), (POINTS, spec2)]
    num = 2
    vols, los, ns, res, xs, npts = [], [], [], [], [], []
    for xyz, (r, idx, val) in pairs:
        v, lo, n = dense_box(idx, val)
        vols.append(v)
        los += list(lo)
        ns += list(n)
        res.append(r)
        xs.append(np.ascontiguousarray(xyz, np.float32))
        npts.append(len(xyz))

    def p(arr, ty):
        return arr.ctypes.data_as(C.POINTER(ty))
    volp = (C.POINTER(C.c_uint16) * num)(*[p(v, C.c_uint16) for v in vols])
    xp = (C.POINTER(C.c_float) * num)(*[p(x, C.c_float) for x in xs])
    lo, n = np.array(los, np.int32), np.array(ns, np.int32)
    rs, npt = np.array(res, np.float32), np.array(npts, np.int32)
    rows = sum(npts) + 6
    op = np.array([10.0, 1.0, 5.0, 30.0])
    tt = np.array([-1.0, 0.0, 0.0])
    for with_jac in (1, 0):
        got_r, got_j = np.zeros(rows), np.zeros((rows, 6))
        emu.emu_ceres_evaluate3d(C.c_int(num), volp, p(lo, C.c_int32), p(n, C.c_int32),
                                 p(rs, C.c_float), xp, p(npt, C.c_int32), p(op, C.c_double),
                                 p(tt, C.c_double), p(tq, C.c_double), p(pose, C.c_double),
                                 C.c_int(with_jac), p(got_r, C.c_double), p(got_j, C.c_double))
        want_r, want_j = oracle.ceres3d_evaluate([(cloud, grid), (POINTS, grid2)], pose, tt, tq,
                                                 jacobian=bool(with_jac))
        assert np.array_equal(got_r, want_r)
        if with_jac:
            assert np.array_equal(got_j, want_j)


@pytest.mark.parametrize("prior_weight,termination", [(1e2, "FUNCTION_TOLERANCE"),
                                                      (1e4, "PARAMETER_TOLERANCE"),
                                                      (1e6, "PARAMETER_TOLERANCE")])
def test_emulated_kernel_tolerance_exits(oracle, emu, prior_weight, termination):
    """Stiff priors: the tolerance exits (before the step is taken) in the kernel as in the
    oracle, including a successful step followed by a parameter-tolerance stop."""
    spec, grid = hybrid(oracle, 1.0, POINTS + np.array([-1, 0, 0], np.float32))
    init = [-0.9, -0.2, 0.2, 1.0, 0.0, 0.0, 0.0]
    want = oracle.ceres3d_match([(POINTS, grid)], init[:3], init, occupied_space_weights=[1.0],
                                translation_weight=prior_weight, rotation_weight=prior_weight,
                                use_nonmonotonic_steps=False, max_num_iterations=30)
    assert want["termination"] == termination
    out = run_emulation(emu, [(POINTS, spec)], init[:3], init,
                        [prior_weight, prior_weight, 0, 30, 1.0, 1.0])
    _check(oracle, out, want)
