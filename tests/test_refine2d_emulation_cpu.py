"""CPU check of the refinement KERNEL's control flow (no GPU in the development container).

tests/emulation/refine2d_emulation.cc includes the device code of
cartographer_b200/csrc/refine2d.cu verbatim and runs one CTA of k_ceres_match2d with one
std::thread per CUDA thread (barriers for __syncthreads and the warp shuffles).  What it can
show: uniform control flow around the barriers, the shared-memory hand-offs, the minimiser's
state machine — against the oracle.  It is test infrastructure, not a fallback: the product
library has no CPU path, and the real parity tests are tests/test_gpu_ceres2d.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.test_oracle_golden_ceres2d import _ceres_test_fixture, smooth_grid

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emulation")
SO = os.path.join(HERE, "_build", "librefine2d_emulation.so")


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "refine2d_emulation.cc")
    csrc = os.path.join(HERE, "..", "..", "cartographer_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("refine2d.cu", "trust_region.cuh",
                                                       "value_conversion.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(map(os.path.getmtime, deps)):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                               "-pthread", "-w", "-x", "c++", src, "-o", SO])
    return C.CDLL(SO)


def _run(emu, grid, xyz, target, init, opts):
    xyz = np.ascontiguousarray(xyz, np.float32)
    cells = np.ascontiguousarray(grid.cells, np.uint16)
    op, t = np.array(opts, np.float64), np.array(target, np.float64)
    ip, out = np.array(init, np.float64), np.zeros(8)

    def p(a, ty):
        return a.ctypes.data_as(C.POINTER(ty))
    emu.emu_ceres_match2d(p(cells, C.c_uint16), C.c_int(grid.num_x), C.c_int(grid.num_y),
                          C.c_double(grid.resolution), C.c_double(grid.max_x),
                          C.c_double(grid.max_y), p(xyz, C.c_float), C.c_int(len(xyz)),
                          p(op, C.c_double), p(t, C.c_double), p(ip, C.c_double),
                          p(out, C.c_double))
    return out


def _check(oracle, out, want):
    assert np.allclose(out[:3], want["pose"], rtol=0, atol=1e-9)
    assert out[3] == pytest.approx(want["initial_cost"], rel=1e-12)
    assert out[4] == pytest.approx(want["final_cost"], rel=1e-9)
    assert int(out[5]) == want["iterations"]
    assert int(out[6]) == want["num_successful_steps"]
    assert oracle.CERES_TERMINATION[int(out[7])] == want["termination"]


@pytest.mark.parametrize("start", [(-0.5, 0.5), (-0.45, 0.3)])
def test_emulated_kernel_on_the_reference_fixture(oracle, emu, start):
    grid, cloud, opts = _ceres_test_fixture(oracle)
    init = [start[0], start[1], 0.0]
    out = _run(emu, grid, cloud, init[:2], init, [1.0, 0.1, 1.5, 1, 50])
    _check(oracle, out, oracle.ceres2d_match(grid, cloud, init[:2], init, **opts))


@pytest.mark.parametrize("nonmonotonic", [1, 0])
def test_emulated_kernel_on_a_smooth_field(oracle, emu, nonmonotonic):
    rng = np.random.RandomState(8)
    grid = smooth_grid(oracle)
    # more points than threads (several strides) and a count that is not a multiple of 32
    ang = rng.uniform(0, 2 * np.pi, 601)
    rad = rng.uniform(0.02, 0.3, 601)
    cloud = np.stack([rad * np.cos(ang), rad * np.sin(ang), np.zeros(601)], 1).astype(np.float32)
    init = np.array([0.525 + 0.05, -0.125 - 0.04, 0.3])
    out = _run(emu, grid, cloud, init[:2], init, [20.0, 10.0, 1.0, nonmonotonic, 15])
    _check(oracle, out, oracle.ceres2d_match(grid, cloud, init[:2], init, 20.0, 10.0, 1.0,
                                             bool(nonmonotonic), 15))


@pytest.mark.parametrize("prior_weight,termination", [(1e3, "FUNCTION_TOLERANCE"),
                                                      (1e5, "PARAMETER_TOLERANCE")])
def test_emulated_kernel_tolerance_exits(oracle, emu, prior_weight, termination):
    """Stiff priors make the first trial step tiny: the function / parameter tolerance exits
    (which stop BEFORE taking the step) are reached in the kernel as in the oracle."""
    rng = np.random.RandomState(8)
    grid = smooth_grid(oracle)
    ang = rng.uniform(0, 2 * np.pi, 200)
    rad = rng.uniform(0.02, 0.3, 200)
    cloud = np.stack([rad * np.cos(ang), rad * np.sin(ang), np.zeros(200)], 1).astype(np.float32)
    init = np.array([0.525 + 0.05, -0.125 - 0.04, 0.3])
    want = oracle.ceres2d_match(grid, cloud, init[:2], init, 20.0, prior_weight, prior_weight,
                                True, 50)
    assert want["termination"] == termination
    out = _run(emu, grid, cloud, init[:2], init, [20.0, prior_weight, prior_weight, 1, 50])
    _check(oracle, out, want)
