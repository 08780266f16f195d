"""CPU check of the 3D refinement kernel's intensity path: the device code of
cartographer_b200/csrc/refine3d.cu runs in tests/emulation's SIMT harness with jobs that carry
IntensityCostFunction3D blocks under HuberLoss, and is compared with the intensity restatement
(tests/intensity3d_oracle.py).  Test infrastructure, not a fallback."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from tests import intensity3d_oracle as iorc
from tests.test_oracle_golden_ceres3d import POINTS
from tests.test_oracle_intensity3d_cpu import FIXTURE_INTENSITY, fixture, hybrid, intensity_grid
from tests.test_refine3d_emulation_cpu import _check, dense_box

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emulation")
SO = os.path.join(HERE, "_build", "librefine3d_intensity_emulation.so")


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "refine3d_intensity_emulation.cc")
    csrc = os.path.join(HERE, "..", "..", "cartographer_b200", "csrc")
    deps = [src, os.path.join(HERE, "refine3d_emulation.cc")] + \
        [os.path.join(csrc, f) for f in ("refine3d.cu", "trust_region.cuh", "value_conversion.h")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(map(os.path.getmtime, deps)):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                               "-pthread", "-w", "-x", "c++", src, "-o", SO])
    return C.CDLL(SO)


def intensity_box(spec):
    """The dense float volume csm_intensity_grid3d_create builds: GetIntensity per voxel."""
    r, idx, sums, counts = spec
    vals = np.where(counts == 0, np.float32(0),
                    sums / np.maximum(counts, 1).astype(np.float32)).astype(np.float32)
    idx = np.asarray(idx, np.int32).reshape(-1, 3)
    lo = idx.min(0)
    n = idx.max(0) - lo + 1
    vol = np.zeros((n[2], n[1], n[0]), np.float32)
    for (x, y, z), v in zip(idx - lo, vals):
        vol[z, y, x] = v
    return np.ascontiguousarray(vol), lo.astype(np.int32), n.astype(np.int32)


def _p(a, ty):
    return a.ctypes.data_as(C.POINTER(ty))


def _args(entries):
    """entries = [(xyz, hybrid spec, intensity spec or None, intensities or None)]"""
    num = len(entries)
    keep, los, ns, res, npts = [], [], [], [], []
    ilos, ins, ires = [], [], []
    volp = (C.POINTER(C.c_uint16) * num)()
    xp = (C.POINTER(C.c_float) * num)()
    ivp = (C.POINTER(C.c_float) * num)()
    ip = (C.POINTER(C.c_float) * num)()
    for b, (xyz, (r, idx, val), ispec, inten) in enumerate(entries):
        v, lo, n = dense_box(idx, val)
        x = np.ascontiguousarray(xyz, np.float32)
        keep += [v, x]
        volp[b], xp[b] = _p(v, C.c_uint16), _p(x, C.c_float)
        los += list(lo)
        ns += list(n)
        res.append(r)
        npts.append(len(x))
        if ispec is None:
            ilos += [0, 0, 0]
            ins += [0, 0, 0]
            ires.append(0.0)
            continue
        iv, ilo, inn = intensity_box(ispec)
        iv_i = np.ascontiguousarray(inten, np.float32)
        keep += [iv, iv_i]
        ivp[b], ip[b] = _p(iv, C.c_float), _p(iv_i, C.c_float)
        ilos += list(ilo)
        ins += list(inn)
        ires.append(ispec[0])
    arrs = [np.array(los, np.int32), np.array(ns, np.int32), np.array(res, np.float32),
            np.array(npts, np.int32), np.array(ilos, np.int32), np.array(ins, np.int32),
            np.array(ires, np.float32)]
    keep += arrs
    return num, volp, xp, ivp, ip, arrs, keep


def run_match(emu, entries, target_t, init, opts, iopts):
    num, volp, xp, ivp, ip, (lo, n, rs, npt, ilo, inn, ir), keep = _args(entries)
    op, io = np.array(opts, np.float64), np.array(iopts, np.float64).reshape(-1)
    tt, pi, out = np.array(target_t, np.float64), np.array(init, np.float64), np.zeros(12)
    emu.emu_ceres_match3d_intensity(
        C.c_int(num), volp, _p(lo, C.c_int32), _p(n, C.c_int32), _p(rs, C.c_float), xp,
        _p(npt, C.c_int32), _p(op, C.c_double), ivp, _p(ilo, C.c_int32), _p(inn, C.c_int32),
        _p(ir, C.c_float), ip, _p(io, C.c_double), _p(tt, C.c_double), _p(pi, C.c_double),
        _p(out, C.c_double))
    return out


def _oracle_entries(oracle, entries):
    out = []
    for xyz, (r, idx, val), ispec, inten in entries:
        g = oracle.HybridGrid(r, idx, val)
        ig = None if ispec is None else iorc.IntensityHybridGrid(*ispec)
        out.append((xyz, g, ig, inten))
    return out


@pytest.mark.parametrize("start,rotate", [((-0.8, 0.0, 0.0), 0.0), ((-0.9, -0.2, 0.2), 0.0),
                                          ((-0.95, -0.05, 0.05), 0.05)])
def test_emulated_kernel_on_the_reference_fixture(oracle, emu, start, rotate):
    cloud, intensities, hspec, _, ispec, _ = fixture(oracle, rotate)
    a = 0.05 if rotate else 0.0
    init = list(start) + [math.cos(a / 2), math.sin(a / 2), 0.0, 0.0]
    entries = [(cloud, hspec, ispec, intensities)]
    out = run_match(emu, entries, init[:3], init, [0.01, 0.1, 1, 10, 1.0, 1.0],
                    [FIXTURE_INTENSITY, (0, 0, 0)])
    _check(oracle, out, iorc.match(
        _oracle_entries(oracle, entries), init[:3], init, [FIXTURE_INTENSITY],
        occupied_space_weights=[1.0], translation_weight=0.01, rotation_weight=0.1,
        use_nonmonotonic_steps=True, max_num_iterations=10))


def _two_clouds(oracle, seed, intensity_on):
    """High- and low-resolution clouds, more points than threads; intensities 5..120 so some
    exceed the threshold of 100; intensity blocks on the clouds in `intensity_on`."""
    rng = np.random.RandomState(seed)
    shifted = POINTS + np.array([-1, 0, 0], np.float32)
    hspec, _ = hybrid(oracle, 1.0, shifted)
    lspec, _ = hybrid(oracle, 2.0, shifted)
    surf = (shifted[rng.randint(0, 7, 400)] + rng.uniform(-0.5, 0.5, (400, 3))).astype(np.float32)
    ispec, _ = intensity_grid(oracle, 1.0, surf, rng.uniform(10, 90, 400).astype(np.float32))
    cloud = (POINTS[rng.randint(0, 7, 300)] + rng.uniform(-0.3, 0.3, (300, 3))).astype(np.float32)
    inten = rng.uniform(5, 120, 300).astype(np.float32)
    low_inten = rng.uniform(5, 120, len(POINTS)).astype(np.float32)
    return [(cloud, hspec, ispec if 0 in intensity_on else None, inten),
            (POINTS, lspec, ispec if 1 in intensity_on else None, low_inten)]


@pytest.mark.parametrize("huber_scale,intensity_on,nonmonotonic",
                         [(0.3, (0,), 1), (55.0, (0,), 0), (0.3, (1,), 0), (2.0, (0, 1), 1)])
def test_emulated_kernel_two_clouds(oracle, emu, huber_scale, intensity_on, nonmonotonic):
    """Both Huber branches (0.3 is outlier-dominated, 55 keeps every block inside a^2),
    returns above the threshold, and an intensity block on either cloud or both."""
    entries = _two_clouds(oracle, 3, intensity_on)
    a = 0.05
    init = [-0.95, -0.05, 0.05, math.cos(a / 2), math.sin(a / 2), 0.0, 0.0]
    io = [(0.5, huber_scale, 100.0), (3.0, huber_scale, 100.0)]
    out = run_match(emu, entries, init[:3], init, [10.0, 1.0, nonmonotonic, 12, 5.0, 30.0], io)
    want = iorc.match(
        _oracle_entries(oracle, entries), init[:3], init, io, occupied_space_weights=[5.0, 30.0],
        translation_weight=10.0, rotation_weight=1.0, use_nonmonotonic_steps=bool(nonmonotonic),
        max_num_iterations=12)
    _check(oracle, out, want)
    # the Huber branch the case is meant to exercise is the one taken at the start
    r, _ = iorc.evaluate(_oracle_entries(oracle, entries), init, init[:3], init[3:], io,
                         occupied_space_weights=[5.0, 30.0], translation_weight=10.0,
                         jacobian=False)
    if intensity_on == (0,):
        n0 = len(entries[0][0])
        sb = float(np.sum(r[n0:2 * n0] ** 2))
        assert (sb > huber_scale ** 2) == (huber_scale == 0.3)


def test_emulated_evaluate_kernel_rows(oracle, emu):
    """k_ceres_evaluate3d's rows in the problem's block order, uncorrected, equal the oracle."""
    entries = _two_clouds(oracle, 4, (0, 1))
    num, volp, xp, ivp, ip, (lo, n, rs, npt, ilo, inn, ir), keep = _args(entries)
    q = np.array([math.cos(0.07), math.sin(0.07) * 0.2, -math.sin(0.07) * 0.3, 0.06])
    pose = np.concatenate([[-0.95, 0.04, 0.06], q / np.linalg.norm(q)])
    tq = np.array([math.cos(0.02), 0.0, 0.0, math.sin(0.02)])
    tt = np.array([-1.0, 0.0, 0.0])
    io = [(0.5, 0.3, 100.0), (3.0, 2.0, 60.0)]
    op, iop = np.array([10.0, 1.0, 5.0, 30.0]), np.array(io, np.float64).reshape(-1)
    rows = 2 * (len(entries[0][0]) + len(entries[1][0])) + 6
    for with_jac in (1, 0):
        got_r, got_j = np.zeros(rows), np.zeros((rows, 6))
        emu.emu_ceres_evaluate3d_intensity(
            C.c_int(num), volp, _p(lo, C.c_int32), _p(n, C.c_int32), _p(rs, C.c_float), xp,
            _p(npt, C.c_int32), _p(op, C.c_double), ivp, _p(ilo, C.c_int32), _p(inn, C.c_int32),
            _p(ir, C.c_float), ip, _p(iop, C.c_double), _p(tt, C.c_double), _p(tq, C.c_double),
            _p(pose, C.c_double), C.c_int(with_jac), _p(got_r, C.c_double),
            _p(got_j, C.c_double))
        want_r, want_j = iorc.evaluate(
            _oracle_entries(oracle, entries), pose, tt, tq, io, occupied_space_weights=[5.0, 30.0],
            translation_weight=10.0, rotation_weight=1.0, jacobian=bool(with_jac))
        assert np.array_equal(got_r, want_r)
        if with_jac:
            assert np.array_equal(got_j, want_j)
