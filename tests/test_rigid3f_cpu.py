"""The host side of cartographer_b200/csrc/rigid3f.h (Eigen's float quaternion and
rigid-transform arithmetic, shared by the host and the device code of the matchers) against the
oracle's restatement of the same arithmetic, bit for bit.

tests/rigid3f_check.cc evaluates every function of the header next to the oracle's function of
the same name; it is built with the oracle's flags.  The inputs include signed zeros, negative
half-angle sines, non-unit quaternions, the zero quaternion and angle-axis vectors on both sides
of the small-angle cutoff."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "rigid3f_check.cc")

_S = np.sin(-0.3)
SPECIAL_QUATERNIONS = [
    [1.0, 0.0, 0.0, 0.0], [-1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0],
    [-0.0, -0.0, -0.0, -0.0], [0.0, -0.0, 0.0, 1.0], [np.cos(-0.3), 0.0, -0.0, _S],
    [np.cos(-0.3), _S * 0.0, _S * 0.0, _S],  # Quaternionf(AngleAxisf(-0.6, UnitZ))
    [2.0, 0.5, -1.0, 3.0], [0.1, -0.2, 0.05, 0.01], [1e-20, 0.0, -1e-21, 0.0],
    [1e20, 3e19, -2e19, 1e19],
]
SPECIAL_VECTORS = [
    [0.0, 0.0, 0.0], [-0.0, -0.0, -0.0], [1.0, 0.0, 0.0], [-0.0, 2.5, -0.0],
    [1e-4, 0.0, 0.0], [0.0, 0.0, 1.0001e-4], [0.0, 0.0, -9.999e-5], [30.0, -12.0, 0.5],
]
SPECIAL_ANGLES = [0.0, -0.0, 1e-6, -1e-6, np.pi, -np.pi, -0.6, 2.0 * np.pi, -7.5]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rigid3f") / "librigid3f_check.so")
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-ffp-contract=off", "-fPIC", "-shared",
                           "-w", HARNESS, os.path.join(ROOT, "oracle", "oracle_3d.cc"), "-o", so])
    lib = C.CDLL(so)
    lib.rigid3f_compare.restype = C.c_int
    return lib


def _compare(lib, records, qd):
    records = np.ascontiguousarray(records, np.float32)
    qd = np.ascontiguousarray(qd, np.float64).reshape(-1, 4)
    assert records.shape[1] == 21
    msg = C.create_string_buffer(256)
    bad = lib.rigid3f_compare(records.ctypes.data_as(C.POINTER(C.c_float)), len(records),
                              qd.ctypes.data_as(C.POINTER(C.c_double)), len(qd), msg, len(msg))
    assert bad == 0, f"{bad} mismatches; first: {msg.value.decode()}"


def _special_records():
    """Every pair of special quaternions, with the special vectors and angles cycled through
    the point, the translations, the angle and the angle-axis vector."""
    q, v, a = SPECIAL_QUATERNIONS, SPECIAL_VECTORS, SPECIAL_ANGLES
    rows = []
    for i, qa in enumerate(q):
        for j, qb in enumerate(q):
            k = i * len(q) + j
            rows.append(qa + qb + v[k % len(v)] + v[(k + 1) % len(v)] + v[(k + 3) % len(v)] +
                        [a[k % len(a)]] + v[(k + 5) % len(v)])
    return np.array(rows, np.float64).astype(np.float32)


def _seeded_records(seed, n):
    rng = np.random.RandomState(seed)
    rec = rng.standard_normal((n, 21))
    rec[:, 0:8] *= rng.choice([1e-3, 1.0, 4.0], (n, 1))                 # non-unit quaternions
    unit = rng.rand(n) < 0.5
    for s in (slice(0, 4), slice(4, 8)):
        rec[unit, s] /= np.linalg.norm(rec[unit, s], axis=1, keepdims=True)
    rec[:, 8:17] *= rng.choice([1e-3, 1.0, 40.0], (n, 1))
    rec[:, 17] = rng.uniform(-2.0 * np.pi, 2.0 * np.pi, n)                 # negative sines too
    rec[:, 18:21] *= rng.choice([1e-5, 1e-4, 0.05, 1.0], (n, 1))          # around the cutoff
    # scattered signed zeros
    zero = rng.rand(n, 21) < 0.05
    rec[zero] = np.where(rng.rand(zero.sum()) < 0.5, 0.0, -0.0)
    return rec.astype(np.float32)


def _special_double_quaternions():
    return [[1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0], [-0.0, 0.0, -0.0, 0.0],
            [0.5, -0.5, 0.5, -0.5], [1e-200, 0.0, 0.0, 0.0], [2.0, -1.0, 0.25, 3.0],
            [np.cos(0.4), 0.0, 0.0, -np.sin(0.4)]]


def test_header_matches_oracle_on_special_inputs(harness):
    _compare(harness, _special_records(), _special_double_quaternions())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_header_matches_oracle_on_seeded_inputs(harness, seed):
    rng = np.random.RandomState(100 + seed)
    qd = rng.standard_normal((5000, 4)) * rng.choice([1e-3, 1.0, 1e3], (5000, 1))
    _compare(harness, _seeded_records(seed, 20000), qd)
