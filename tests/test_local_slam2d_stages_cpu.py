"""The host pieces under the device stages of 2D local SLAM, without a device: local_slam.py's
float32 Rigid3f arithmetic against csrc/rigid3f.h bit for bit, the builder's range_data_poses,
gravity transform and prediction against a float64 restatement, and the float32 per-point
restatement (tests/local_slam2d_oracle.py) against the float64 geometry of
tests/local_slam2d_chain.py."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from cartographer_b200 import local_slam as L
from tests import local_slam2d_chain as K
from tests import local_slam2d_oracle as O
from tests.test_rigid3f_cpu import _seeded_records, _special_records

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- local_slam.py's Rigid3f arithmetic against the header ----
@pytest.fixture(scope="module")
def header(tmp_path_factory):
    """rigid3f_eval.cc linked with rigid3f_check.cc and the oracle: the header's values, and
    the check that they equal the oracle's on the same records."""
    so = str(tmp_path_factory.mktemp("rigid3f_eval") / "librigid3f_eval.so")
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-ffp-contract=off", "-fPIC", "-shared",
                           "-w", os.path.join(ROOT, "tests", "rigid3f_eval.cc"),
                           os.path.join(ROOT, "tests", "rigid3f_check.cc"),
                           os.path.join(ROOT, "oracle", "oracle_3d.cc"), "-o", so])
    lib = C.CDLL(so)
    lib.rigid3f_compare.restype = C.c_int
    return lib


def _header_values(lib, records):
    records = np.ascontiguousarray(records, np.float32)
    msg = C.create_string_buffer(256)
    assert lib.rigid3f_compare(records.ctypes.data_as(C.POINTER(C.c_float)), len(records),
                               None, 0, msg, len(msg)) == 0, msg.value.decode()
    out = np.zeros_like(records)
    lib.rigid3f_eval(records.ctypes.data_as(C.c_void_p), len(records),
                     out.ctypes.data_as(C.c_void_p))
    return out


def _python_values(records):
    n = len(records)
    out = np.zeros((n, 21), np.float32)
    col = [records[:, k] for k in range(21)]
    ra = ((col[11], col[12], col[13]), (col[0], col[1], col[2], col[3]))
    with np.errstate(all="ignore"):
        out[:, 0:3] = np.stack(L.rigid3f_apply(ra, (col[8], col[9], col[10])), 1)
        inv = L.rigid3f_inverse(ra)
        out[:, 10:13] = np.stack(inv[0], 1)
        out[:, 13:17] = np.stack(inv[1], 1)
        for i, r in enumerate(records):
            a = ((r[11], r[12], r[13]), (r[0], r[1], r[2], r[3]))
            b = ((r[14], r[15], r[16]), (r[4], r[5], r[6], r[7]))
            t, q = L.rigid3f_mul(a, b)
            out[i, 3:10] = list(t) + list(q)
            out[i, 17:21] = L.embed3d_f((0.0, 0.0, r[17]))[1]
    return out


def _assert_bits_equal(got, want):
    """Bit for bit; a NaN equals any NaN (the payload is not part of the arithmetic)."""
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    bad = np.argwhere(~same)
    names = ["apply"] * 3 + ["mul"] * 7 + ["inverse"] * 7 + ["embed3d_f"] * 4
    assert len(bad) == 0, "%d mismatches; first: record %d %s (%r vs %r)" % (
        len(bad), bad[0][0], names[bad[0][1]], got[tuple(bad[0])], want[tuple(bad[0])])


def test_python_rigid3f_equals_header_on_special_inputs(header):
    rec = _special_records()
    _assert_bits_equal(_python_values(rec), _header_values(header, rec))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_python_rigid3f_equals_header_on_seeded_inputs(header, seed):
    rec = _seeded_records(seed, 3000)
    _assert_bits_equal(_python_values(rec), _header_values(header, rec))


# ---- range_data_poses, the gravity transform and the prediction ----
class _FakeSlam:
    """Records what AddRangeData hands the device and drops every scan."""

    def __init__(self):
        self.calls = []

    def accumulate(self, hits, origins, origin_index, poses, pose_index):
        self.calls.append(("accumulate", np.array(poses, np.float32), np.array(pose_index)))
        return {}

    def match(self, to_gravity, origin, prediction, grid):
        self.calls.append(("match", np.array(to_gravity, np.float32),
                           np.array(origin, np.float32), np.array(prediction, np.float64)))
        r = L.CsmLocalSlamMatch2D()
        r.status = L.DROPPED_EMPTY_RETURNS
        return r, {}


class _NoSubmaps:
    def submaps(self):
        return []


def _host_builder(extrapolator, num_accumulated=1):
    b = L.LocalTrajectoryBuilder2D.__new__(L.LocalTrajectoryBuilder2D)
    b.options = L.LocalTrajectoryBuilderOptions2D(num_accumulated_range_data=num_accumulated)
    b.extrapolator = extrapolator
    b.slam = _FakeSlam()
    b.active_submaps = _NoSubmaps()
    b.motion_filter = L.MotionFilter()
    b.num_accumulated = 0
    b.last_stats = None
    return b


def _trajectory(n=40, seed=5):
    rng = np.random.RandomState(seed)
    steps = np.stack([rng.uniform(0.05, 0.1, n), rng.uniform(-0.03, 0.03, n),
                      rng.uniform(-0.05, 0.05, n)], 1)
    return np.cumsum(steps, 0) + [3.0, -2.0, 0.4]


POINT_TIMES = {
    "repeated": [-0.05, -0.05, -0.03, -0.03, -0.03, -0.01, 0.0, 0.0],
    "unsorted": [-0.01, -0.04, -0.02, -0.03, -0.005, 0.0],
    "before the last extrapolation": [-0.15, -0.12, -0.1, -0.08, -0.02, 0.0],
    "single point": [0.0],
    "uniform": list(np.linspace(-0.05, 0.0, 11, dtype=np.float32)),
}


@pytest.mark.parametrize("case", list(POINT_TIMES))
def test_poses_gravity_and_prediction_against_float64(case):
    traj = _trajectory()
    ex_b, ex_r = K.TiltedExtrapolator(traj), K.TiltedExtrapolator(traj)
    b = _host_builder(ex_b)
    times = np.asarray(POINT_TIMES[case], np.float32)
    n = len(times)
    rng = np.random.RandomState(1)
    clamped = 0
    for k in range(6):
        time = 0.3 + 0.07 * k
        hw = np.concatenate([rng.uniform(-5, 5, (n, 3)), times[:, None]], 1).astype(np.float32)
        last_before = ex_r.GetLastExtrapolatedTime()
        clamped += int(np.sum(time + times.astype(np.float64) < last_before))
        want = K.range_data_poses(ex_r, time, times)
        gq = ex_r.EstimateGravityOrientation(time)
        want_pred = K.prediction64(ex_r.ExtrapolatePose(time), gq)
        b.slam.calls.clear()
        assert b.AddRangeData(time, hw, np.zeros((1, 3), np.float32), np.zeros(n, np.int32)) \
            is None
        (_, table, index), (_, to_gravity, origin, prediction) = b.slam.calls
        # one pose per point: the table entry of each point is its own extrapolated pose
        for i in range(n):
            assert table[index[i]].tobytes() == np.array(want[i][0] + want[i][1], F).tobytes()
        assert origin.tobytes() == np.array(want[-1][0], F).tobytes()
        R, t = K.to_gravity64(gq, want[-1])
        T = (to_gravity[:3], to_gravity[3:])
        got_R = K.rotation64(T[1])
        assert np.abs(got_R - R).max() <= 8 * 2.0 ** -24
        assert np.all(np.abs(T[0] - t) <= 8 * K.ulp32(np.abs(t).max() + 1.0))
        assert np.abs(prediction - want_pred).max() <= 1e-12
        assert ex_b.GetLastExtrapolatedTime() == ex_r.GetLastExtrapolatedTime()
    if case == "before the last extrapolation":
        assert clamped > 0
    if case == "single point":
        assert len(table) == 1


def test_unsorted_times_clamp_to_the_latest():
    """A point time before a later one already extrapolated takes that later pose."""
    ex = K.TiltedExtrapolator(_trajectory())
    poses = K.range_data_poses(ex, 0.3, POINT_TIMES["unsorted"])
    assert all(p == poses[0] for p in poses[1:4])       # -0.04, -0.02, -0.03 after -0.01
    assert poses[4] != poses[0] and poses[5] != poses[4]


# ---- the float32 restatement against the float64 geometry ----
def _random_pose(rng, reach):
    yaw, roll, pitch = rng.uniform(-math.pi, math.pi), rng.uniform(-0.3, 0.3), \
        rng.uniform(-0.3, 0.3)
    q = K.quat_mul64((math.cos(yaw / 2), 0, 0, math.sin(yaw / 2)),
                     K.quat_mul64((math.cos(pitch / 2), 0, math.sin(pitch / 2), 0),
                                  (math.cos(roll / 2), math.sin(roll / 2), 0, 0)))
    return L.rigid3f(rng.uniform(-reach, reach, 3), q)


@pytest.mark.parametrize("reach", [1.0, 1e3, 1e4])
def test_restatement_against_float64_geometry(reach):
    rng = np.random.RandomState(int(reach))
    n, min_range, max_range, ray = 1500, 0.5, 30.0, 5.0
    poses = [_random_pose(rng, reach) for _ in range(9)]
    origins = rng.uniform(-0.3, 0.3, (7, 3)).astype(np.float32)
    oi, pi = rng.randint(0, 7, n), rng.randint(0, 9, n)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rr = rng.uniform(0.0, 40.0, n)
    spread = 64 * float(K.ulp32(reach + 40.0))               # around both thresholds
    rr[:100] = min_range + rng.uniform(-spread, spread, 100)
    rr[100:200] = max_range + rng.uniform(-spread, spread, 100)
    rr[200:300] = rng.uniform(0.0, 0.4, 100)
    hits = (origins[oi] + d * rr[:, None]).astype(np.float32)
    g = K.geometry64(hits, origins, oi, poses, pi, ray)
    tol = K.F32_GEOMETRY_ULPS * K.ulp32(g["scale"])
    counts = {"return": 0, "miss": 0, "dropped": 0, "undecided": 0}
    for i in range(n):
        r, m = O.accumulate(hits[i:i + 1], origins, oi[i:i + 1], poses, pi[i:i + 1],
                            min_range, max_range, ray)
        kind = "return" if len(r) else "miss" if len(m) else "dropped"
        rg = g["range"][i]
        if abs(rg - min_range) <= tol[i] or abs(rg - max_range) <= tol[i]:
            counts["undecided"] += 1
        else:
            want = ("dropped" if rg < min_range else "return" if rg <= max_range else "miss")
            assert kind == want, (i, rg, kind)
            counts[kind] += 1
        if kind == "return":
            assert np.abs(r[0] - g["hit"][i]).max() <= tol[i], i
        elif kind == "miss":
            mtol = K.F32_GEOMETRY_ULPS * (K.ulp32(g["scale"][i]) * (1 + ray / rg) + K.ulp32(ray))
            assert np.abs(m[0] - g["miss"][i]).max() <= mtol, i
    assert min(counts["return"], counts["miss"], counts["dropped"]) > 20, counts
    assert 0 < counts["undecided"] < 100, counts


@pytest.mark.parametrize("reach", [1.0, 1e3])
def test_gravity_crop_against_float64_geometry(reach):
    rng = np.random.RandomState(7 + int(reach))
    n = 2000
    T = _random_pose(rng, reach)
    Tinv = L.rigid3f_inverse(T)
    z = rng.uniform(-3.0, 4.0, n)
    z[:50] = -0.8 + rng.uniform(-1e-5, 1e-5, 50)
    z[50:100] = 2.0 + rng.uniform(-1e-5, 1e-5, 50)
    local = np.stack([rng.uniform(-30, 30, n), rng.uniform(-30, 30, n), z], 1)
    pts = K.transform64(local, (np.asarray(Tinv[0], np.float64), Tinv[1])).astype(np.float32)
    got = O.transform(pts, T)
    want = K.transform64(pts, T)
    scale = np.maximum(np.abs(pts).max(1), np.abs(np.asarray(T[0], np.float64)).max())
    scale = np.maximum(scale, np.abs(want).max(1))
    tol = K.F32_GEOMETRY_ULPS * K.ulp32(scale)
    assert np.all(np.abs(got - want).max(1) <= tol)
    kept = np.zeros(n, bool)
    kept[np.flatnonzero((F(-0.8) <= got[:, 2]) & (got[:, 2] <= F(2.0)))] = True
    assert O.crop(got, -0.8, 2.0).tobytes() == got[kept].tobytes()
    clear = (np.abs(want[:, 2] + 0.8) > tol) & (np.abs(want[:, 2] - 2.0) > tol)
    assert np.array_equal(kept[clear], ((-0.8 <= want[:, 2]) & (want[:, 2] <= 2.0))[clear])
    assert clear.sum() > n - 150 and kept.sum() > 100 and (~kept).sum() > 100


def test_column_restatement_equals_the_scalar_one():
    """The chain's column form of accumulate / transform, bit for bit with the scalar
    restatement, with -0.0, zero ranges, both thresholds and per-point poses."""
    rng = np.random.RandomState(11)
    n = 600
    poses = [_random_pose(rng, r) for r in (0.0, 1.0, 1e3, 1e4)] + [
        L.rigid3f((-0.0, 0.0, -0.0), (1.0, -0.0, 0.0, -0.0))]
    origins = np.vstack([rng.uniform(-0.3, 0.3, (6, 3)), [[-0.0, 0.0, -0.0]]]).astype(np.float32)
    oi, pi = rng.randint(0, 7, n), rng.randint(0, 5, n)
    hits = (origins[oi] + rng.normal(size=(n, 3)) * rng.choice([0.0, 0.2, 5.0, 35.0], (n, 1)))
    hits = hits.astype(np.float32)
    hits[::17] = -0.0
    for args in ((0.0, 30.0, 5.0), (0.2, 30.0, 1e6)):
        want = O.accumulate(hits, origins, oi, poses, pi, *args)
        got = K.accumulate(hits, origins, oi, poses, pi, *args)
        assert want[0].tobytes() == got[0].tobytes() and want[1].tobytes() == got[1].tobytes()
    for p in poses:
        assert O.transform(hits, p).tobytes() == K.transform(hits, p).tobytes()
