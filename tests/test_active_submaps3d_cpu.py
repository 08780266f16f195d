"""Submap3D::InsertData's host-side arithmetic, without a GPU: the g++ restatement in
tests/submap_insert3d_oracle.cc (the submap-frame transform, the high-resolution range filter,
the cells, the yaw and RotateHistogram) against hand-derived cases, the Python histogram
accumulation against it bit for bit, and the new entry point's symbol, declaration, struct
layout and refusals."""
import ctypes as C
import math
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("submap_insert3d") / "libsubmap_insert3d_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                           os.path.join(ROOT, "tests", "submap_insert3d_oracle.cc"), "-o", so])
    lib = C.CDLL(so)
    lib.submap_yaw.restype = C.c_float
    return lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def transform(oracle, pose, origin, returns, max_range):
    pose = np.asarray(pose, np.float64)
    pts = np.ascontiguousarray(returns, F).reshape(-1, 3)
    org = np.asarray(origin, F)
    out_o, out_p = np.zeros(3, F), np.zeros_like(pts)
    kept = np.zeros(len(pts), np.uint8)
    oracle.submap_transform(_p(pose, C.c_double), _p(org, C.c_float), _p(pts, C.c_float),
                            len(pts), C.c_float(max_range), _p(out_o, C.c_float),
                            _p(out_p, C.c_float), _p(kept, C.c_uint8))
    return out_o, out_p, kept.astype(bool)


def cells(oracle, pts, resolution):
    pts = np.ascontiguousarray(pts, F).reshape(-1, 3)
    out = np.zeros(pts.shape, np.int32)
    ok = np.zeros(len(pts), np.uint8)
    oracle.submap_cells(_p(pts, C.c_float), len(pts), C.c_float(resolution),
                        _p(out, C.c_int32), _p(ok, C.c_uint8))
    return out, ok.astype(bool)


def yaw_pose(yaw, t=(0.0, 0.0, 0.0)):
    return [*t, math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)]


def test_identity_pose_keeps_every_point(oracle):
    pts = np.float32([[1.5, -2.25, 0.125], [-0.0, 0.0, -7.0], [19.0, 3.0, -1.0]])
    o, p, kept = transform(oracle, yaw_pose(0.0), [0.5, 0.25, -0.5], pts, 20.0)
    np.testing.assert_array_equal(o, F([0.5, 0.25, -0.5]))
    np.testing.assert_array_equal(p, pts)
    assert kept.tolist() == [True, True, True]


@pytest.mark.parametrize("yaw", [math.pi / 2, math.pi / 4, -math.pi / 2])
def test_yawed_pose(oracle, yaw):
    # submap at (1, 2, 0.5) turned by yaw: the local point t + R (a, b, c) is (a, b, c) there
    t = np.array([1.0, 2.0, 0.5])
    c, s = math.cos(yaw), math.sin(yaw)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    want = np.array([[3.0, 0.0, 0.25], [0.0, -2.0, 1.0], [0.5, 0.5, 0.0]])
    local = (want @ R.T + t).astype(F)
    o, p, _ = transform(oracle, yaw_pose(yaw, t), t.astype(F), local, 20.0)
    np.testing.assert_allclose(p, want, atol=2e-6)
    np.testing.assert_allclose(o, 0.0, atol=5e-7)   # a few ulps of the 2 m translation


def test_tilted_pose(oracle):
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(4)
    q = Rotation.from_rotvec([0.3, -0.5, 0.2])
    x, y, z, w = q.as_quat()
    t = np.array([2.0, -1.0, 0.75])
    local = rng.uniform(-10, 10, (50, 3)).astype(F)
    _, p, _ = transform(oracle, [*t, w, x, y, z], t.astype(F), local, 20.0)
    want = q.inv().apply(local.astype(np.float64) - t)
    np.testing.assert_allclose(p, want, atol=1e-5)
    # the inverse in double, then cast, as Rigid3d::inverse().cast<float>() gives it
    inv = np.zeros(7, F)
    oracle.submap_inverse(_p(np.array([*t, w, x, y, z]), C.c_double), _p(inv, C.c_float))
    np.testing.assert_array_equal(inv[3:], F([w, -x, -y, -z]))
    np.testing.assert_array_equal(inv[:3], (-q.inv().apply(t)).astype(F))


def test_range_filter_edge(oracle):
    above = np.nextafter(F(20.0), F(np.inf))
    pts = np.float32([[20.0, 0, 0], [above, 0, 0], [0, -20.0, 0], [0, 0, above],
                      [12.0, 16.0, 0.0], [np.nan, 0, 0]])
    _, _, kept = transform(oracle, yaw_pose(0.0), [0, 0, 0], pts, 20.0)
    assert kept.tolist() == [True, False, True, False, True, False]
    # the filter measures from the transformed origin
    _, _, kept = transform(oracle, yaw_pose(0.0, (5.0, 0.0, 0.0)), [5.0, 0, 0],
                           np.float32([[25.0, 0, 0], [-15.0, 0, 0], [-15.5, 0, 0]]), 20.0)
    assert kept.tolist() == [True, True, False]


def test_half_cell_ties_after_the_transform(oracle):
    # a 0.25 m shift puts these returns on ±0.5 cell ties at 0.5 m: lround rounds them away
    # from zero
    pose = yaw_pose(0.0, (0.25, -0.25, 0.0))
    pts = np.float32([[0.5, 0.0, 0.25], [0.0, -0.5, -0.25], [1.0, 0.5, 0.75]])
    _, p, _ = transform(oracle, pose, [0.25, -0.25, 0], pts, 20.0)
    np.testing.assert_array_equal(p, F([[0.25, 0.25, 0.25], [-0.25, -0.25, -0.25],
                                        [0.75, 0.75, 0.75]]))
    c, ok = cells(oracle, p, 0.5)
    assert ok.all()
    np.testing.assert_array_equal(c, [[1, 1, 1], [-1, -1, -1], [2, 2, 2]])


def test_cells_cube_and_nonfinite(oracle):
    # at 0.5 m: 8191.4 and -8192.4 cells are inside, 8191.6 and -8192.6 outside
    c, ok = cells(oracle, np.float32([[4095.7, 0, 0], [4095.8, 0, 0], [-4096.2, 0, 0],
                                      [-4096.3, 0, 0], [np.inf, 0, 0], [0, np.nan, 0]]), 0.5)
    assert ok.tolist() == [True, False, True, False, False, False]
    assert c[0, 0] == 8191 and c[2, 0] == -8192


def _accumulate(oracle, hist, scan, angle):
    h = np.ascontiguousarray(hist, F).copy()
    s = np.ascontiguousarray(scan, F)
    oracle.submap_accumulate_histogram(_p(h, C.c_float), _p(s, C.c_float), len(s),
                                       C.c_float(angle))
    return h


def test_rotate_histogram_hand_values(oracle):
    from cartographer_b200 import scan_matching as sm
    h = F([1, 2, 3, 4])
    z = np.zeros(4, F)
    cases = [(0.0, [1, 2, 3, 4]),                          # fraction 1 onto the same bucket
             (-math.pi / 4, [2, 3, 4, 1]),                 # one bucket
             (-math.pi / 8, [1.5, 2.5, 3.5, 2.5]),         # half a bucket
             (math.pi / 4, [4, 1, 2, 3])]                  # one bucket the other way
    for angle, want in cases:
        got = _accumulate(oracle, z, h, angle)
        np.testing.assert_allclose(got, want, rtol=1e-6)
        np.testing.assert_array_equal(got.view(np.uint32),
                                      sm.rotate_histogram(h, angle).view(np.uint32))
    assert len(sm.rotate_histogram(np.zeros(0, F), 1.0)) == 0


def test_histogram_accumulation_python_equals_cpp(oracle):
    from cartographer_b200 import scan_matching as sm
    rng = np.random.RandomState(9)
    hist_c = np.zeros(120, F)
    hist_py = np.zeros(120, F)
    for k in range(200):
        pose = [*rng.uniform(-5, 5, 3), *rng.normal(size=4)]
        pose[3:] = list(np.asarray(pose[3:]) / np.linalg.norm(pose[3:]))
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        if k % 10 == 0:
            q = np.array([1.0, 0.0, 0.0, 0.0])   # gravity-aligned local frame
        scan = rng.uniform(0, 50, 120).astype(F)
        yaw_c = oracle.submap_yaw(_p(np.asarray(pose, np.float64), C.c_double),
                                  _p(np.asarray(q, np.float64), C.c_double))
        yaw_py = sm.yaw_in_submap_from_gravity(pose, q)
        assert F(yaw_c).view(np.uint32) == F(yaw_py).view(np.uint32)
        hist_c = _accumulate(oracle, hist_c, scan, yaw_c)
        hist_py = hist_py + sm.rotate_histogram(scan, yaw_py)
    np.testing.assert_array_equal(hist_c.view(np.uint32), hist_py.view(np.uint32))
    # a pure yaw: the submap frame's yaw is the difference of the two
    assert abs(sm.yaw_in_submap_from_gravity(yaw_pose(0.5), yaw_pose(1.25)[3:]) - 0.75) < 1e-6


def test_symbol_declaration_and_layout():
    from cartographer_b200 import scan_matching as sm
    from cartographer_b200._lib import SO_PATH
    syms = subprocess.run(["nm", "-D", "--defined-only", SO_PATH], capture_output=True,
                          text=True, check=True).stdout
    assert re.search(r"\bcsm_range_inserter3d_insert_submaps\b", syms)
    header = open(os.path.join(ROOT, "include", "csm_abi.h")).read()
    assert re.search(r"csm_status csm_range_inserter3d_insert_submaps\(const csm_range_inserter3d\* "
                     r"inserter,\s+const csm_submap_insert3d\* submaps,", header)
    struct = re.search(r"typedef struct csm_submap_insert3d \{(.*?)\} csm_submap_insert3d;",
                       header, re.S).group(1)
    fields = re.findall(r"^\s*([\w ]+?\*?)\s*(\w+)(\[\d+\])?;", struct, re.M)
    assert [f[1] for f in fields] == ["local_pose", "high_resolution", "low_resolution",
                                      "intensity"]
    S = sm.CsmSubmapInsert3D
    assert C.sizeof(S) == 80
    assert [S.local_pose.offset, S.high_resolution.offset, S.low_resolution.offset,
            S.intensity.offset] == [0, 56, 64, 72]


def test_refusals_without_a_device():
    from cartographer_b200._lib import lib
    L = lib()
    org = np.zeros(3, F)
    entries = (C.c_byte * 80)()
    pts = np.zeros((1, 3), F)
    op, pp = _p(org, C.c_float), _p(pts, C.c_float)
    # null inserter, null entries, null origin, no entries, returns missing
    assert L.csm_range_inserter3d_insert_submaps(None, entries, 1, op, pp, None, 1,
                                                 C.c_float(20), None) == 1
    assert L.csm_range_inserter3d_insert_submaps(C.c_void_p(8), None, 1, op, pp, None, 1,
                                                 C.c_float(20), None) == 1
    assert L.csm_range_inserter3d_insert_submaps(C.c_void_p(8), entries, 1, None, pp, None, 1,
                                                 C.c_float(20), None) == 1
    assert L.csm_range_inserter3d_insert_submaps(C.c_void_p(8), entries, 0, op, pp, None, 1,
                                                 C.c_float(20), None) == 1
    assert L.csm_range_inserter3d_insert_submaps(C.c_void_p(8), entries, 1, op, None, None, 1,
                                                 C.c_float(20), None) == 1
    assert L.csm_range_inserter3d_insert_submaps(C.c_void_p(8), entries, 1, op, pp, None, -1,
                                                 C.c_float(20), None) == 1
