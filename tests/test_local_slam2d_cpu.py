"""LocalTrajectoryBuilder2D's host pieces without a device: the float32 restatement on
hand-derived cases, the motion filter at its thresholds, the ABI's symbols and layouts, and
the refusals that come before any device work."""
import ctypes as C
import math

import numpy as np
import pytest

from cartographer_b200 import _lib
from cartographer_b200 import local_slam as L
from tests import local_slam2d_oracle as O

F = np.float32
IDENTITY = L.rigid3f((0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0))


def test_range_edges():
    above = np.nextafter(F(30.0), F(31.0))
    hits = np.array([[0.2, 0, 0], [30.0, 0, 0], [above, 0, 0], [0.19, 0, 0]], np.float32)
    r, m = O.accumulate(hits, [[0, 0, 0]], [0] * 4, [IDENTITY], [0] * 4, 0.2, 30.0, 5.0)
    assert r.tolist() == [[F(0.2), 0, 0], [30.0, 0, 0]]    # exactly min_range and max_range
    assert m.shape == (1, 3) and m[0, 0] == F(5.0) * above / above


def test_poses_and_origins():
    p0 = L.rigid3f((1.0, 2.0, 0.0), (1.0, 0.0, 0.0, 0.0))
    p1 = L.rigid3f((0.0, 0.0, 0.0), (math.cos(0.5), 0.0, 0.0, math.sin(0.5)))
    hits = np.array([[1, 0, 0], [2, 0, 0], [3, 0, 0]], np.float32)
    origins = np.array([[0, 0, 0], [1, 0, 0]], np.float32)
    r, _ = O.accumulate(hits, origins, [0, 1, 1], [p0, p1], [0, 0, 1], 0.0, 30.0, 5.0)
    assert r[0].tolist() == [2, 2, 0] and r[1].tolist() == [3, 2, 0]
    assert np.allclose(r[2], [3 * math.cos(1.0), 3 * math.sin(1.0), 0], atol=1e-6)
    # a hit on its origin has range 0: below any positive min_range
    r, m = O.accumulate([[1, 0, 0]], origins, [1], [p1], [0], 0.1, 30.0, 5.0)
    assert len(r) == 0 and len(m) == 0


def test_crop_edges():
    p = np.array([[0, 0, -0.8], [0, 0, 2.0], [0, 0, np.nextafter(F(2.0), F(3))],
                  [0, 0, np.nextafter(F(-0.8), F(-1))]], np.float32)
    assert O.crop(p, -0.8, 2.0).tolist() == p[:2].tolist()


def test_accumulation_over_three_scans():
    scans = [np.array([[1, 0, 0], [40, 0, 0]], np.float32) * (k + 1) for k in range(3)]
    parts = [O.accumulate(s, [[0, 0, 0]], [0, 0], [IDENTITY], [0, 0], 0.0, 30.0, 5.0)
             for s in scans]
    ret = np.concatenate([p[0] for p in parts])
    mis = np.concatenate([p[1] for p in parts])
    assert ret[:, 0].tolist() == [1, 2, 3] and mis[:, 0].tolist() == [5, 5, 5]


def _pose(x, yaw):
    return ((x, 0.0, 0.0), (math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)))


@pytest.mark.parametrize("dt,dx,dyaw,similar", [
    (5.0, 0.0, 0.0, True), (5.0 + 1e-7, 0.0, 0.0, False),
    (1.0, 0.2, 0.0, True), (1.0, 0.2 + 1e-9, 0.0, False),
    (1.0, 0.0, math.radians(1.0) * (1 - 1e-9), True), (1.0, 0.0, math.radians(1.0) * 1.001, False)])
def test_motion_filter_thresholds(dt, dx, dyaw, similar):
    mf = L.MotionFilter()
    assert not mf.IsSimilar(10.0, _pose(1.0, 0.3))
    assert mf.IsSimilar(10.0 + dt, _pose(1.0 + dx, 0.3 + dyaw)) == similar
    assert mf.num_different == (1 if similar else 2)


def test_options_defaults():
    o = L.LocalTrajectoryBuilderOptions2D()
    assert (o.min_range, o.max_range, o.min_z, o.max_z) == (0.0, 30.0, -0.8, 2.0)
    assert o.missing_data_ray_length == 5.0 and o.voxel_filter_size == 0.025
    assert o.num_accumulated_range_data == 1 and not o.use_online_correlative_scan_matching
    c = o.ceres_scan_matcher_options
    assert (c.occupied_space_weight, c.translation_weight, c.rotation_weight) == (1.0, 10.0, 40.0)
    assert c.max_num_iterations == 20 and not c.use_nonmonotonic_steps


def test_symbols_and_layouts():
    lib = _lib.lib()
    for name in ("csm_local_slam2d_create", "csm_local_slam2d_destroy",
                 "csm_local_slam2d_accumulate", "csm_local_slam2d_match",
                 "csm_local_slam2d_insert", "csm_local_slam2d_read"):
        assert hasattr(lib, name)
    # float fields, int fields, the nested option records, then the doubles
    assert C.sizeof(L.CsmLocalSlamOptions2D) == 32 + 16 + 32 + 32 + 24
    assert C.sizeof(L.CsmLocalSlamMatch2D) == 24 + 24 + 8 + 56
    with open(_lib.os.path.join(_lib._PKG, "..", "include", "csm_abi.h")) as f:
        abi = f.read()
    assert "csm_local_slam_options2d" in abi and "csm_local_slam2d_read" in abi


def test_refusals_before_the_device():
    lib = _lib.lib()
    h = C.c_void_p()
    o = L.c_options(L.LocalTrajectoryBuilderOptions2D())
    o.voxel_filter_size = 0.0
    assert lib.csm_local_slam2d_create(C.byref(o), 0, C.byref(h)) == 1
    o = L.c_options(L.LocalTrajectoryBuilderOptions2D())
    o.num_accumulated_range_data = 0
    assert lib.csm_local_slam2d_create(C.byref(o), 0, C.byref(h)) == 1
    o = L.c_options(L.LocalTrajectoryBuilderOptions2D())
    o.max_z = float("nan")
    assert lib.csm_local_slam2d_create(C.byref(o), 0, C.byref(h)) == 1
    assert lib.csm_local_slam2d_accumulate(None, None, 0, None, 0, None, None, 0, None, None) == 1
    assert lib.csm_local_slam2d_match(None, None, None, None, None, None, None) == 1
    assert lib.csm_local_slam2d_insert(None, None, None, 0, None, None) == 1
    assert lib.csm_local_slam2d_read(None, 0, None, 0, None) == 1
    assert h.value is None


def test_vectorised_recipe_equals_the_restatement():
    from benchmarks import local_slam2d_recipe as R
    rng = np.random.RandomState(3)
    n = 400
    hits = (rng.uniform(-40, 40, (n, 3)) * [1, 1, 0.05]).astype(np.float32)
    origins = rng.uniform(-0.2, 0.2, (3, 3)).astype(np.float32)
    oi = rng.randint(0, 3, n)
    poses = [L.rigid3f(rng.uniform(-5, 5, 3), L._quatd_normalized(tuple(rng.normal(size=4))))
             for _ in range(7)]
    pi = rng.randint(0, 7, n)
    want = O.accumulate(hits, origins, oi, poses, pi, 0.2, 30.0, 5.0)
    got = R.accumulate(hits, origins, oi, poses, pi, 0.2, 30.0, 5.0)
    for w, g in zip(want, got):
        assert w.tobytes() == g.tobytes()
    T = poses[0]
    assert O.transform(hits, T).tobytes() == R.transform(hits, T).tobytes()
    assert O.crop(hits, -0.8, 0.5).tobytes() == R.crop(hits, -0.8, 0.5).tobytes()


def test_project2d_is_getyaw():
    for yaw in (0.0, 0.3, -2.9, math.pi - 1e-6):
        q = (math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2))
        assert abs(L.project2d(((1.0, 2.0, 3.0), q))[2] - yaw) < 1e-12
