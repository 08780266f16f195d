"""The float64 references of tests/map_writing3d_refs.py against their own brute-force or exact
versions: ulp neighbours, the submap transform, the range and cell sides, the slack box and the
keep patterns."""
import ctypes as C
import math
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from tests import insert3d_oracle as O
from tests import map_writing3d_refs as M
from tests.test_gpu_active_submaps3d import host_transform

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

F = np.float32


def test_ulp_neighbours_are_adjacent_floats():
    x = F([1.0, -1.0, 8191.5, -8192.5, 20.0, 1e-30, 3.4e38, 40.0])
    lo, mid, hi = M.ulp_neighbours(x)
    bits = x.view(np.int32).astype(np.int64)
    # the neighbours are the adjacent bit patterns (magnitudes grow away from zero)
    for v, step in ((lo, -1), (hi, 1)):
        vb = v.view(np.int32).astype(np.int64)
        np.testing.assert_array_equal(vb - bits, np.where(x > 0, step, -step))
    np.testing.assert_array_equal(mid, x)
    assert float(hi[2]) - 8191.5 == 2.0 ** -11 and 8191.5 - float(lo[2]) == 2.0 ** -11


def test_rotation_matches_quaternion_product():
    rng = np.random.RandomState(1)
    for _ in range(50):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        v = rng.normal(size=3)
        w, x, y, z = q
        # q v q*, by Hamilton products
        def mul(a, b):
            return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                             a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                             a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
                             a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])
        want = mul(mul(q, np.r_[0.0, v]), np.array([w, -x, -y, -z]))[1:]
        np.testing.assert_allclose(M.rotation64(q) @ v, want, rtol=0, atol=1e-12)


def test_submap_frame_inverts_the_pose():
    rng = np.random.RandomState(2)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    pose = [3.0, -2.0, 0.5, *q]
    s = rng.normal(size=(20, 3)) * 10
    p = s @ M.rotation64(q).T + np.array(pose[:3])
    got, scale = M.submap_frame64(pose, p)
    np.testing.assert_allclose(got, s, rtol=0, atol=1e-12)
    assert (scale >= np.abs(got).max(1)).all()


def _exact_range_side(o, p, max_range):
    d2 = sum((Fraction(float(a)) - Fraction(float(b))) ** 2 for a, b in zip(p, o))
    r2 = Fraction(float(max_range)) ** 2
    return 1 if d2 <= r2 else -1


def test_range_sides_agree_with_exact_arithmetic_where_decided():
    rng = np.random.RandomState(3)
    ident = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    max_range = 5.0
    d = rng.normal(size=(400, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = max_range * (1 + rng.choice([-1e-3, -1e-6, 0.0, 1e-6, 1e-3], 400))
    o = np.zeros(3)
    p = (d * r[:, None]).astype(F)
    side = M.range_sides64(ident, o, p, max_range)
    for s, pt in zip(side, p):
        if s != 0:
            assert s == _exact_range_side(o, pt, max_range)
    assert (side == 0).any() and (side == 1).any() and (side == -1).any()
    # float32 evaluation (what the device does) agrees wherever the float64 side is decided
    dd = (p - F(0)).astype(F)
    f32 = np.sqrt((dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]) <= F(max_range)
    assert ((side == 0) | ((side == 1) == f32)).all()


def test_cell_sides_agree_with_float32_quotient_where_decided():
    rng = np.random.RandomState(4)
    for res in (0.1, 0.45, 0.5, 1.0):
        q = rng.randint(-8000, 8000, 3000) + 0.5 + rng.choice([-1e-3, -1e-7, 0.0, 1e-7, 1e-3], 3000)
        p = (q * float(F(res))).astype(F)
        pts = np.stack([p, p[::-1], np.roll(p, 7)], 1)
        cells, decided = M.cell_sides64(pts, res)
        want = O.cell_index(res, pts)   # float32 division, then lround
        if res in (0.5, 1.0):   # exact quotients: every tie decided, halves away from zero
            assert decided.all()
        else:
            assert decided.any() and (~decided).any()
        np.testing.assert_array_equal(cells[decided], want[decided])


def test_lround_halves_away_from_zero():
    v = np.array([-2.5, -1.5, -0.5, 0.5, 1.5, 2.5, 2.4999, -2.4999, 0.0])
    np.testing.assert_array_equal(M.lround64(v), [-3, -2, -1, 1, 2, 3, 2, -2, 0])
    np.testing.assert_array_equal(M.lround64(v), [int(math.copysign(math.floor(abs(x) + 0.5), x))
                                                  for x in v])


def test_slack_box_brute_force():
    rng = np.random.RandomState(5)
    for _ in range(200):
        lo = rng.randint(-8192, 8192, 3)
        hi = np.minimum(lo + rng.randint(0, 3000, 3), 8191)
        blo, dims = M.slack_box(lo, hi)
        for a in range(3):
            s = (hi[a] - lo[a] + 1) // 8
            cells = [c for c in (lo[a] - s, hi[a] + s)]
            want_lo = max(-8192, cells[0])
            want_hi = min(8191, cells[1])
            assert blo[a] == want_lo and blo[a] + dims[a] - 1 == want_hi
        assert (blo >= -8192).all() and (blo + dims <= 8192).all()


def test_lane_keep_patterns():
    n = 257
    for name in M.KEEP_PATTERNS:
        k = M.lane_keep(name, n)
        assert k.shape == (n,)
        for i in range(n):
            want = {"all": True, "none": False, "lane0": i % 32 == 0, "lane31": i % 32 == 31,
                    "alternating": i % 2 == 0, "warps_dropped": (i // 32) % 3 != 1}[name]
            assert k[i] == want


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    """The float32 submap transform the device agrees with (rigid3f.h), on the host."""
    so = str(tmp_path_factory.mktemp("map_writing3d_refs") / "libsubmap_insert3d_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                           os.path.join(ROOT, "tests", "submap_insert3d_oracle.cc"), "-o", so])
    return C.CDLL(so)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_rotated_sides_agree_with_the_float32_transform(host, seed):
    """Under tilted, translated poses, returns placed (in float64) near max_range and near half
    cells of the submap frame: wherever range_sides64 and cell_sides64(scale) decide, the
    float32 transform, range filter and GetCellIndex decide the same."""
    rng = np.random.RandomState(seed)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    pose = [*rng.uniform(-30, 30, 3), *q]
    origin = rng.uniform(-2, 2, 3).astype(F)
    res, max_range, n = 0.1, 7.5, 4000
    o64, _ = M.submap_frame64(pose, origin)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    delta = rng.choice([-1e-2, -1e-4, -1e-6, 0.0, 1e-6, 1e-4, 1e-2], (n, 1))
    sub = o64 + d * max_range * (1 + delta)
    # half the returns moved onto a half cell of one axis, plus a small offset
    a = rng.randint(0, 3, n)
    half = rng.rand(n) < 0.5
    c = (np.floor(sub[np.arange(n), a] / float(F(res))) + 0.5 + delta[:, 0]) * float(F(res))
    sub[half, a[half]] = c[half]
    pts = (sub @ M.rotation64(q).T + np.asarray(pose[:3])).astype(F)
    _, p32, kept = host_transform(host, pose, origin, pts, max_range)
    side = M.range_sides64(pose, origin, pts, max_range)
    assert (side != 0).sum() > n // 3 and (side == 0).any()
    np.testing.assert_array_equal(kept[side != 0], side[side != 0] == 1)
    p64, scale = M.submap_frame64(pose, pts)
    cells, decided = M.cell_sides64(p64, res, scale)
    assert decided.sum() > n // 3 and (~decided[half]).any()
    np.testing.assert_array_equal(cells[decided], O.cell_index(res, p32)[decided])
