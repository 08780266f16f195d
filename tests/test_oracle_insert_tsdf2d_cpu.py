"""The CPU restatement of TSDFRangeDataInserter2D and NormalEstimation2D
(tests/insert_tsdf2d_oracle.cc) against the reference's known answers
(tsdf_range_data_inserter_2d_test.cc, normal_estimation_2d_test.cc) and the numpy fixture builder
tests/tsdf_inserter.py; the TSDF inserter's C ABI record and status codes without a device."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import insert_tsdf2d_oracle as O
from tests import tsdf2d_oracle
from tests import tsdf_inserter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Opts:
    """TSDFRangeDataInserterOptions2D fields without importing the product package."""

    def __init__(self, **kw):
        self.truncation_distance = 0.3
        self.maximum_weight = 10.0
        self.update_free_space = False
        self.num_normal_samples = 4
        self.sample_radius = 0.5
        self.project_sdf_distance_to_scan_normal = True
        self.update_weight_range_exponent = 0
        self.update_weight_angle_scan_normal_to_ray_kernel_bandwidth = 0.5
        self.update_weight_distance_cell_to_hit_kernel_bandwidth = 0.5
        self.__dict__.update(kw)


# ---- tsdf_range_data_inserter_2d_test.cc ----
def _ref_options(**kw):
    base = dict(truncation_distance=2.0, maximum_weight=10.0, update_free_space=False,
                num_normal_samples=2, sample_radius=10.0,
                project_sdf_distance_to_scan_normal=False, update_weight_range_exponent=0,
                update_weight_angle_scan_normal_to_ray_kernel_bandwidth=0.0,
                update_weight_distance_cell_to_hit_kernel_bandwidth=0.0)
    base.update(kw)
    return _Opts(**base)


def _ref_grid():
    """MapLimits(1., (1., 7.), CellLimits(8, 1)), truncation 2, maximum weight 10."""
    return O.TsdfGrid(1.0, 1.0, 7.0, 8, 1, 2.0, 10.0)


ORIGIN = np.float32([-0.5, -0.5, 0])
POINT = np.float32([[-0.5, 3.5, 0]])


def _cell(g, x, y):
    return g.get(*g.cell_index(x, y))


def _expect(got, known, tsd, weight):
    assert got[0] == known
    assert abs(got[1] - tsd) < 1e-4, got
    assert abs(got[2] - weight) < 1e-2, got


def _insert_point_case(free_space):
    opts = _ref_options(update_free_space=free_space)
    ins, g = O.TsdfInserter(opts), _ref_grid()
    assert ins.insert(ORIGIN, POINT, g)
    ys = np.arange(-0.5 if free_space else 1.5, 6.0, 1.0)
    for y in ys:
        _expect(_cell(g, -0.5, y), True, max(min(3.5 - y, 2.0), -2.0), 1.0)
        for x in (0.5, 1.5):
            _expect(_cell(g, x, y), False, -2.0, 0.0)
    _expect(_cell(g, 0.5 if not free_space else -0.5, 6.5), False, -2.0, 0.0)
    _expect(_cell(g, -0.5, -1.5), False, -2.0, 0.0)
    for _ in range(1000):
        assert ins.insert(ORIGIN, POINT, g)
    for y in ys:
        _expect(_cell(g, -0.5, y), True, max(min(3.5 - y, 2.0), -2.0), 10.0)
    return g


def test_insert_point():
    g = _insert_point_case(False)
    assert g.limits[3] > 8   # grew out of the 8 x 1 grid


def test_insert_point_with_free_space_update():
    _insert_point_case(True)


@pytest.mark.parametrize("exponent,weight", [(1, 1.0 / 4.0), (2, 1.0 / 16.0)])
def test_insert_point_range_weight(exponent, weight):
    ins, g = O.TsdfInserter(_ref_options(update_weight_range_exponent=exponent)), _ref_grid()
    assert ins.insert(ORIGIN, POINT, g)
    for y in np.arange(1.5, 6.0, 1.0):
        _expect(_cell(g, -0.5, y), True, max(min(3.5 - y, 2.0), -2.0), weight)


def test_insert_small_angle_point_without_normal_projection():
    ins, g = O.TsdfInserter(_ref_options()), _ref_grid()
    assert ins.insert(ORIGIN, np.float32([[-0.5, 3.5, 0], [5.5, 3.5, 0], [10.5, 3.5, 0]]), g)
    ray = np.float32([-0.5, -0.5]) - np.float32([5.5, 3.5])
    to_cell = np.float32([4.5, 2.5]) - np.float32([-0.5, -0.5])
    tsd = np.float32(math.sqrt(float(ray @ ray))) - np.float32(math.sqrt(float(to_cell @ to_cell)))
    _expect(_cell(g, 4.5, 2.5), True, float(tsd), 1.0)


def test_insert_small_angle_point_with_normal_projection():
    ins = O.TsdfInserter(_ref_options(project_sdf_distance_to_scan_normal=True))
    g = _ref_grid()
    assert ins.insert(ORIGIN, np.float32([[-0.5, 3.5, 0], [5.5, 3.5, 0]]), g)
    _expect(_cell(g, 4.5, 2.5), True, 1.0, 1.0)
    _expect(_cell(g, 6.5, 4.5), True, -1.0, 1.0)


def test_insert_points_with_angle_scan_normal_to_ray_weight():
    bw = 10.0
    ins = O.TsdfInserter(_ref_options(update_weight_angle_scan_normal_to_ray_kernel_bandwidth=bw))
    g = _ref_grid()
    assert ins.insert(ORIGIN, np.float32([[-0.5, 3.5, 0], [5.5, 3.5, 0]]), g)
    perpendicular = 1.0 / (math.sqrt(2 * math.pi) * bw)
    assert abs(_cell(g, -0.5, 3.5)[2] - perpendicular) < 1e-3
    assert abs(_cell(g, 6.5, 4.5)[2] - perpendicular) < 1e-3
    angle = math.atan(7.0 / 5.0)
    inclined = perpendicular * math.exp(angle * angle / (2 * bw ** 2))
    assert abs(_cell(g, 6.5, 4.5)[2] - inclined) < 1e-3


def test_insert_points_with_distance_cell_to_hit():
    bw = 10.0
    ins = O.TsdfInserter(_ref_options(update_weight_distance_cell_to_hit_kernel_bandwidth=bw))
    g = _ref_grid()
    assert ins.insert(ORIGIN, POINT, g)
    for y in np.arange(1.5, 6.0, 1.0):
        tsd = max(min(3.5 - y, 2.0), -2.0)
        weight = 1.0 / (math.sqrt(2 * math.pi) * bw) * math.exp(tsd ** 2 / (2 * bw ** 2))
        _expect(_cell(g, -0.5, y), True, tsd, weight)


# ---- normal_estimation_2d_test.cc ----
def _normalize(d):
    while d > math.pi:
        d -= 2 * math.pi
    while d < -math.pi:
        d += 2 * math.pi
    return d


def _circle(num_angles=100):
    angles = [i / num_angles * 2.0 * math.pi - math.pi for i in range(num_angles)]
    return angles, np.float32([[math.cos(a), math.sin(a), 0.0] for a in angles])


def test_normal_estimation_single_point():
    angles, pts = _circle()
    for a, p in zip(angles, pts):
        n = O.estimate_normals(p[None], [0, 0, 0], 2, 10.0)[0]
        assert abs(_normalize(a - float(n) - math.pi)) < 2.0 * math.pi / 100 + 1e-4


@pytest.mark.parametrize("points,want", [
    ([[-1, 1, 0], [0, 1, 0], [1, 1, 0]], -math.pi / 2),
    ([[1, 1, 0], [1, 0, 0], [1, -1, 0]], math.pi),
    ([[1, -1, 0], [0, -1, 0], [-1, -1, 0]], math.pi / 2),
    ([[-1, -1, 0], [-1, 0, 0], [-1, 1, 0]], 0.0),
])
def test_normal_estimation_straight_line_geometry(points, want):
    for n in O.estimate_normals(np.float32(points), [0, 0, 0], 2, 10.0):
        if want == math.pi:
            assert abs(abs(float(n)) - math.pi) < 1e-4
        else:
            assert abs(float(n) - want) < 1e-4


@pytest.mark.parametrize("num_samples", [1, 2, 4, 5, 8])
def test_normal_estimation_circular_geometry(num_samples):
    _, pts = _circle()
    normals = O.estimate_normals(pts, [0, 0, 0], num_samples, 10.0)
    for i, n in enumerate(normals):
        angle = i / 100 * 2.0 * math.pi
        assert abs(_normalize(float(n) - angle)) < 2.0 * math.pi / 100 * num_samples / 2.0 + 1e-4


# ---- against the numpy fixture builder ----
def _fixture_scan(seed, n=240):
    """Returns on a noisy closed contour around the origin: distinct directions, inside a
    200 x 200 grid of 0.05 m with room for the truncation band."""
    rng = np.random.RandomState(seed)
    angles = np.sort(rng.uniform(-math.pi, math.pi, n))
    angles = angles[np.concatenate([[True], np.diff(angles) > 1e-3])]
    radius = 2.0 + 0.8 * np.sin(3 * angles + seed) + rng.uniform(-0.05, 0.05, len(angles))
    origin = np.float32([0.013 * seed, -0.021 * seed, 0])
    pts = np.stack([origin[0] + radius * np.cos(angles), origin[1] + radius * np.sin(angles),
                    np.zeros(len(angles))], 1).astype(np.float32)
    return origin, pts


# Where the numpy fixture builder departs from the reference, in double where the reference is
# float.  The builder stays as it is (the cost-function fixtures use it); the comparison gives it
# the reference's float steps instead:
#   * the normal (NormalTo2DAngle) and the angle between normal and ray call the float overload
#     of std::atan2 (common::atan2 -> ceres::atan2);
#   * GaussianKernel's kSqrtTwoPi is a float, and kSqrtTwoPi * sigma a float product.
# The builder also wraps that angle by 2 pi in double where NormalizeAngleDifference<float> rounds
# to float after each step, so the fixtures with angle weighting keep their rays away from the +x
# direction, where the angle wraps.
_atan2f = C.CDLL(None).atan2f
_atan2f.restype = C.c_float
_atan2f.argtypes = [C.c_float, C.c_float]


class _FloatAtan2:
    def __getattr__(self, name):
        return getattr(math, name)

    @staticmethod
    def atan2(y, x):
        return _atan2f(float(y), float(x))


def _float_gaussian(x, sigma):
    s = np.float32(np.float32(math.sqrt(2.0 * math.pi)) * np.float32(sigma))
    s2 = np.float32(np.float32(sigma) * np.float32(sigma))
    return np.float32(1.0 / float(s) * math.exp(-0.5 * float(x) * float(x) / float(s2)))


@pytest.mark.parametrize("angle_weight", [False, True])
@pytest.mark.parametrize("variant", ["defaults", "free_space", "exponent1", "exponent2",
                                     "no_projection"])
def test_equals_the_numpy_fixture_builder(variant, angle_weight, monkeypatch):
    kw = {"defaults": {}, "free_space": dict(update_free_space=True),
          "exponent1": dict(update_weight_range_exponent=1),
          "exponent2": dict(update_weight_range_exponent=2),
          "no_projection": dict(project_sdf_distance_to_scan_normal=False)}[variant]
    monkeypatch.setattr(tsdf_inserter, "_gaussian", _float_gaussian)
    if angle_weight:
        monkeypatch.setattr(tsdf_inserter, "math", _FloatAtan2())
    else:
        kw["update_weight_angle_scan_normal_to_ray_kernel_bandwidth"] = 0.0
    opts = _Opts(**kw)
    res, max_x, max_y, n = 0.05, 5.0, 5.0, 200
    ora = O.TsdfGrid(res, max_x, max_y, n, n, 0.3, 10.0)
    npy = tsdf2d_oracle.TSDF2D(n, n, res, max_x, max_y, 0.3, 10.0)
    ins = O.TsdfInserter(opts)
    for seed in range(3):
        origin, pts = _fixture_scan(seed)
        if angle_weight:
            pts = pts[np.abs(np.arctan2(pts[:, 1] - origin[1], pts[:, 0] - origin[0])) > 0.3]
        assert ins.insert(origin, pts, ora)
        tsdf_inserter.insert(npy, origin[:2], list(pts), opts)
        t, w = ora.arrays()
        assert ora.limits == (res, max_x, max_y, n, n)
        np.testing.assert_array_equal(t, npy.tsd_cells)
        np.testing.assert_array_equal(w, npy.weight_cells)


def test_refused_inserts_leave_the_restated_grid_unchanged():
    ins = O.TsdfInserter(_Opts())
    g = O.TsdfGrid.create_grid([0, 0], 0.05)
    origin, pts = _fixture_scan(1)
    assert ins.insert(origin, pts, g)
    before = (g.limits, g.known_box) + g.arrays()
    res, max_x, max_y, nx, ny = g.limits
    centre = np.float32([max_x - 0.5 * ny * res, max_y - 0.5 * nx * res, 0])
    # a steep return near the edge: the growth, along the 3D ray, stays inside the grid, the
    # truncation band along the 2D ray does not
    assert not ins.insert(centre, np.float32([[max_x - 0.1, centre[1], 40.0]]), g)
    assert not ins.insert(centre, np.float32([[1.0e4, 0, 0]]), g)   # past 30000 cells
    after = (g.limits, g.known_box) + g.arrays()
    assert before[:2] == after[:2]
    for a, b in zip(before[2:], after[2:]):
        np.testing.assert_array_equal(a, b)


# ---- the C ABI without a device ----
@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def test_record_layout(csm):
    from cartographer_b200 import scan_matching as sm
    ctype, cname = sm.CsmTsdfInserterOptions2D, "csm_tsdf_inserter_options2d"
    head = '#include <stdio.h>\n#include <stddef.h>\n#include "include/csm_abi.h"\nint main(){'
    body = 'printf("%%zu\\n", sizeof(%s));' % cname + "".join(
        'printf("%%zu\\n", offsetof(%s, %s));' % (cname, f) for f, _ in ctype._fields_)
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(head + body + "}")
        subprocess.check_call(["gcc", "-I", ROOT, os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        got = [int(v) for v in subprocess.check_output([os.path.join(d, "t")]).split()]
    assert got == [C.sizeof(ctype)] + [getattr(ctype, f).offset for f, _ in ctype._fields_]
    assert got[0] == 56


def test_symbols_are_exported(csm):
    out = subprocess.check_output(["nm", "-D", "--defined-only", csm.SO_PATH], text=True)
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for sym in ("csm_tsdf_inserter2d_create", "csm_tsdf_inserter2d_destroy",
                "csm_tsdf_inserter2d_insert", "csm_rt_grid2d_create_empty_tsdf",
                "csm_rt_grid2d_read_weights"):
        assert sym in names, sym


def test_invalid_calls_and_no_device(csm):
    from cartographer_b200 import scan_matching as sm
    lib = csm.lib()
    out = C.c_void_p()
    for bad in (dict(num_normal_samples=0), dict(sample_radius=0.0), dict(sample_radius=-1.0),
                dict(truncation_distance=0.0), dict(truncation_distance=-0.3),
                dict(maximum_weight=0.0), dict(maximum_weight=-1.0)):
        o = sm.TSDFRangeDataInserterOptions2D(**bad)._c()
        assert lib.csm_tsdf_inserter2d_create(C.byref(o), 0, C.byref(out)) == 1, bad
    assert lib.csm_tsdf_inserter2d_create(None, 0, C.byref(out)) == 1
    assert lib.csm_tsdf_inserter2d_insert(None, None, None, 0, None, None) == 1
    assert lib.csm_tsdf_inserter2d_destroy(None) == 0
    assert lib.csm_rt_grid2d_read_weights(None, None, C.c_int64(0)) == 1
    d, f = C.c_double, C.c_float
    for args in ((d(0.0), d(1.0), d(1.0), 100, 100, f(0.3), f(10.0)),
                 (d(0.05), d(1.0), d(1.0), 30000, 100, f(0.3), f(10.0)),
                 (d(0.05), d(1.0), d(1.0), 100, 100, f(0.0), f(10.0)),
                 (d(0.05), d(1.0), d(1.0), 100, 100, f(0.3), f(0.0))):
        assert lib.csm_rt_grid2d_create_empty_tsdf(*args, 0, C.byref(out)) == 1, args
    count = C.c_int32(0)
    if lib.csm_device_count(C.byref(count)) == 0 and count.value > 0:
        pytest.skip("GPU present")
    o = sm.TSDFRangeDataInserterOptions2D()._c()
    assert lib.csm_tsdf_inserter2d_create(C.byref(o), 0, C.byref(out)) == 2, "expected CSM_E_CUDA"
    assert lib.csm_rt_grid2d_create_empty_tsdf(d(0.05), d(1.0), d(1.0), 100, 100, f(0.3), f(10.0),
                                               0, C.byref(out)) == 2
