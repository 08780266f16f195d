"""ctypes loader of the CPU restatement of TSDFRangeDataInserter2D, TSDF2D and
NormalEstimation2D (tests/insert_tsdf2d_oracle.cc): the parity reference of the device TSDF
inserter and the CPU column of benchmarks/bench_insert_tsdf2d.py.  The library is compiled on
first use into a temporary directory, so that nothing is written into the tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "insert_tsdf2d_oracle.cc")

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="insert_tsdf2d_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libinsert_tsdf2d_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.i2t_grid_new.restype = vp
        L.i2t_grid_new.argtypes = [C.c_double] * 3 + [C.c_int] * 2 + [C.c_float] * 2 + [vp, vp]
        L.i2t_grid_free.argtypes = [vp]
        L.i2t_grid_info.argtypes = [vp, vp, vp]
        L.i2t_grid_cells.argtypes = [vp, vp, vp]
        L.i2t_grid_get.argtypes = [vp, C.c_int, C.c_int, vp]
        L.i2t_grid_cell_index.argtypes = [vp, C.c_float, C.c_float, vp]
        L.i2t_inserter_new.restype = vp
        L.i2t_inserter_new.argtypes = [vp]
        L.i2t_inserter_free.argtypes = [vp]
        L.i2t_insert.argtypes = [vp, vp, vp, vp, C.c_int]
        L.i2t_estimate_normals.argtypes = [vp, C.c_int, vp, C.c_int, C.c_float, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class TsdfGrid:
    """A TSDF2D: limits, tsd and weight cells[y, x], the converter and the known-cells box."""

    def __init__(self, resolution, max_x, max_y, num_x, num_y, truncation, max_weight,
                 tsd_cells=None, weight_cells=None):
        t = w = None
        if tsd_cells is not None:
            self._tsd = np.ascontiguousarray(tsd_cells, np.uint16)
            self._w = np.ascontiguousarray(weight_cells, np.uint16)
            assert self._tsd.shape == self._w.shape == (num_y, num_x)
            t, w = _p(self._tsd), _p(self._w)
        self.truncation, self.max_weight = float(truncation), float(max_weight)
        self._h = lib().i2t_grid_new(resolution, max_x, max_y, num_x, num_y, truncation,
                                     max_weight, t, w)

    @classmethod
    def create_grid(cls, origin, resolution, truncation=0.3, max_weight=10.0):
        """ActiveSubmaps2D::CreateGrid for GridType::TSDF: 100 x 100 cells around origin."""
        r = float(np.float32(resolution))
        o = np.asarray(origin, np.float32).astype(np.float64)
        return cls(r, o[0] + 0.5 * 100 * r, o[1] + 0.5 * 100 * r, 100, 100, truncation, max_weight)

    @property
    def limits(self):
        """(resolution, max_x, max_y, num_x, num_y)"""
        lim, ints = np.zeros(3), np.zeros(7, np.int32)
        lib().i2t_grid_info(self._h, _p(lim), _p(ints))
        return (float(lim[0]), float(lim[1]), float(lim[2]), int(ints[0]), int(ints[1]))

    @property
    def known_box(self):
        lim, ints = np.zeros(3), np.zeros(7, np.int32)
        lib().i2t_grid_info(self._h, _p(lim), _p(ints))
        return None if ints[2] else tuple(int(v) for v in ints[3:7])

    def arrays(self):
        """(tsd cells, weight cells), each [num_y, num_x]"""
        _, _, _, nx, ny = self.limits
        t, w = np.zeros((ny, nx), np.uint16), np.zeros((ny, nx), np.uint16)
        lib().i2t_grid_cells(self._h, _p(t), _p(w))
        return t, w

    def get(self, x, y):
        """(IsKnown, GetTSD, GetWeight) of cell (x, y)"""
        out = np.zeros(3, np.float32)
        lib().i2t_grid_get(self._h, int(x), int(y), _p(out))
        return bool(out[0]), float(out[1]), float(out[2])

    def cell_index(self, px, py):
        out = np.zeros(2, np.int32)
        lib().i2t_grid_cell_index(self._h, float(px), float(py), _p(out))
        return int(out[0]), int(out[1])

    def close(self):
        if getattr(self, "_h", None):
            lib().i2t_grid_free(self._h)
            self._h = None

    __del__ = close


class TsdfInserter:
    """TSDFRangeDataInserter2D(options); options has the fields of
    cartographer_b200.scan_matching.TSDFRangeDataInserterOptions2D."""

    def __init__(self, options):
        o = options
        v = np.array([o.truncation_distance, o.maximum_weight, float(bool(o.update_free_space)),
                      o.num_normal_samples, o.sample_radius,
                      float(bool(o.project_sdf_distance_to_scan_normal)),
                      o.update_weight_range_exponent,
                      o.update_weight_angle_scan_normal_to_ray_kernel_bandwidth,
                      o.update_weight_distance_cell_to_hit_kernel_bandwidth], np.float64)
        self._h = lib().i2t_inserter_new(_p(v))

    def insert(self, origin, returns, grid):
        """Insert + FinishUpdate; False (grid unchanged) where the device refuses the insert."""
        o = np.ascontiguousarray(origin, np.float32).reshape(3)
        r = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
        return bool(lib().i2t_insert(self._h, grid._h, _p(o), _p(r), len(r)))

    def close(self):
        if getattr(self, "_h", None):
            lib().i2t_inserter_free(self._h)
            self._h = None

    __del__ = close


def estimate_normals(returns, origin, num_normal_samples, sample_radius):
    """NormalEstimation2D::EstimateNormals over returns in the given order."""
    r = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
    o = np.ascontiguousarray(origin, np.float32).reshape(3)
    out = np.zeros(len(r), np.float32)
    lib().i2t_estimate_normals(_p(r), len(r), _p(o), int(num_normal_samples), float(sample_radius),
                               _p(out))
    return out
