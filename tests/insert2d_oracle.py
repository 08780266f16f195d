"""ctypes loader of the CPU restatement of ProbabilityGridRangeDataInserter2D
(tests/insert2d_oracle.cc): the parity reference of the device inserter and the CPU column of
benchmarks/bench_insert2d.py.  The library is compiled on first use into a temporary
directory, so that nothing is written into the tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "insert2d_oracle.cc")
VALUE_COUNT = 32768
UPDATE_MARKER = 1 << 15

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="insert2d_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libinsert2d_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.i2d_grid_new.restype = vp
        L.i2d_grid_new.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, vp]
        L.i2d_grid_free.argtypes = [vp]
        L.i2d_grid_info.argtypes = [vp, vp, vp]
        L.i2d_grid_cells.argtypes = [vp, vp]
        L.i2d_grid_get_probability.restype = C.c_float
        L.i2d_grid_get_probability.argtypes = [vp, C.c_int, C.c_int]
        L.i2d_grid_set_probability.argtypes = [vp, C.c_int, C.c_int, C.c_float]
        L.i2d_grid_apply_odds.argtypes = [vp, C.c_int, C.c_int, C.c_float]
        L.i2d_grid_finish_update.argtypes = [vp]
        L.i2d_grid_cell_index.argtypes = [vp, C.c_float, C.c_float, vp]
        L.i2d_grid_crop.restype = vp
        L.i2d_grid_crop.argtypes = [vp]
        L.i2d_inserter_new.restype = vp
        L.i2d_inserter_new.argtypes = [C.c_double, C.c_double, C.c_int]
        L.i2d_inserter_free.argtypes = [vp]
        L.i2d_inserter_tables.argtypes = [vp, vp, vp]
        L.i2d_insert.argtypes = [vp, vp, vp, vp, C.c_int, vp, C.c_int]
        L.i2d_ray_to_pixel_mask.argtypes = [C.c_int] * 5 + [vp, C.c_int]
        L.i2d_crop_table.argtypes = [vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Grid:
    """A ProbabilityGrid: limits, correspondence-cost cells[y, x] and the known-cells box."""

    def __init__(self, resolution, max_x, max_y, num_x, num_y, cells=None, _handle=None):
        if _handle is not None:
            self._h = _handle
            return
        c = None
        if cells is not None:
            cells = np.ascontiguousarray(cells, np.uint16)
            assert cells.shape == (num_y, num_x)
            c = _p(cells)
        self._h = lib().i2d_grid_new(resolution, max_x, max_y, num_x, num_y, c)

    @classmethod
    def create_grid(cls, origin, resolution):
        """ActiveSubmaps2D::CreateGrid (submap_2d.cc:192-204): 100 x 100 cells around origin;
        resolution is the float option."""
        r = float(np.float32(resolution))
        o = np.asarray(origin, np.float32).astype(np.float64)
        return cls(r, o[0] + 0.5 * 100 * r, o[1] + 0.5 * 100 * r, 100, 100)

    def info(self):
        lim, ints = np.zeros(3), np.zeros(7, np.int32)
        lib().i2d_grid_info(self._h, _p(lim), _p(ints))
        return lim, ints

    @property
    def limits(self):
        """(resolution, max_x, max_y, num_x, num_y)"""
        lim, ints = self.info()
        return (float(lim[0]), float(lim[1]), float(lim[2]), int(ints[0]), int(ints[1]))

    @property
    def known_box(self):
        """None if empty, else (min_x, min_y, max_x, max_y)."""
        _, ints = self.info()
        return None if ints[2] else tuple(int(v) for v in ints[3:7])

    @property
    def cells(self):
        _, ints = self.info()
        out = np.zeros((ints[1], ints[0]), np.uint16)
        lib().i2d_grid_cells(self._h, _p(out))
        return out

    def get_probability(self, x, y):
        return lib().i2d_grid_get_probability(self._h, int(x), int(y))

    def set_probability(self, x, y, p):
        assert lib().i2d_grid_set_probability(self._h, int(x), int(y), float(p)) == 1

    def apply_odds(self, x, y, odds):
        return bool(lib().i2d_grid_apply_odds(self._h, int(x), int(y), float(odds)))

    def finish_update(self):
        lib().i2d_grid_finish_update(self._h)

    def cell_index(self, px, py):
        out = np.zeros(2, np.int32)
        lib().i2d_grid_cell_index(self._h, float(px), float(py), _p(out))
        return int(out[0]), int(out[1])

    def crop(self):
        return Grid(0, 0, 0, 0, 0, _handle=lib().i2d_grid_crop(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().i2d_grid_free(self._h)
            self._h = None

    __del__ = close


class Inserter:
    """ProbabilityGridRangeDataInserter2D(options)."""

    def __init__(self, hit_probability, miss_probability, insert_free_space=True):
        self._h = lib().i2d_inserter_new(hit_probability, miss_probability,
                                         1 if insert_free_space else 0)

    def tables(self):
        hit, miss = np.zeros(VALUE_COUNT, np.uint16), np.zeros(VALUE_COUNT, np.uint16)
        lib().i2d_inserter_tables(self._h, _p(hit), _p(miss))
        return hit, miss

    def insert(self, origin, returns, grid, misses=None):
        o = np.ascontiguousarray(origin, np.float32).reshape(3)
        r = np.ascontiguousarray(returns, np.float32).reshape(-1, 3)
        m = np.ascontiguousarray(np.zeros((0, 3)) if misses is None else misses,
                                 np.float32).reshape(-1, 3)
        lib().i2d_insert(self._h, grid._h, _p(o), _p(r), len(r), _p(m), len(m))

    def close(self):
        if getattr(self, "_h", None):
            lib().i2d_inserter_free(self._h)
            self._h = None

    __del__ = close


def ray_to_pixel_mask(begin, end, subpixel_scale):
    """RayToPixelMask: list of (x, y) pixels in the reference's order."""
    cap = abs(end[0] - begin[0]) // subpixel_scale + abs(end[1] - begin[1]) // subpixel_scale + 4
    out = np.zeros(2 * cap, np.int32)
    n = lib().i2d_ray_to_pixel_mask(int(begin[0]), int(begin[1]), int(end[0]), int(end[1]),
                                    int(subpixel_scale), _p(out), cap)
    assert n <= cap
    return [(int(out[2 * i]), int(out[2 * i + 1])) for i in range(n)]


def crop_table():
    out = np.zeros(VALUE_COUNT, np.uint16)
    lib().i2d_crop_table(_p(out))
    return out
