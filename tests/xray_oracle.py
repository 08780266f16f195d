"""ctypes loader of the CPU restatement of XRayPointsProcessor (tests/xray_oracle.cc): the parity
reference of the device processor and the host column of benchmarks/bench_xray.py.  The library
is compiled on first use into a temporary directory, so that nothing is written into the tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "xray_oracle.cc")

IDENTITY = (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="xray_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libxray_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.xo_create.restype = vp
        L.xo_create.argtypes = [C.c_double, C.c_double, vp, C.c_int]
        L.xo_destroy.argtypes = [vp]
        L.xo_insert.argtypes = [vp, C.c_int, vp, vp, C.c_int]
        L.xo_box.argtypes = [vp, vp, vp]
        L.xo_channel.argtypes = [C.c_float, C.c_float]
        L.xo_draw.argtypes = [vp, C.c_int, vp, vp, vp]
        L.xo_voxels.restype = C.c_longlong
        L.xo_voxels.argtypes = [vp, C.c_int, vp]
        L.xo_columns.restype = C.c_longlong
        L.xo_columns.argtypes = [vp, C.c_int, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f3(a):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, 3))


class Processor:
    """The aggregations and shared box of one XRayPointsProcessor.  insert returns False,
    changing nothing, where the reference would abort (a cell outside the grid's
    [-8192, 8192)^3)."""

    def __init__(self, voxel_size, saturation_factor=1.0, transform=IDENTITY,
                 num_aggregations=1):
        t = np.asarray(transform, np.float32).reshape(7)
        self.h = lib().xo_create(voxel_size, saturation_factor, _p(t), num_aggregations)

    def __del__(self):
        if getattr(self, "h", None):
            lib().xo_destroy(self.h)
            self.h = None

    def insert(self, points, colors=None, aggregation=0):
        pts = _f3(points)
        rgb = None if colors is None else _f3(colors)
        return lib().xo_insert(self.h, aggregation, _p(pts), None if rgb is None else _p(rgb),
                               len(pts)) == 0

    def bounding_box(self):
        """(min (3,), max (3,), empty)."""
        lo, hi = np.zeros(3, np.int32), np.zeros(3, np.int32)
        empty = lib().xo_box(self.h, _p(lo), _p(hi))
        return lo, hi, bool(empty)

    def draw(self, aggregation=0):
        """The cairo words as a (height, width) uint32 array, or None for an empty box."""
        w, ht = C.c_int(), C.c_int()
        if lib().xo_draw(self.h, aggregation, None, C.byref(w), C.byref(ht)) < 0:
            return None
        px = np.zeros(max(w.value * ht.value, 1), np.uint32)
        lib().xo_draw(self.h, aggregation, _p(px), C.byref(w), C.byref(ht))
        return px[:w.value * ht.value].reshape(ht.value, w.value)

    def voxels(self, aggregation=0):
        """(n, 3) cell indices in ascending (z, y, x)."""
        n = lib().xo_voxels(self.h, aggregation, None)
        idx = np.zeros((max(n, 1), 3), np.int32)
        lib().xo_voxels(self.h, aggregation, _p(idx))
        idx = idx[:n]
        return idx[np.lexsort((idx[:, 0], idx[:, 1], idx[:, 2]))]

    def columns(self, aggregation=0):
        """(yz (n, 2), sums (n, 3) float32, counts (n,) uint32) in ascending (y, z)."""
        n = lib().xo_columns(self.h, aggregation, None, None, None)
        m = max(n, 1)
        yz, sums, counts = np.zeros((m, 2), np.int32), np.zeros((m, 3), np.float32), \
            np.zeros(m, np.uint32)
        lib().xo_columns(self.h, aggregation, _p(yz), _p(sums), _p(counts))
        return yz[:n], sums[:n], counts[:n]


def channel(mean, saturation):
    """One byte of IntoImage: Mix(1.f, mean, saturation) clamped, scaled and rounded."""
    return lib().xo_channel(float(np.float32(mean)), float(np.float32(saturation)))
