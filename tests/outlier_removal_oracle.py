"""ctypes loader of the CPU restatement of OutlierRemovingPointsProcessor
(tests/outlier_removal_oracle.cc): the parity reference of the device processor and the host
column of benchmarks/bench_outlier_removal.py.  The library is compiled on first use into a
temporary directory, so that nothing is written into the tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "outlier_removal_oracle.cc")

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="outlier_removal_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "liboutlier_removal_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.oro_create.restype = vp
        L.oro_create.argtypes = [C.c_double, C.c_double]
        L.oro_destroy.argtypes = [vp]
        L.oro_add_hits.argtypes = [vp, vp, C.c_int]
        L.oro_ray_samples.restype = C.c_longlong
        L.oro_ray_samples.argtypes = [C.c_double, C.c_float, vp, C.c_longlong]
        L.oro_count_rays.restype = C.c_longlong
        L.oro_count_rays.argtypes = [vp, vp, vp, C.c_int]
        L.oro_filter.argtypes = [vp, vp, C.c_int, vp]
        L.oro_voxels.restype = C.c_longlong
        L.oro_voxels.argtypes = [vp, vp, vp, vp]
        L.oro_cell_index.argtypes = [C.c_float] * 4 + [vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _points(points):
    return np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))


class Processor:
    """One OutlierRemovingPointsProcessor's voxel map and its three phases, batch by batch.
    add_hits and count_rays return False, changing nothing, where the reference would abort
    (a hit outside the grid's [-8192, 8192)^3 voxels) or never return (a ray longer than where
    x += voxel_size stops growing)."""

    def __init__(self, voxel_size, miss_per_hit_limit=3.0):
        self.h = lib().oro_create(voxel_size, miss_per_hit_limit)

    def __del__(self):
        if getattr(self, "h", None):
            lib().oro_destroy(self.h)
            self.h = None

    def add_hits(self, points):
        pts = _points(points)
        return lib().oro_add_hits(self.h, _p(pts), len(pts)) == 0

    def count_rays(self, origin, points):
        pts = _points(points)
        o = np.ascontiguousarray(origin, np.float32).reshape(3)
        return lib().oro_count_rays(self.h, _p(o), _p(pts), len(pts)) >= 0

    def filter(self, points):
        """Kept indices, in input order."""
        pts = _points(points)
        kept = np.zeros(max(len(pts), 1), np.int32)
        n = lib().oro_filter(self.h, _p(pts), len(pts), _p(kept))
        return kept[:n].copy()

    def voxels(self):
        """(indices (n, 3), hits, rays) of every voxel with hits, in ascending (z, y, x)."""
        n = lib().oro_voxels(self.h, None, None, None)
        idx = np.zeros((max(n, 1), 3), np.int32)
        hits = np.zeros(max(n, 1), np.int32)
        rays = np.zeros(max(n, 1), np.int32)
        lib().oro_voxels(self.h, _p(idx), _p(hits), _p(rays))
        order = np.lexsort((idx[:n, 0], idx[:n, 1], idx[:n, 2]))
        return idx[:n][order], hits[:n][order], rays[:n][order]


def ray_samples(voxel_size, length, cap=1 << 20):
    """The x that `for (float x = 0; x < length; x += voxel_size)` visits (voxel_size a
    double), or None when x stops growing below length."""
    out = np.zeros(cap, np.float32)
    k = lib().oro_ray_samples(voxel_size, length, _p(out), cap)
    return None if k < 0 else out[:min(k, cap)].copy()


def cell_index(point, resolution):
    out = np.zeros(3, np.int32)
    lib().oro_cell_index(*[float(v) for v in np.float32(point)], resolution, _p(out))
    return tuple(int(v) for v in out)


def run(batches, voxel_size, miss_per_hit_limit=3.0):
    """The whole stream: batches are (origin, points) pairs.  Returns the voxels after phase 1
    and after phase 2 (as Processor.voxels) and the kept indices of every batch."""
    p = Processor(voxel_size, miss_per_hit_limit)
    for _, pts in batches:
        assert p.add_hits(pts)
    after_hits = p.voxels()
    for o, pts in batches:
        assert p.count_rays(o, pts)
    after_rays = p.voxels()
    return after_hits, after_rays, [p.filter(pts) for _, pts in batches]
