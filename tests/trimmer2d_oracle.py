"""ctypes loader of the CPU restatement of OverlappingSubmapsTrimmer2D's coverage pass
(tests/trimmer2d_oracle.cc), used by the tests and as the CPU column of
benchmarks/bench_trimmer2d.py.  The library is compiled on first use into a temporary directory,
so that nothing is written into the tree.

A submap is (cells, known_box, limits, pose, freshness): cells[y, x] (uint16, 0 = unknown), the
known-cells box (min_x, min_y, max_x, max_y) or None when it is empty, limits (max_x, max_y,
resolution), global_frame_from_local_frame (tx, ty, tz, qw, qx, qy, qz) and the freshness ticks."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "trimmer2d_oracle.cc")

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="trimmer2d_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libtrimmer2d_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.tro_trim.restype = None
        L.tro_trim.argtypes = [C.c_int32, vp, vp, vp, vp, vp, vp, C.c_double, C.c_double,
                               C.c_double, C.c_uint16, C.c_uint16, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def cropped_limits(known_box):
    """Grid2D::ComputeCroppedLimits: (offset x, offset y, num_x, num_y), 1 x 1 at 0 if empty."""
    if known_box is None:
        return (0, 0, 1, 1)
    x0, y0, x1, y1 = known_box
    return (x0, y0, x1 - x0 + 1, y1 - y0 + 1)


def trim(submaps, first_limits, fresh_submaps_count, min_covered_cells_count):
    """(trim flags, covered entries per submap before the uint16 wrap, stats) as the reference's
    AddSubmapsToSubmapCoverageGrid2D + FindSubmapIdsToTrim compute them.  stats: entries,
    coverage_cells and sorted_large (cells whose cut std::sort'ed more than 16 entries)."""
    n = len(submaps)
    cells = [np.ascontiguousarray(s[0], np.uint16) for s in submaps]
    ptrs = (C.c_void_p * max(n, 1))(*[c.ctypes.data for c in cells])
    num_x = np.array([c.shape[1] for c in cells] or [0], np.int32)
    box = np.array([cropped_limits(s[1]) for s in submaps] or [(0, 0, 0, 0)], np.int32)
    limits = np.array([s[2] for s in submaps] or [(0, 0, 1)], np.float64)
    poses = np.array([np.asarray(s[3], np.float64).reshape(7) for s in submaps] or
                     [np.zeros(7)], np.float64)
    freshness = np.array([int(s[4]) for s in submaps] or [0], np.int64)
    out_trim = np.zeros(max(n, 1), np.uint8)
    counts = np.zeros(max(n, 1), np.uint32)
    stats = np.zeros(3, np.int64)
    lib().tro_trim(n, C.cast(ptrs, C.c_void_p), _p(num_x), _p(box), _p(limits), _p(poses),
                   _p(freshness), first_limits[0], first_limits[1], first_limits[2],
                   fresh_submaps_count, min_covered_cells_count, _p(out_trim), _p(counts),
                   _p(stats))
    return (out_trim[:n].astype(bool), counts[:n],
            {"entries": int(stats[0]), "coverage_cells": int(stats[1]),
             "sorted_large": int(stats[2])})
