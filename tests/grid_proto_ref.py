"""Test-side references for saving device grids — TEST INFRASTRUCTURE ONLY.

* walk(): HybridGrid's iteration order from a restatement of its storage
  (tests/hybrid_grid_walk.cc: DynamicGrid -> NestedGrid -> FlatGrid, bits_ and Grow), compiled on
  first use into a temporary directory so that nothing is written into the tree.
* hybrid_grid_message() / grid2d_message(): proto::HybridGrid and proto::Grid2D as
  HybridGrid::ToProto (hybrid_grid.h:528-540) and Grid2D::ToProto plus ProbabilityGrid::ToProto /
  TSDF2D::ToProto (grid_2d.cc:166-183, probability_grid.cc:84-89, tsdf_2d.cc:107-116) fill them,
  serialised with the proto3 rules protobuf C++ applies: fields in field-number order, zero scalars
  omitted (a float or double only when its bit pattern is all zeros, so -0.0 is written), repeated
  scalars packed and omitted when empty, a present empty sub-message written with length 0.  Built
  from tests/protowire.py's field writers.
"""
import atexit
import ctypes as C
import os
import shutil
import struct
import subprocess
import tempfile

import numpy as np

from tests import protowire as pw

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hybrid_grid_walk.cc")
K_MIN_CORRESPONDENCE_COST = float(np.float32(1) - np.float32(np.float32(1) - np.float32(0.1)))
K_MAX_CORRESPONDENCE_COST = float(np.float32(1) - np.float32(0.1))

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="hybrid_grid_walk_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libhybrid_grid_walk.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.hgw_new.restype = vp
        L.hgw_free.argtypes = [vp]
        L.hgw_bits.argtypes = [vp]
        L.hgw_set.argtypes = [vp, vp, vp, C.c_int64]
        L.hgw_walk.restype = C.c_int64
        L.hgw_walk.argtypes = [vp, vp, vp, C.c_int64]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def walk(*writes):
    """Writes each (indices n x 3, values n) batch into a fresh HybridGrid in order
    (*mutable_value(index) = value), then iterates it: (indices, values, bits_)."""
    L = lib()
    g = L.hgw_new()
    try:
        for idx, val in writes:
            idx = np.ascontiguousarray(idx, np.int32).reshape(-1, 3)
            val = np.ascontiguousarray(val, np.uint16).reshape(-1)
            L.hgw_set(g, _p(idx), _p(val), len(val))
        n = L.hgw_walk(g, None, None, 0)
        idx = np.zeros((n, 3), np.int32)
        val = np.zeros(n, np.uint16)
        L.hgw_walk(g, _p(idx), _p(val), n)
        return idx, val, L.hgw_bits(g)
    finally:
        L.hgw_free(g)


def _float_present(v, fmt):
    return struct.pack(fmt, v) != b"\0" * struct.calcsize(fmt)


def f_float(field, v):
    return pw.f_float(field, v) if _float_present(v, "<f") else b""


def f_double(field, v):
    return pw.f_double(field, v) if _float_present(v, "<d") else b""


def f_int32(field, v):
    return pw.f_varint(field, int(v)) if v else b""


def packed_varints(values):
    """The payload of a packed repeated field of non-negative integers below 2^21 (vectorised
    form of b"".join(protowire.varint(v) for v in values))."""
    v = np.asarray(values, np.int64).reshape(-1)
    assert v.size == 0 or (v.min() >= 0 and v.max() < 1 << 21)
    n = 1 + (v >= 1 << 7) + (v >= 1 << 14)
    out = np.zeros((v.size, 3), np.uint8)
    out[:, 0] = (v & 0x7F) | np.where(n > 1, 0x80, 0)
    out[:, 1] = ((v >> 7) & 0x7F) | np.where(n > 2, 0x80, 0)
    out[:, 2] = (v >> 14) & 0x7F
    keep = np.arange(3)[None, :] < n[:, None]
    return out[keep].tobytes()


def hybrid_grid_message(resolution, indices, values):
    """HybridGrid::ToProto of the voxel list (already in iteration order): for a non-empty list
    the bytes of protowire.hybrid_grid, vectorised; for an empty one the resolution alone."""
    if len(values) == 0:
        return f_float(1, resolution)
    idx = np.asarray(indices, np.int64).reshape(-1, 3)
    zz = (idx << 1) ^ (idx >> 63)
    return (pw.f_float(1, resolution) +
            b"".join(pw.f_bytes(3 + a, packed_varints(zz[:, a])) for a in range(3)) +
            pw.f_bytes(6, packed_varints(values)))


def grid2d_message(cells, resolution, max_x, max_y, known_cells_box=None, weight_cells=None,
                   truncation_distance=None, max_weight=None):
    """ProbabilityGrid::ToProto (weight_cells None) or TSDF2D::ToProto of a grid of cells[y, x];
    known_cells_box is (min_x, min_y, max_x, max_y) or None when empty."""
    ny, nx = cells.shape
    limits = (f_double(1, resolution) + pw.f_bytes(2, f_double(1, max_x) + f_double(2, max_y)) +
              pw.f_bytes(3, f_int32(1, nx) + f_int32(2, ny)))
    msg = pw.f_bytes(1, limits) + pw.f_bytes(2, packed_varints(cells))
    if known_cells_box is not None:
        mn_x, mn_y, mx_x, mx_y = known_cells_box
        msg += pw.f_bytes(3, f_int32(1, mx_x) + f_int32(2, mx_y) + f_int32(3, mn_x) +
                          f_int32(4, mn_y))
    if weight_cells is None:
        msg += pw.f_bytes(4, b"")
        lo, hi = K_MIN_CORRESPONDENCE_COST, K_MAX_CORRESPONDENCE_COST
    else:
        t = float(np.float32(truncation_distance))
        msg += pw.f_bytes(5, f_float(1, t) + f_float(2, max_weight) +
                          pw.f_bytes(3, packed_varints(weight_cells)))
        lo, hi = -t, t
    return msg + f_float(6, lo) + f_float(7, hi)
