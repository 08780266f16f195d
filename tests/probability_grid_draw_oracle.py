"""ctypes loader of the CPU restatement of io::DrawProbabilityGrid
(tests/probability_grid_draw_oracle.cc): the parity reference of csm_rt_grid2d_draw.  The library
is compiled on first use into a temporary directory, so that nothing is written into the tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "probability_grid_draw_oracle.cc")

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="probability_grid_draw_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libprobability_grid_draw_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.pgd_grey.argtypes = [C.c_int]
        L.pgd_scaled.restype = C.c_float
        L.pgd_scaled.argtypes = [C.c_int]
        L.pgd_draw.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def grey(value):
    return lib().pgd_grey(int(value))


def scaled(value):
    """255 * ((1 - GetProbability) - kMin) / (kMax - kMin) in float, before RoundToInt."""
    return np.float32(lib().pgd_scaled(int(value)))


def draw(cells, known_cells_box):
    """(pixels (height, width) uint32, (offset x, offset y)) of a grid of cells[y, x] whose
    known-cells box is (min_x, min_y, max_x, max_y), or None when empty."""
    cells = np.ascontiguousarray(cells, np.uint16)
    box = None if known_cells_box is None else np.asarray(known_cells_box, np.int32)
    out = np.zeros(4, np.int32)
    lib().pgd_draw(_p(cells), cells.shape[1], cells.shape[0],
                   None if box is None else _p(box), _p(out), None)
    pixels = np.zeros((out[1], out[0]), np.uint32)
    lib().pgd_draw(_p(cells), cells.shape[1], cells.shape[0],
                   None if box is None else _p(box), _p(out), _p(pixels))
    return pixels, (int(out[2]), int(out[3]))
