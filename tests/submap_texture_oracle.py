"""ctypes loader of the CPU restatement of the submap textures (tests/submap_texture_oracle.cc),
the message encoder and decoder the tests compare with, and the host route of
benchmarks/bench_submap_texture.py.  The library is compiled on first use into a temporary
directory, so that nothing is written into the tree.

A texture is a dict: cells (the raw value / alpha bytes, before gzip), width, height, resolution
and slice_pose (tx, ty, tz, qw, qx, qy, qz)."""
import atexit
import ctypes as C
import os
import shutil
import struct
import subprocess
import tempfile
import zlib

import numpy as np

from tests import protowire as pw

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "submap_texture_oracle.cc")

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="submap_texture_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libsubmap_texture_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so, "-lz"])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.sto_log_odds_integer.argtypes = [C.c_float]
        L.sto_log_odds_from_steps.argtypes = [C.c_float]
        L.sto_steps.argtypes = [vp]
        L.sto_log_odds_exhaustive.restype = C.c_int64
        L.sto_log_odds_exhaustive.argtypes = [vp, vp]
        L.sto_texture3d.restype = C.c_int64
        L.sto_texture3d.argtypes = [vp, vp, C.c_int64, C.c_float, vp, vp, C.c_int64, vp, vp, vp]
        L.sto_texture2d.restype = C.c_int64
        L.sto_texture2d.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, C.c_double, C.c_double,
                                    C.c_double, C.c_float, C.c_float, vp, vp, C.c_int64, vp, vp,
                                    vp]
        L.sto_zlib_version.restype = C.c_char_p
        L.sto_gzip.restype = C.c_int64
        L.sto_gzip.argtypes = [vp, C.c_int64, vp, C.c_int64]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _pose(pose):
    return np.ascontiguousarray(pose, np.float64).reshape(7)


def log_odds_integer(p):
    return lib().sto_log_odds_integer(p)


def log_odds_from_steps(p):
    return lib().sto_log_odds_from_steps(p)


def steps():
    out = np.zeros(254, np.float32)
    lib().sto_steps(_p(out))
    return out


def log_odds_exhaustive():
    """(floats checked, mismatches, first mismatching float or None)."""
    checked = np.zeros(1, np.int64)
    first = np.zeros(1, np.float32)
    bad = lib().sto_log_odds_exhaustive(_p(checked), _p(first))
    return int(checked[0]), int(bad), (float(first[0]) if bad else None)


def _finish(n, buf, w, h, slice_, resolution):
    assert n >= 0
    return dict(cells=buf[:n].tobytes(), width=int(w[0]), height=int(h[0]),
                resolution=float(resolution), slice_pose=tuple(float(v) for v in slice_))


def texture3d(indices, values, resolution, global_submap_pose):
    """AddToTextureProto's texture of the voxels (n x 3 indices, n values) listed in HybridGrid's
    iteration order, under the global submap pose."""
    idx = np.ascontiguousarray(indices, np.int32).reshape(-1, 3)
    val = np.ascontiguousarray(values, np.uint16).reshape(-1)
    w, h = np.zeros(1, np.int32), np.zeros(1, np.int32)
    slice_ = np.zeros(7, np.float64)
    pose = _pose(global_submap_pose)
    cap = 1 << 16
    while True:
        buf = np.zeros(cap, np.uint8)
        n = lib().sto_texture3d(_p(idx), _p(val), len(val), resolution, _p(pose), _p(buf), cap,
                                _p(w), _p(h), _p(slice_))
        if n >= 0:
            return _finish(n, buf, w, h, slice_, np.float32(resolution))
        cap = 2 * int(w[0]) * int(h[0])


def texture2d(cells, resolution, max_x, max_y, known_cells_box, local_pose, weight_cells=None,
              truncation=0.0, max_weight=0.0):
    """DrawToSubmapTexture of a ProbabilityGrid (cells[y, x] correspondence-cost values) or, with
    weight_cells, a TSDF2D (cells are its tsd values) with that converter; known_cells_box is
    (min_x, min_y, max_x, max_y) or None."""
    c = np.ascontiguousarray(cells, np.uint16)
    wc = None if weight_cells is None else np.ascontiguousarray(weight_cells, np.uint16)
    box = np.array(known_cells_box if known_cells_box is not None else (1, 1, 0, 0), np.int32)
    w, h = np.zeros(1, np.int32), np.zeros(1, np.int32)
    slice_ = np.zeros(7, np.float64)
    pose = _pose(local_pose)
    cap = 2 * c.size + 2
    buf = np.zeros(cap, np.uint8)
    n = lib().sto_texture2d(_p(c), None if wc is None else _p(wc), c.shape[1], c.shape[0],
                            _p(box), resolution, max_x, max_y, truncation, max_weight, _p(pose),
                            _p(buf), cap, _p(w), _p(h), _p(slice_))
    return _finish(n, buf, w, h, slice_, resolution)


def zlib_version():
    """The zlib version the restatement (and so the library's gzip code) was compiled with."""
    return lib().sto_zlib_version().decode()


def library_gzip(data):
    """The library's gzip member (csrc/submap_texture.h GzipMember) of `data`."""
    src = np.frombuffer(bytes(data), np.uint8).copy() if data else np.zeros(1, np.uint8)
    cap = len(data) + len(data) // 100 + 1024
    out = np.zeros(cap, np.uint8)
    n = lib().sto_gzip(_p(src), len(data), _p(out), cap)
    assert n > 0
    return out[:n].tobytes()


# ---- the gzip member and the message, as the reference writes them ----
GZIP_HEADER = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x04\xff"   # boost gzip_compressor, best_speed


def gzip_member(data):
    """common::FastGzipString: boost's header, a raw deflate stream at level 1 (window 15,
    memLevel 8), CRC-32 and ISIZE."""
    z = zlib.compressobj(1, zlib.DEFLATED, -15, 8, zlib.Z_DEFAULT_STRATEGY)
    body = z.compress(bytes(data)) + z.flush()
    return (GZIP_HEADER + body + struct.pack("<I", zlib.crc32(bytes(data)) & 0xFFFFFFFF) +
            struct.pack("<I", len(data) & 0xFFFFFFFF))


def _double_present(v):
    return struct.pack("<d", v) != b"\0" * 8


def _f_double(field, v):
    return pw.f_double(field, v) if _double_present(v) else b""


def _f_int32(field, v):
    return pw.f_varint(field, v) if v != 0 else b""


def message(texture, gzipped=None):
    """proto::SubmapQuery::Response::SubmapTexture of `texture` serialised (proto3 rules: zero
    scalars omitted, -0.0 written, the slice pose's sub-messages always present); the cells
    gzip'd by gzip_member unless `gzipped` gives them."""
    cells = gzip_member(texture["cells"]) if gzipped is None else gzipped
    tx, ty, tz, qw, qx, qy, qz = texture["slice_pose"]
    translation = _f_double(1, tx) + _f_double(2, ty) + _f_double(3, tz)
    rotation = _f_double(1, qx) + _f_double(2, qy) + _f_double(3, qz) + _f_double(4, qw)
    pose = pw.f_bytes(1, translation) + pw.f_bytes(2, rotation)
    return (pw.f_bytes(1, cells) + _f_int32(2, texture["width"]) +
            _f_int32(3, texture["height"]) + _f_double(4, texture["resolution"]) +
            pw.f_bytes(5, pose))


def _read_varint(b, i):
    v, s = 0, 0
    while True:
        c = b[i]
        i += 1
        v |= (c & 0x7F) << s
        s += 7
        if not c & 0x80:
            return v, i


def _fields(b):
    out, i = [], 0
    while i < len(b):
        k, i = _read_varint(b, i)
        f, wt = k >> 3, k & 7
        if wt == 0:
            v, i = _read_varint(b, i)
        elif wt == 1:
            v, i = b[i:i + 8], i + 8
        elif wt == 5:
            v, i = b[i:i + 4], i + 4
        elif wt == 2:
            n, i = _read_varint(b, i)
            v, i = b[i:i + n], i + n
        else:
            raise ValueError("wire type %d" % wt)
        out.append((f, wt, v))
    return out


def parse(msg):
    """A serialised SubmapTexture back into a texture dict (cells decompressed, 'gzipped' the
    member as stored); absent fields read as proto3 defaults."""
    t = dict(cells=b"", gzipped=b"", width=0, height=0, resolution=0.0,
             slice_pose=(0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0))
    pose = [0.0] * 7
    for f, wt, v in _fields(msg):
        if f == 1:
            t["gzipped"] = bytes(v)
            t["cells"] = zlib.decompress(bytes(v), 16 + 15)
        elif f in (2, 3):
            x = v - (1 << 64) if v >= 1 << 63 else v
            t["width" if f == 2 else "height"] = x
        elif f == 4:
            t["resolution"] = struct.unpack("<d", v)[0]
        elif f == 5:
            for g, _, sub in _fields(v):
                for h, _, d in _fields(sub):
                    x = struct.unpack("<d", d)[0]
                    # translation {x, y, z} -> 0..2; rotation {x, y, z, w} -> 4, 5, 6, 3
                    pose[h - 1 if g == 1 else (4, 5, 6, 3)[h - 1]] = x
    t["slice_pose"] = tuple(pose)
    return t


def same_bits(a, b):
    return len(a) == len(b) and struct.pack("<%dd" % len(a), *a) == struct.pack("<%dd" % len(b), *b)
