"""ctypes loader of the CPU restatement of VoxelFilter / AdaptiveVoxelFilter
(tests/voxel_filter_oracle.cc): the parity reference of the device voxel filter and the host
column of benchmarks/bench_voxel_filter.py.  The library is compiled on first use into a
temporary directory, so that nothing is written into the tree."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "voxel_filter_oracle.cc")

_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="voxel_filter_oracle_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libvoxel_filter_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", SRC, "-o", so])
        L = C.CDLL(so)
        vp = C.c_void_p
        L.vfo_key.restype = C.c_uint64
        L.vfo_key.argtypes = [C.c_float] * 4
        L.vfo_generator.argtypes = [C.c_int, vp]
        L.vfo_uniform.argtypes = [C.c_int, vp, vp]
        L.vfo_voxel_filter.argtypes = [vp, C.c_int, C.c_float, vp, vp, vp]
        L.vfo_adaptive_voxel_filter.argtypes = [vp, C.c_int] + [C.c_float] * 3 + [vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _cloud(points):
    return np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))


def key(x, y, z, resolution):
    return int(lib().vfo_key(x, y, z, resolution))


def generator(count):
    out = np.zeros(count, np.uint32)
    lib().vfo_generator(count, _p(out))
    return out


def uniform(k, raw):
    """uniform_int_distribution<int>(1, k) on the raw outputs `raw`: (result, outputs used)."""
    raw = np.ascontiguousarray(raw, np.uint32)
    used = np.zeros(1, np.int32)
    r = lib().vfo_uniform(k, _p(raw), _p(used))
    return r, int(used[0])


def voxel_filter(points, resolution):
    """Kept input indices and {"calls", "draws", "rejections"} of VoxelFilter."""
    pts = _cloud(points)
    kept = np.zeros(max(len(pts), 1), np.int32)
    calls = np.zeros(1, np.int64)
    draws = np.zeros(1, np.int64)
    n = lib().vfo_voxel_filter(_p(pts), len(pts), resolution, _p(kept), _p(calls), _p(draws))
    return kept[:n].copy(), {"calls": int(calls[0]), "draws": int(draws[0]),
                             "rejections": int(draws[0] - calls[0])}


def adaptive_voxel_filter(points, max_length, min_num_points, max_range):
    """Kept input indices and {"length", "trials"} of AdaptiveVoxelFilter (length 0: the
    range-filtered cloud was returned)."""
    pts = _cloud(points)
    kept = np.zeros(max(len(pts), 1), np.int32)
    length = np.zeros(1, np.float32)
    trials = np.zeros(1, np.int32)
    n = lib().vfo_adaptive_voxel_filter(_p(pts), len(pts), max_length, min_num_points,
                                        max_range, _p(kept), _p(length), _p(trials))
    return kept[:n].copy(), {"length": float(length[0]), "trials": int(trials[0])}


def box_room_scan(seed, rings=64, azimuths=1024, vfov_deg=15.0, noise=0.01):
    """A config-5-like lidar scan (rings x azimuths rays) of a box room, in the sensor frame:
    the room's size and the sensor's place in it come from the seed."""
    rng = np.random.RandomState(seed)
    half = rng.uniform([4.0, 3.0], [15.0, 10.0])
    lo = np.array([-half[0], -half[1], 0.0]) - np.append(rng.uniform(-1, 1, 2) * half * 0.5, 0)
    hi = lo + np.array([2 * half[0], 2 * half[1], rng.uniform(2.5, 6.0)])
    o = np.array([0.0, 0.0, rng.uniform(0.5, 2.0)])
    el = np.deg2rad(np.linspace(-vfov_deg, vfov_deg, rings))
    az = np.linspace(-np.pi, np.pi, azimuths, endpoint=False)
    E, A = np.meshgrid(el, az, indexing="ij")
    d = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)
    with np.errstate(divide="ignore"):
        t = np.where(d > 0, (hi - o) / d, np.where(d < 0, (lo - o) / d, np.inf)).min(axis=1)
    t = t + rng.normal(0.0, noise, len(t))
    return (o + d * t[:, None]).astype(np.float32)


def planar_scan(seed, beams=1081, fov_deg=270.0, max_range=30.0, noise=0.01):
    """A 2D scan (beams over fov_deg, z = 0) of a box room, as box_room_scan with one ring."""
    rng = np.random.RandomState(seed)
    lo = -rng.uniform(1.0, 20.0, 2)
    hi = rng.uniform(1.0, 20.0, 2)
    a = np.deg2rad(np.linspace(-fov_deg / 2, fov_deg / 2, beams))
    d = np.stack([np.cos(a), np.sin(a)], -1)
    with np.errstate(divide="ignore"):
        t = np.where(d > 0, hi / d, np.where(d < 0, lo / d, np.inf)).min(axis=1)
    t = np.minimum(t + rng.normal(0.0, noise, beams), max_range)
    return np.stack([d[:, 0] * t, d[:, 1] * t, np.zeros(beams)], -1).astype(np.float32)
