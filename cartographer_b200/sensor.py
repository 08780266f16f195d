"""cartographer::sensor on the device: VoxelFilter and AdaptiveVoxelFilter
(sensor/internal/voxel_filter.cc), bit for bit with the reference's reservoir sampling.

Points are (n, 3) float32 arrays.  The filters return the kept points in input order, and their
intensities when intensities are given; the batch forms return the kept input indices of many
clouds from one device call (csm_voxel_filter_batch / csm_adaptive_voxel_filter_batch).
"""
import ctypes as C
from collections import namedtuple

import numpy as np

from . import _lib

# proto AdaptiveVoxelFilterOptions (sensor/proto/adaptive_voxel_filter_options.proto); all
# three fields are floats there.
AdaptiveVoxelFilterOptions = namedtuple("AdaptiveVoxelFilterOptions",
                                        "max_length min_num_points max_range")


class CsmAdaptiveVoxelFilterOptions(C.Structure):
    _fields_ = [("max_length", C.c_float), ("min_num_points", C.c_float),
                ("max_range", C.c_float), ("reserved", C.c_int32)]


def _clouds(clouds):
    return [np.ascontiguousarray(np.asarray(c, np.float32).reshape(-1, 3)) for c in clouds]


def _run(fn, clouds, params, device):
    clouds = _clouds(clouds)
    n = len(clouds)
    counts = np.array([len(c) for c in clouds], np.int32)
    ptrs = (C.POINTER(C.c_float) * max(n, 1))(*[_lib.ptr(c, C.c_float) for c in clouds])
    kept = np.zeros(max(int(counts.sum()), 1), np.int32)
    num_kept = np.zeros(max(n, 1), np.int32)
    stats = _lib.CsmStats()
    _lib.check(fn(ptrs, _lib.ptr(counts, C.c_int32), params, n, device,
                  _lib.ptr(kept, C.c_int32), _lib.ptr(num_kept, C.c_int32), C.byref(stats)))
    out, at = [], 0
    for k in num_kept[:n]:
        out.append(kept[at:at + k].copy())
        at += k
    return out, stats.as_dict()


def voxel_filter_batch(clouds, resolutions, device=0):
    """Kept input indices of VoxelFilter(clouds[c], resolutions[c]) for every cloud, and the
    call's stats (host_syncs, device_ms)."""
    res = np.ascontiguousarray(np.broadcast_to(np.asarray(resolutions, np.float32),
                                               (len(clouds),)))
    return _run(_lib.lib().csm_voxel_filter_batch, clouds, _lib.ptr(res, C.c_float), device)


def adaptive_voxel_filter_batch(clouds, options, device=0):
    """Kept input indices of AdaptiveVoxelFilter(clouds[c], options[c]) for every cloud (one
    AdaptiveVoxelFilterOptions serves them all), and the call's stats."""
    if isinstance(options, AdaptiveVoxelFilterOptions):
        options = [options] * len(clouds)
    opts = (CsmAdaptiveVoxelFilterOptions * max(len(clouds), 1))(
        *[CsmAdaptiveVoxelFilterOptions(o.max_length, o.min_num_points, o.max_range, 0)
          for o in options])
    return _run(_lib.lib().csm_adaptive_voxel_filter_batch, clouds, opts, device)


def _gather(points, intensities, kept):
    pts = np.asarray(points, np.float32).reshape(-1, 3)[kept]
    if intensities is None:
        return pts
    return pts, np.asarray(intensities, np.float32)[kept]


def VoxelFilter(points, resolution, intensities=None, device=0):
    """sensor::VoxelFilter: the kept points (and intensities) in input order."""
    (kept,), _ = voxel_filter_batch([points], [resolution], device)
    return _gather(points, intensities, kept)


def AdaptiveVoxelFilter(points, options, intensities=None, device=0):
    """sensor::AdaptiveVoxelFilter: the kept points (and intensities) in input order."""
    (kept,), _ = adaptive_voxel_filter_batch([points], [options], device)
    return _gather(points, intensities, kept)
