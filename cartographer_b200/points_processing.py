"""cartographer::io points processing on the device: OutlierRemovingPointsProcessor
(io/outlier_removing_points_processor.cc), the assets writer's
voxel_filter_and_remove_moving_objects stage, with its voxel map on the GPU and every count and
kept point bit for bit the reference's.

OutlierRemover is the device handle (csm_outlier_remover_*): its three phases each take many
batches per call.  OutlierRemovingPointsProcessor is the pipeline stage with the reference's
Process / Flush state machine over it.  Points are (n, 3) float32 arrays.
"""
import ctypes as C
import enum

import numpy as np

from . import _lib


class FlushResult(enum.Enum):
    """PointsProcessor::FlushResult (io/points_processor.h)."""
    kRestartStream = 0
    kFinished = 1


class PointsBatch:
    """io::PointsBatch (io/points_batch.h): points captured around one time from one origin, with
    optional per-point intensities and colors."""

    def __init__(self, points, origin=(0.0, 0.0, 0.0), intensities=None, colors=None,
                 frame_id="", trajectory_id=0, start_time=0):
        self.points = np.ascontiguousarray(np.asarray(points, np.float32).reshape(-1, 3))
        self.origin = np.asarray(origin, np.float32).reshape(3)
        self.intensities = None if intensities is None else np.asarray(intensities, np.float32)
        self.colors = None if colors is None else np.asarray(colors, np.float32).reshape(-1, 3)
        self.frame_id = frame_id
        self.trajectory_id = trajectory_id
        self.start_time = start_time

    def keep_points(self, kept):
        """What io::RemovePoints leaves: the points at the ascending indices `kept`, with their
        intensities and colors."""
        self.points = self.points[kept]
        if self.intensities is not None and len(self.intensities):
            self.intensities = self.intensities[kept]
        if self.colors is not None and len(self.colors):
            self.colors = self.colors[kept]


def _batches(points_list):
    pts = [np.ascontiguousarray(np.asarray(p, np.float32).reshape(-1, 3)) for p in points_list]
    n = len(pts)
    counts = np.array([len(p) for p in pts], np.int32)
    ptrs = (C.POINTER(C.c_float) * max(n, 1))(*[_lib.ptr(p, C.c_float) for p in pts])
    return pts, counts, ptrs


class OutlierRemover:
    """The device voxel map of one OutlierRemovingPointsProcessor and its three phases.  Each
    call takes any number of batches and makes one stream synchronisation; phases only move
    forward.  Refusals raise _lib.CsmError and change nothing."""

    def __init__(self, voxel_size, miss_per_hit_limit=3.0, device=0):
        self._L = _lib.lib()
        h = C.c_void_p()
        _lib.check(self._L.csm_outlier_remover_create(C.c_double(voxel_size),
                                                      C.c_double(miss_per_hit_limit),
                                                      device, C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._L.csm_outlier_remover_destroy(self._h)
            self._h = None

    __del__ = close

    def add_hits(self, points_list):
        """Phase 1 over the batches' points; returns the call's stats."""
        pts, counts, ptrs = _batches(points_list)
        stats = _lib.CsmStats()
        _lib.check(self._L.csm_outlier_remover_add_hits(self._h, ptrs, _lib.ptr(counts, C.c_int32),
                                                        len(pts), C.byref(stats)))
        return stats.as_dict()

    def count_rays(self, origins, points_list):
        """Phase 2: origins[b] is batch b's origin; returns the call's stats."""
        pts, counts, ptrs = _batches(points_list)
        org = np.ascontiguousarray(np.asarray(origins, np.float32).reshape(-1, 3))
        if len(org) != len(pts):
            raise ValueError("one origin per batch")
        stats = _lib.CsmStats()
        _lib.check(self._L.csm_outlier_remover_count_rays(
            self._h, _lib.ptr(org, C.c_float), ptrs, _lib.ptr(counts, C.c_int32), len(pts),
            C.byref(stats)))
        return stats.as_dict()

    def filter(self, points_list):
        """Phase 3: the kept indices of every batch (in input order) and the call's stats."""
        pts, counts, ptrs = _batches(points_list)
        kept = np.zeros(max(int(counts.sum()), 1), np.int32)
        num_kept = np.zeros(max(len(pts), 1), np.int32)
        stats = _lib.CsmStats()
        _lib.check(self._L.csm_outlier_remover_filter(
            self._h, ptrs, _lib.ptr(counts, C.c_int32), len(pts), _lib.ptr(kept, C.c_int32),
            _lib.ptr(num_kept, C.c_int32), C.byref(stats)))
        out, at = [], 0
        for k in num_kept[:len(pts)]:
            out.append(kept[at:at + k].copy())
            at += k
        return out, stats.as_dict()

    def voxels(self):
        """(indices (n, 3), hits, rays) of every voxel with hits, in ascending (z, y, x)."""
        n = C.c_int64()
        _lib.check(self._L.csm_outlier_remover_voxels(self._h, None, None, None, 0, C.byref(n)))
        m = max(n.value, 1)
        idx = np.zeros((m, 3), np.int32)
        hits = np.zeros(m, np.int32)
        rays = np.zeros(m, np.int32)
        _lib.check(self._L.csm_outlier_remover_voxels(
            self._h, _lib.ptr(idx, C.c_int32), _lib.ptr(hits, C.c_int32),
            _lib.ptr(rays, C.c_int32), C.c_int64(m), C.byref(n)))
        k = n.value
        return idx[:k], hits[:k], rays[:k]

    def info(self):
        """{"phase", "voxels", "slots"}: the current phase (1, 2, 3), the voxel count and the
        map's slot count."""
        phase, voxels, slots = C.c_int32(), C.c_int64(), C.c_int64()
        _lib.check(self._L.csm_outlier_remover_info(self._h, C.byref(phase), C.byref(voxels),
                                                    C.byref(slots)))
        return {"phase": phase.value, "voxels": voxels.value, "slots": slots.value}


class OutlierRemovingPointsProcessor:
    """io::OutlierRemovingPointsProcessor: Process(batch) and Flush() with the reference's
    kPhase1 -> kPhase2 -> kPhase3 state machine; each Flush before the last returns
    kRestartStream, so the pipeline streams every batch again.  In phase 3 the batch loses the
    points in obstructed voxels (with their intensities and colors) and goes to `next`.  With
    next=None the filtered batches collect in `.output` and the final Flush finishes."""

    kConfigurationFileActionName = "voxel_filter_and_remove_moving_objects"

    def __init__(self, voxel_size, miss_per_hit_limit=3.0, next=None, device=0):
        self.remover = OutlierRemover(voxel_size, miss_per_hit_limit, device)
        self.next = next
        self.output = []
        self.phase = 1

    def Process(self, batch):
        if self.phase == 1:
            self.remover.add_hits([batch.points])
        elif self.phase == 2:
            self.remover.count_rays([batch.origin], [batch.points])
        else:
            (kept,), _ = self.remover.filter([batch.points])
            batch.keep_points(kept)
            if self.next is None:
                self.output.append(batch)
            else:
                self.next.Process(batch)

    def Flush(self):
        if self.phase < 3:
            self.phase += 1
            return FlushResult.kRestartStream
        if self.next is not None and self.next.Flush() != FlushResult.kFinished:
            raise RuntimeError("Voxel filtering and outlier removal must be configured to occur "
                               "after any stages that require multiple passes.")
        return FlushResult.kFinished
