"""cartographer::io points processing on the device: OutlierRemovingPointsProcessor
(io/outlier_removing_points_processor.cc), the assets writer's
voxel_filter_and_remove_moving_objects stage, with its voxel map on the GPU and every count and
kept point bit for bit the reference's; and XRayPointsProcessor (io/xray_points_processor.cc),
its write_xray_image stage, with its voxels, column sums and image on the GPU and every pixel the
reference's; and the map-writing stages ProbabilityGridPointsProcessor
(io/probability_grid_points_processor.cc, write_probability_grid) and HybridGridPointsProcessor
(io/hybrid_grid_points_processor.cc, write_hybrid_grid), whose grids grow on the GPU from the first
batch to the image or proto they save.

OutlierRemover and XRay are the device handles (csm_outlier_remover_*, csm_xray_*): each call
takes many batches.  OutlierRemovingPointsProcessor and XRayPointsProcessor are the pipeline
stages with the reference's Process / Flush over them; the map-writing stages insert into the
device grids of scan_matching (RealTimeGrid2D, DeviceHybridGrid).  Points are (n, 3) float32
arrays.
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


def _colors(colors_list, pts):
    out = []
    for c, p in zip(colors_list, pts):
        if c is None or len(c) == 0:
            out.append(None)
        else:
            c = np.ascontiguousarray(np.asarray(c, np.float32).reshape(-1, 3))
            if len(c) != len(p):
                raise ValueError("one colour per point, or none")
            out.append(c)
    return out


class XRay:
    """The device aggregations of one XRayPointsProcessor (csm_xray_*): per aggregation (one per
    floor, or one) its voxels and per (y, z) column the float sums and count of its colours, and
    one bounding box shared by all.  `transform` is (t x, y, z, q w, x, y, z), a Rigid3f.  Each
    insert takes any number of batches and makes one stream synchronisation.  Refusals raise
    _lib.CsmError and change nothing."""

    def __init__(self, voxel_size, transform=(0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0),
                 saturation_factor=1.0, num_aggregations=1, device=0):
        self._L = _lib.lib()
        t = np.ascontiguousarray(np.asarray(transform, np.float32).reshape(7))
        h = C.c_void_p()
        _lib.check(self._L.csm_xray_create(C.c_double(voxel_size), C.c_double(saturation_factor),
                                           _lib.ptr(t, C.c_float), num_aggregations, device,
                                           C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._L.csm_xray_destroy(self._h)
            self._h = None

    __del__ = close

    def insert(self, points_list, colors_list=None, aggregation=0):
        """Inserts the batches, in order; colors_list[b] is None (black) or (n, 3) float32.
        Returns the call's stats."""
        pts, counts, ptrs = _batches(points_list)
        cols = _colors(colors_list if colors_list is not None else [None] * len(pts), pts)
        rgb = (C.POINTER(C.c_float) * max(len(pts), 1))(
            *[_lib.ptr(c, C.c_float) if c is not None else None for c in cols])
        stats = _lib.CsmStats()
        _lib.check(self._L.csm_xray_insert(self._h, aggregation, ptrs, rgb,
                                           _lib.ptr(counts, C.c_int32), len(pts),
                                           C.byref(stats)))
        return stats.as_dict()

    def bounding_box(self):
        """(min (3,), max (3,), empty) of the shared box of cell indices."""
        lo, hi, empty = np.zeros(3, np.int32), np.zeros(3, np.int32), C.c_int32()
        _lib.check(self._L.csm_xray_bounding_box(self._h, _lib.ptr(lo, C.c_int32),
                                                 _lib.ptr(hi, C.c_int32), C.byref(empty)))
        return lo, hi, bool(empty.value)

    def draw(self, aggregation=0):
        """(pixels, stats): the aggregation's image as a (height, width) uint32 array of cairo
        ARGB32 words, or None when nothing was ever inserted."""
        w, ht = C.c_int32(), C.c_int32()
        _lib.check(self._L.csm_xray_draw(self._h, aggregation, None, C.c_int64(0), C.byref(w),
                                         C.byref(ht), None))
        if w.value == 0:
            return None, {"host_syncs": 0, "device_ms": 0.0}
        px = np.empty((ht.value, w.value), np.uint32)
        stats = _lib.CsmStats()
        _lib.check(self._L.csm_xray_draw(self._h, aggregation, _lib.ptr(px, C.c_uint32),
                                         C.c_int64(px.size), C.byref(w), C.byref(ht),
                                         C.byref(stats)))
        return px, stats.as_dict()

    def voxels(self, aggregation=0):
        """(n, 3) cell indices of the aggregation's voxels in ascending (z, y, x)."""
        n = C.c_int64()
        _lib.check(self._L.csm_xray_voxels(self._h, aggregation, None, C.c_int64(0), C.byref(n)))
        idx = np.zeros((max(n.value, 1), 3), np.int32)
        _lib.check(self._L.csm_xray_voxels(self._h, aggregation, _lib.ptr(idx, C.c_int32),
                                           C.c_int64(len(idx)), C.byref(n)))
        return idx[:n.value]

    def columns(self, aggregation=0):
        """(yz (n, 2), sums (n, 3) float32, counts (n,) uint32) in ascending (y, z)."""
        n = C.c_int64()
        _lib.check(self._L.csm_xray_columns(self._h, aggregation, None, None, None, C.c_int64(0),
                                            C.byref(n)))
        m = max(n.value, 1)
        yz, sums, counts = np.zeros((m, 2), np.int32), np.zeros((m, 3), np.float32), \
            np.zeros(m, np.uint32)
        _lib.check(self._L.csm_xray_columns(self._h, aggregation, _lib.ptr(yz, C.c_int32),
                                            _lib.ptr(sums, C.c_float),
                                            _lib.ptr(counts, C.c_uint32), C.c_int64(m),
                                            C.byref(n)))
        k = n.value
        return yz[:k], sums[:k], counts[:k]


def cairo_to_rgb(pixels):
    """(height, width, 3) uint8 of cairo ARGB32 words (0xFF << 24 | r << 16 | g << 8 | b)."""
    p = np.asarray(pixels, np.uint32)
    return np.stack([(p >> 16) & 0xFF, (p >> 8) & 0xFF, p & 0xFF], -1).astype(np.uint8)


def encode_png(pixels):
    """An 8-bit RGB PNG of cairo ARGB32 words: IHDR, one IDAT holding one zlib stream of the
    unfiltered scanlines, IEND.  The pixels are the reference's; the bytes are not cairo's (which
    writes RGBA with its own filters and compression), so compare decoded pixels, not files."""
    import struct
    import zlib
    rgb = cairo_to_rgb(pixels)
    height, width = rgb.shape[:2]
    raw = np.concatenate([np.zeros((height, 1), np.uint8), rgb.reshape(height, 3 * width)], 1)

    def chunk(kind, data):
        return struct.pack(">I", len(data)) + kind + data + \
            struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)
    return (b"\x89PNG\r\n\x1a\n" +
            chunk(b"IHDR", struct.pack(">IIBBBBB", width, height, 8, 2, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(raw.tobytes())) + chunk(b"IEND", b""))


def decode_png(data):
    """(height, width, 3) uint8 of a PNG that encode_png wrote."""
    import struct
    import zlib
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    at, idat, width, height = 8, b"", 0, 0
    while at < len(data):
        n, = struct.unpack(">I", data[at:at + 4])
        kind, body = data[at + 4:at + 8], data[at + 8:at + 8 + n]
        if kind == b"IHDR":
            width, height = struct.unpack(">II", body[:8])
            assert body[8:] == bytes([8, 2, 0, 0, 0])
        elif kind == b"IDAT":
            idat += body
        at += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(height, 1 + 3 * width)
    assert not raw[:, 0].any()
    return raw[:, 1:].reshape(height, width, 3)


def _file_writer(filename):
    return open(filename, "wb")


class XRayPointsProcessor:
    """io::XRayPointsProcessor: X-ray cuts through the points with pixels voxel_size big, drawn
    on the device.  Process inserts the batch into every floor whose timespans contain its
    start_time (or into the one aggregation without floors) and passes it on; Flush writes
    filename + ".png", or filename + str(i) + ".png" per floor, and then flushes `next`.
    `floors` is a list of floors, each a list of (start, end) timespans compared with
    PointsBatch.start_time; `file_writer_factory(name)` returns an object with write and close
    (a binary file by default).  The PNG carries the pixels only (see encode_png); trajectories
    are not drawn here.  With next=None the batches collect in `.output`."""

    kConfigurationFileActionName = "write_xray_image"

    def __init__(self, voxel_size, transform, filename, saturation_factor=1.0, floors=None,
                 file_writer_factory=None, next=None, device=0):
        self.floors = [list(f) for f in floors] if floors else []
        self.xray = XRay(voxel_size, transform, saturation_factor,
                         max(1, len(self.floors)), device)
        self.filename = filename
        self.file_writer_factory = file_writer_factory or _file_writer
        self.next = next
        self.output = []

    def bounding_box(self):
        return self.xray.bounding_box()

    def Process(self, batch):
        if not self.floors:
            self.xray.insert([batch.points], [batch.colors])
        else:
            for i, spans in enumerate(self.floors):
                if any(start <= batch.start_time <= end for start, end in spans):
                    self.xray.insert([batch.points], [batch.colors], aggregation=i)
        if self.next is None:
            self.output.append(batch)
        else:
            self.next.Process(batch)

    def _write(self, aggregation, name):
        pixels, _ = self.xray.draw(aggregation)
        if pixels is None:
            import warnings
            warnings.warn("Not writing output: bounding box is empty.")
            return
        f = self.file_writer_factory(name)
        f.write(encode_png(pixels))
        f.close()

    def Flush(self):
        if not self.floors:
            self._write(0, self.filename + ".png")
        else:
            for i in range(len(self.floors)):
                self._write(i, self.filename + str(i) + ".png")
        if self.next is not None and self.next.Flush() != FlushResult.kFinished:
            raise RuntimeError("X-Ray generation must be configured to occur after any stages "
                               "that require multiple passes.")
        return FlushResult.kFinished


class ProbabilityGridPointsProcessor:
    """io::ProbabilityGridPointsProcessor: every batch goes into one ProbabilityGrid on the
    device (CreateProbabilityGrid: 100 x 100 cells, max = 0.5 * 100 * resolution on both axes)
    as ProbabilityGridRangeDataInserter2D inserts {origin, points, no misses}, and passes on.
    Flush writes filename + ".png", DrawProbabilityGrid's pixels (see encode_png; trajectories
    are not drawn here), or filename + ".pb", the serialised proto::Grid2D, and then flushes
    `next`.  The file writer is made at construction, as FromDictionary makes it.  An insert that
    would grow the grid to 30 000 cells per axis raises _lib.CsmError and leaves the grid as it
    was.  With next=None the batches collect in `.output`."""

    kConfigurationFileActionName = "write_probability_grid"
    kInitialProbabilityGridSize = 100

    def __init__(self, resolution, range_data_inserter_options, filename, output_type="png",
                 file_writer_factory=None, next=None, device=0):
        from . import scan_matching as sm
        if output_type not in ("png", "pb"):
            raise ValueError("OutputType %s does not exist!" % output_type)
        self.output_type = output_type
        half = 0.5 * self.kInitialProbabilityGridSize * resolution
        self.grid = sm.RealTimeGrid2D.empty(resolution, half, half,
                                            self.kInitialProbabilityGridSize,
                                            self.kInitialProbabilityGridSize, device)
        self.inserter = sm.ProbabilityGridRangeDataInserter2D(range_data_inserter_options, device)
        self.file_writer = (file_writer_factory or _file_writer)(filename + "." + output_type)
        self.next = next
        self.output = []

    def Process(self, batch):
        self.inserter.Insert(batch.origin, batch.points, self.grid)
        if self.next is None:
            self.output.append(batch)
        else:
            self.next.Process(batch)

    def Flush(self):
        if self.output_type == "png":
            pixels, _ = self.grid.draw()
            self.file_writer.write(encode_png(pixels))
        else:
            self.file_writer.write(self.grid.to_proto())
        self.file_writer.close()
        if self.next is not None and self.next.Flush() != FlushResult.kFinished:
            raise RuntimeError("ProbabilityGrid generation must be configured to occur after any "
                               "stages that require multiple passes.")
        return FlushResult.kFinished


class HybridGridPointsProcessor:
    """io::HybridGridPointsProcessor: every batch goes into one HybridGrid(float(voxel_size)) on
    the device as RangeDataInserter3D inserts {origin, points, no misses} without an intensity
    grid, and passes on.  Flush writes the serialised proto::HybridGrid to exactly `filename`
    and then flushes `next`.  The grid is the dense device box of DeviceHybridGrid: a cell
    outside [-8192, 8192)^3, or a box the device cannot hold, raises _lib.CsmError and leaves
    the grid as it was.  With next=None the batches collect in `.output`."""

    kConfigurationFileActionName = "write_hybrid_grid"

    def __init__(self, voxel_size, range_data_inserter_options, filename,
                 file_writer_factory=None, next=None, device=0):
        from . import scan_matching as sm
        self.grid = sm.DeviceHybridGrid.empty(float(np.float32(voxel_size)), device)
        self.inserter = sm.RangeDataInserter3D(range_data_inserter_options, device)
        self.file_writer = (file_writer_factory or _file_writer)(filename)
        self.next = next
        self.output = []

    def Process(self, batch):
        self.inserter.Insert(batch.origin, batch.points, None, self.grid)
        if self.next is None:
            self.output.append(batch)
        else:
            self.next.Process(batch)

    def Flush(self):
        self.file_writer.write(self.grid.to_proto())
        self.file_writer.close()
        if self.next is not None and self.next.Flush() != FlushResult.kFinished:
            raise RuntimeError("Hybrid grid generation must be configured to occur after any "
                               "stages that require multiple passes.")
        return FlushResult.kFinished
