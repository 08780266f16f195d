"""The assets writer's map-writing stages on the device (ProbabilityGridPointsProcessor,
HybridGridPointsProcessor) versus their CPU restatements.

Workload: `--batches` 1081-beam scans (8 m range, cast in a 30 m synthetic floor plan from
seeded poses, beams without a hit kept at 8 m as the assets writer keeps them) go one after
another into the 2D stage at 0.05 m, which grows its grid from 100 x 100 cells; `--batches3d`
config-5-size scans (64 rings x 1024 azimuths, 20 m range, in a 40 m synthetic building) go into
the 3D stage at 0.10 m.  Prints one JSON line: per-batch device and wall ms of the inserts, the
Flush costs (the 2D draw on the device and its wall time, the Grid2D and HybridGrid protos), the
same streams through the single-threaded restatements on the host (the C++ 2D insert and draw of
tests/, and the numpy 3D insert) with the host's core count, whether the device's grids, pixels
and protos equal the restatements', and the card name and power limit.

    python benchmarks/bench_points_to_grid.py --batches 200 --batches3d 20
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks import synthetic  # noqa: E402
from cartographer_b200 import points_processing as pp  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402
from tests import grid_proto_ref as R  # noqa: E402
from tests import insert2d_oracle as I2  # noqa: E402
from tests import insert3d_oracle as I3  # noqa: E402
from tests import probability_grid_draw_oracle as O  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


class Sink:
    """A file writer that keeps the bytes."""

    def __init__(self, name):
        self.data = b""

    def write(self, b):
        self.data += bytes(b)

    def close(self):
        pass


def batches2d(n):
    spec, occ = synthetic.make_grid2d(21, size_cells=600)
    rng = np.random.RandomState(7)
    centre = np.array([spec.max_x - 0.5 * occ.shape[0] * spec.resolution,
                       spec.max_y - 0.5 * occ.shape[1] * spec.resolution])
    out = []
    for k in range(n):
        pose = synthetic.random_free_pose(occ, spec, rng, margin_cells=40)
        pts = synthetic.cast_scan(occ, spec, pose, beams=1081, max_range=8.0, seed=k)
        c, s = math.cos(pose[2]), math.sin(pose[2])
        xy = np.stack([c * pts[:, 0] - s * pts[:, 1], s * pts[:, 0] + c * pts[:, 1]], 1) + \
            (pose[:2] - centre)
        out.append(pp.PointsBatch(np.concatenate([xy, np.zeros((len(xy), 1))], 1),
                                  origin=np.float32([*(pose[:2] - centre), 0.0])))
    return out


def batches3d(n):
    rng = np.random.RandomState(0)
    occ, cell, origin = synthetic.make_building(5, size_m=40.0)
    out = []
    for k in range(n):
        pose = synthetic.random_free_pose_3d(occ, cell, origin, rng)
        cloud = synthetic.cast_lidar_3d(occ, cell, origin, pose, rings=64, azimuths=1024,
                                        max_range=20.0, seed=k)
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (cloud.astype(np.float64) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T +
               pose[:3]).astype(np.float32)
        out.append(pp.PointsBatch(pts, origin=pose[:3].astype(np.float32)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=200)
    ap.add_argument("--batches3d", type=int, default=20)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    opts2 = sm.ProbabilityGridRangeDataInserterOptions2D(0.55, 0.49, True)
    opts3 = sm.RangeDataInserterOptions3D(0.55, 0.49, 2, 40.0)
    b2, b3 = batches2d(args.batches), batches3d(args.batches3d)

    # warm-up: every kernel and workspace once
    warm = pp.ProbabilityGridPointsProcessor(0.05, opts2, "w", "png", Sink)
    for b in b2[:3]:
        warm.Process(b)
    warm.grid.draw()
    warm.grid.to_proto()
    warm3 = pp.HybridGridPointsProcessor(0.10, opts3, "w", Sink)
    warm3.Process(b3[0])
    warm3.grid.to_proto()

    # 2D on the device
    stage = pp.ProbabilityGridPointsProcessor(0.05, opts2, "map", "png", Sink)
    dev_ms, t0 = 0.0, time.perf_counter()
    for b in b2:
        stage.Process(b)
        dev_ms += stage.inserter.last_stats["device_ms"]
    insert_wall = time.perf_counter() - t0
    lib = sm.lib()
    w, h = C.c_int32(), C.c_int32()
    offset = np.zeros(2, np.int32)
    op = offset.ctypes.data_as(C.POINTER(C.c_int32))
    sm.check(lib.csm_rt_grid2d_draw(stage.grid._h, None, C.c_int64(0), C.byref(w), C.byref(h),
                                    op, None))
    pixels = np.empty((h.value, w.value), np.uint32)
    stats = sm.CsmStats()
    t0 = time.perf_counter()
    sm.check(lib.csm_rt_grid2d_draw(stage.grid._h, pixels.ctypes.data_as(C.POINTER(C.c_uint32)),
                                    C.c_int64(pixels.size), C.byref(w), C.byref(h), op,
                                    C.byref(stats)))
    draw_wall = time.perf_counter() - t0
    t0 = time.perf_counter()
    proto2 = stage.grid.to_proto()
    proto2_wall = time.perf_counter() - t0
    st = stage.grid.read()

    # 2D on the host: the C++ restatements, one thread
    ora, ins = I2.Grid(0.05, 2.5, 2.5, 100, 100), I2.Inserter(0.55, 0.49, True)
    t0 = time.perf_counter()
    for b in b2:
        ins.insert(b.origin, b.points, ora)
    host_insert = time.perf_counter() - t0
    cells, box = ora.cells, ora.known_box
    O.lib()                                   # compiled on first use: not part of the timing
    t0 = time.perf_counter()
    want, want_offset = O.draw(cells, box)
    host_draw = time.perf_counter() - t0
    _, max_x, max_y, nx, ny = ora.limits
    parity2 = (np.array_equal(st.cells, cells) and st.known_cells_box == box and
               np.array_equal(pixels, want) and tuple(offset) == want_offset and
               proto2 == R.grid2d_message(cells, 0.05, max_x, max_y, box))

    # 3D on the device
    stage3 = pp.HybridGridPointsProcessor(0.10, opts3, "map_3d", Sink)
    dev3_ms, t0 = 0.0, time.perf_counter()
    for b in b3:
        stage3.Process(b)
        dev3_ms += stage3.inserter.last_stats["device_ms"]
    insert3_wall = time.perf_counter() - t0
    t0 = time.perf_counter()
    proto3 = stage3.grid.to_proto()
    proto3_wall = time.perf_counter() - t0

    # 3D on the host: the numpy restatement
    ora3, ins3 = I3.HybridGrid(0.10), I3.RangeDataInserter3D(**opts3.__dict__)
    t0 = time.perf_counter()
    for b in b3:
        ins3.insert(b.origin, b.points, None, ora3)
    host3 = time.perf_counter() - t0
    keep = ora3.values != 0
    idx, val, _ = R.walk((ora3.indices()[keep], ora3.values[keep]))
    parity3 = proto3 == R.hybrid_grid_message(np.float32(0.10), idx, val)

    print(json.dumps({
        "bench": "points_to_grid", "card": card(),
        "grid2d": {"batches": len(b2), "points_per_batch": 1081, "resolution": 0.05,
                   "final_cells": [int(nx), int(ny)], "image": [int(w.value), int(h.value)],
                   "insert_device_ms_per_batch": dev_ms / len(b2),
                   "insert_wall_ms_per_batch": 1e3 * insert_wall / len(b2),
                   "draw_device_ms": stats.device_ms, "draw_wall_ms": 1e3 * draw_wall,
                   "draw_host_syncs": stats.host_syncs, "proto_wall_ms": 1e3 * proto2_wall,
                   "proto_bytes": len(proto2),
                   "host_insert_ms_per_batch": 1e3 * host_insert / len(b2),
                   "host_draw_ms": 1e3 * host_draw, "parity": bool(parity2)},
        "grid3d": {"batches": len(b3), "points_per_batch": int(np.mean([len(b.points)
                                                                        for b in b3])),
                   "voxel_size": 0.10, "voxels": int(len(val)),
                   "insert_device_ms_per_batch": dev3_ms / len(b3),
                   "insert_wall_ms_per_batch": 1e3 * insert3_wall / len(b3),
                   "proto_wall_ms": 1e3 * proto3_wall, "proto_bytes": len(proto3),
                   "host_numpy_insert_ms_per_batch": 1e3 * host3 / len(b3),
                   "parity": bool(parity3)},
        "host_threads_used": 1, "host_cores": os.cpu_count()}))


if __name__ == "__main__":
    main()
