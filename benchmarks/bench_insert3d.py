"""Inserting scans into device-resident 3D grids (RangeDataInserter3D on the device) versus
what it replaces: inserting on the host and re-creating the device handles from the whole
grid after every scan.

Workload: `--scans` config-5-like scans (64 rings x 1024 azimuths, 20 m max range, cast in a
40 m synthetic building from a few seeded poses and moved around them) go one after another
into a high-resolution (0.10 m) grid with its intensity grid and a low-resolution (0.45 m)
grid, all starting empty — LocalTrajectoryBuilder3D's two inserts per scan into one submap
(Submap3D::InsertData, submap_3d.cc:271-290).  Prints one JSON line: per-insert device and
wall ms of the device path, the host path's per-scan costs (the numpy CPU restatement's
insert, and re-creating the three handles from the grids' voxel lists), whether the final
grids are bit-equal to the restatement's, and the card name and power limit.

    python benchmarks/bench_insert3d.py --scans 100
"""
import argparse
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
from cartographer_b200 import scan_matching as sm  # noqa: E402
from tests import insert3d_oracle as O  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--recreate-every", type=int, default=10,
                    help="time the handle re-creation on every k-th scan")
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    rng = np.random.RandomState(0)
    occ, cell, origin = synthetic.make_building(5, size_m=40.0)
    world = (occ, cell, origin)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng) for _ in range(4)]
    clouds = [synthetic.cast_lidar_3d(occ, cell, origin, p, rings=64, azimuths=1024,
                                      max_range=20.0, seed=i) for i, p in enumerate(poses)]
    opts = dict(hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
                intensity_threshold=40.0)   # trajectory_builder_3d.lua
    dev_ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(**opts))
    ora_ins = O.RangeDataInserter3D(**opts)
    hi, lo, ig = (sm.DeviceHybridGrid.empty(0.10), sm.DeviceHybridGrid.empty(0.45),
                  sm.DeviceIntensityGrid.empty(0.10))
    ohi, olo, oig = O.HybridGrid(0.10), O.HybridGrid(0.45), O.IntensityHybridGrid(0.10)
    dev_ms, wall_ms, host_ms, recreate_ms, points = [], [], [], [], []
    for k in range(args.scans):
        base = poses[k % len(poses)]
        pose = base + np.array([rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5), 0.0,
                                rng.uniform(-0.5, 0.5)])
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (clouds[k % len(clouds)].astype(np.float64) @
               np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T + pose[:3]).astype(np.float32)
        inten = synthetic.surface_intensity(world, pts, seed=k)
        org = pose[:3].astype(np.float32)
        near = np.linalg.norm(pts - org, axis=1) <= 20.0   # FilterRangeDataByMaxRange
        points.append(len(pts))
        t0 = time.perf_counter()
        dev_ins.Insert(org, pts[near], inten[near], hi, ig)
        d = dev_ins.last_stats["device_ms"]
        dev_ins.Insert(org, pts, None, lo)
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        dev_ms.append(d + dev_ins.last_stats["device_ms"])
        t0 = time.perf_counter()
        ora_ins.insert(org, pts[near], inten[near], ohi, oig)
        ora_ins.insert(org, pts, None, olo)
        host_ms.append((time.perf_counter() - t0) * 1e3)
        if k % args.recreate_every == args.recreate_every - 1:
            t0 = time.perf_counter()
            handles = [sm.DeviceHybridGrid(synthetic.HybridGridSpec(0.10, ohi.indices(), ohi.values)),
                       sm.DeviceHybridGrid(synthetic.HybridGridSpec(0.45, olo.indices(), olo.values)),
                       sm.DeviceIntensityGrid(sm.IntensityGridSpec(0.10, oig.indices(), oig.sums,
                                                                   oig.counts))]
            recreate_ms.append((time.perf_counter() - t0) * 1e3)
            for h in handles:
                h.close()
    equal = True
    for dev, ora in ((hi, ohi), (lo, olo)):
        l, vol = dev.read()
        equal &= bool(np.array_equal(vol, ora.dense(l, vol.shape[::-1])))
    l, mean, sums, counts = ig.read()
    dims = mean.shape[::-1]
    equal &= bool(np.array_equal(counts, oig.dense(l, dims, 1)) and
                  np.array_equal(sums.view(np.uint32), oig.dense(l, dims, 0).view(np.uint32)) and
                  np.array_equal(mean.view(np.uint32), oig.dense_mean(l, dims).view(np.uint32)))
    steady = slice(min(5, args.scans - 1), None)   # the first inserts grow the boxes
    med = lambda v: float(np.median(v[steady] if len(v) == args.scans else v))  # noqa: E731
    print(json.dumps({
        "metric": "insert3d", "scans": args.scans, "mean_points": float(np.mean(points)),
        "device_ms_per_scan": med(dev_ms), "wall_ms_per_scan": med(wall_ms),
        "device_ms_first_scan": dev_ms[0], "wall_ms_first_scan": wall_ms[0],
        "host_numpy_insert_ms_per_scan": med(host_ms),
        "recreate_3_handles_ms_per_scan": float(np.median(recreate_ms)) if recreate_ms else None,
        "final_voxels": {"high": int((ohi.values != 0).sum()), "low": int((olo.values != 0).sum()),
                         "intensity": int(len(oig.keys))},
        "dense_boxes": {"high": [int(v) for v in hi.read()[1].shape[::-1]],
                        "low": [int(v) for v in lo.read()[1].shape[::-1]]},
        "bit_equal_to_oracle": equal, "card": card()}))
    for h in (hi, lo, ig, dev_ins):
        h.close()
    if not equal:
        raise SystemExit("device grids differ from the CPU restatement")


if __name__ == "__main__":
    main()
