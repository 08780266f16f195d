"""Voxel-filtering scans on the device (csm_voxel_filter_batch, csm_adaptive_voxel_filter_batch)
versus the host restatement of sensor::VoxelFilter / AdaptiveVoxelFilter on one thread
(tests/voxel_filter_oracle.cc, std::unordered_map, g++ -O2).

Workloads, the two per-scan chains of local SLAM:
  3D: a config-5-like scan (64 rings x 1024 azimuths of a seeded box room), VoxelFilter at
      0.15 m (trajectory_builder_3d.lua voxel_filter_size), then the high (2.0 / 150 / 15) and
      low (4.0 / 200 / max) resolution adaptive filters of the filtered cloud as one batch;
  2D: a 1081-beam / 270 degree scan, VoxelFilter at 0.025 m, then the adaptive filter
      0.5 / 200 / 50 (trajectory_builder_2d.lua).
Prints one JSON line: per chain, the median over `--scans` scans of the device ms (CUDA events
of both calls), the wall ms (host clock around both calls: upload, filter, index read-back,
the gather between them), the host syncs per chain, the restatement's ms, and whether every kept
index equals the restatement's; and the card's name, power limit and clocks.

    python benchmarks/bench_voxel_filter.py --scans 200
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_insert2d import card  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402
from cartographer_b200 import sensor  # noqa: E402
from tests import voxel_filter_oracle as O  # noqa: E402

CHAINS = {
    "3d": dict(scan=O.box_room_scan, size=0.15,
               adaptive=[(2.0, 150.0, 15.0), (4.0, 200.0, float(np.finfo(np.float32).max))]),
    "2d": dict(scan=O.planar_scan, size=0.025, adaptive=[(0.5, 200.0, 50.0)]),
}


def device_chain(pts, size, adaptive):
    (kept,), s1 = sensor.voxel_filter_batch([pts], [size])
    filtered = pts[kept]
    opts = [sensor.AdaptiveVoxelFilterOptions(*t) for t in adaptive]
    out, s2 = sensor.adaptive_voxel_filter_batch([filtered] * len(opts), opts)
    return kept, out, s1["device_ms"] + s2["device_ms"], s1["host_syncs"] + s2["host_syncs"]


def host_chain(pts, size, adaptive):
    kept, _ = O.voxel_filter(pts, size)
    filtered = pts[kept]
    return kept, [O.adaptive_voxel_filter(filtered, *t)[0] for t in adaptive]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    result = {"bench": "voxel_filter", "scans": args.scans, "card": card()}
    for name, ch in CHAINS.items():
        scans = [ch["scan"](seed) for seed in range(args.scans)]
        for pts in scans[:args.warmup]:
            device_chain(pts, ch["size"], ch["adaptive"])
            host_chain(pts, ch["size"], ch["adaptive"])
        dev, wall, host, syncs, points, kept_n, equal = [], [], [], [], [], [], True
        for pts in scans:
            t0 = time.perf_counter()
            kept, out, d, n_sync = device_chain(pts, ch["size"], ch["adaptive"])
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(d)
            syncs.append(n_sync)
            t0 = time.perf_counter()
            hk, hout = host_chain(pts, ch["size"], ch["adaptive"])
            host.append((time.perf_counter() - t0) * 1e3)
            equal &= np.array_equal(kept, hk) and all(np.array_equal(a, b)
                                                      for a, b in zip(out, hout))
            points.append(len(pts))
            kept_n.append(len(kept))
        result[name] = {
            "points": int(np.median(points)), "kept_by_voxel_filter": int(np.median(kept_n)),
            "device_ms": round(float(np.median(dev)), 4),
            "wall_ms": round(float(np.median(wall)), 4),
            "wall_ms_p90": round(float(np.percentile(wall, 90)), 4),
            "host_restatement_ms": round(float(np.median(host)), 4),
            "host_syncs_per_chain": int(max(syncs)),
            "speedup_wall_vs_host": round(float(np.median(host) / np.median(wall)), 2),
            "equal_to_restatement": bool(equal),
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
