"""Building a FastCorrelativeScanMatcher3D from device-resident submap grids
(csm_matcher3d_create_from_grid3d) versus the path it replaces: reading both dense boxes
back (csm_grid3d_read), extracting the non-zero voxels on the host, and building the matcher
from the voxel lists (csm_matcher3d_create).

Workload: a config-5-like submap built on the device as benchmarks/bench_insert3d.py builds
it — `--scans` scans of 64 rings x 1024 azimuths (20 m max range, in a 40 m synthetic
building) inserted into empty 0.10 m and 0.45 m grids — and the pose_graph.lua matcher
options (depth 8, full resolution depth 3).  The two paths run alternately, `--reps` times
each after `--warmup` rounds.  Prints one JSON line: the median wall ms of each path, the
median device ms of (a) (its two profiled device spans), the voxel counts and boxes, whether
every precomputation level of (a) is byte-equal to (b)'s, and the card name and power limit.

    python benchmarks/bench_matcher3d_from_grid.py --scans 20
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
from cartographer_b200 import scan_matching as sm  # noqa: E402
from cartographer_b200._lib import lib  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def host_path(hi, lo, hist, opts):
    """(b): both boxes to the host, non-zero voxels, matcher from the lists."""
    specs = []
    for g in (hi, lo):
        blo, vol = g.read()
        z, y, x = np.nonzero(vol)
        idx = (np.stack([x, y, z], 1) + blo).astype(np.int32)
        specs.append(synthetic.HybridGridSpec(g.resolution, idx, vol[z, y, x]))
    return sm.FastCorrelativeScanMatcher3D(specs[0], specs[1], hist, opts), specs


def profiled_ms():
    buf = C.create_string_buffer(8192)
    lib().csm_profile_read(buf, 8192)
    total = 0.0
    for ln in buf.value.decode().strip().splitlines():
        name, _, ms, _ = ln.split()
        if name.startswith("m3g_"):
            total += float(ms)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    rng = np.random.RandomState(0)
    occ, cell, origin = synthetic.make_building(5, size_m=40.0)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng) for _ in range(4)]
    clouds = [synthetic.cast_lidar_3d(occ, cell, origin, p, rings=64, azimuths=1024,
                                      max_range=20.0, seed=i) for i, p in enumerate(poses)]
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(0.55, 0.49, 2, 40.0))
    hi, lo = sm.DeviceHybridGrid.empty(0.10), sm.DeviceHybridGrid.empty(0.45)
    for k in range(args.scans):
        pose = poses[k % len(poses)] + np.array([rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5),
                                                 0.0, rng.uniform(-0.5, 0.5)])
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (clouds[k % len(clouds)].astype(np.float64) @
               np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T + pose[:3]).astype(np.float32)
        org = pose[:3].astype(np.float32)
        ins.Insert(org, pts, None, hi)
        ins.Insert(org, pts, None, lo)
    opts = sm.FastCorrelativeScanMatcherOptions3D()   # pose_graph.lua: depth 8, frd 3
    hist = np.ones(120, np.float32)

    wall_a, wall_b, dev_a = [], [], []
    for r in range(args.warmup + args.reps):
        t0 = time.perf_counter()
        a = sm.FastCorrelativeScanMatcher3D.from_device_grids(hi, lo, hist, opts)
        ta = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        b, specs = host_path(hi, lo, hist, opts)
        tb = (time.perf_counter() - t0) * 1e3
        # the device spans of (a), in a separate call: profiling waits on its events
        lib().csm_profile_enable(1)
        sm.FastCorrelativeScanMatcher3D.from_device_grids(hi, lo, hist, opts).close()
        da = profiled_ms()
        lib().csm_profile_enable(0)
        if r >= args.warmup:
            wall_a.append(ta)
            wall_b.append(tb)
            dev_a.append(da)
        if r < args.warmup + args.reps - 1:
            a.close()
            b.close()
    equal = True
    levels = []
    for d in range(opts.branch_and_bound_depth):
        la, va = a.precomputation_grid(d)
        lb, vb = b.precomputation_grid(d)
        equal &= bool(np.array_equal(la, lb) and va.shape == vb.shape and np.array_equal(va, vb))
        levels.append([int(v) for v in va.shape[::-1]])
    boxes = {"high": [int(v) for v in hi.read()[1].shape[::-1]],
             "low": [int(v) for v in lo.read()[1].shape[::-1]]}
    print(json.dumps({
        "metric": "matcher3d_from_grid", "scans": args.scans, "reps": args.reps,
        "from_grid3d_wall_ms": float(np.median(wall_a)),
        "from_grid3d_device_ms": float(np.median(dev_a)),
        "host_roundtrip_wall_ms": float(np.median(wall_b)),
        "voxels": {"high": int(len(specs[0].values)), "low": int(len(specs[1].values))},
        "handle_boxes": boxes, "level_boxes": levels,
        "levels_byte_equal": equal, "card": card()}))
    for h in (a, b, hi, lo, ins):
        h.close()
    if not equal:
        raise SystemExit("the two paths built different levels")


if __name__ == "__main__":
    main()
