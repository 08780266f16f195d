"""Inserting each scan into the two active 3D submaps with one call
(csm_range_inserter3d_insert_submaps, Submap3D::InsertData on the device) versus the recipe it
replaces: per submap, the host transform into the submap frame and the high-resolution range
filter, then two csm_range_inserter3d_insert calls (four calls per scan).

Workload: `--scans` config-5-like scans (64 rings x 1024 azimuths, 20 m max range, cast in a
40 m synthetic building from a few seeded poses and moved around them, 5 % of the returns
pushed past the 20 m high-resolution range) go, in the local frame, into two submaps at two
different local poses: 0.10 m and 0.45 m grids and a 0.10 m intensity grid each, all starting
empty (the steady state of ActiveSubmaps3D).  The two paths run on separate handles, scan by
scan alternately.  Prints one JSON line: per-scan device and wall ms of both paths, the old
path's wall time split into the host transform and filter, a host cell pass of the same points
(the C++ restatement of CellIndex, standing in for the single-grid call's host loop), the
upload of those cells (timed as a pinned host-to-device copy of the same bytes) and the rest
(the calls' device work, synchronisation and remaining host work); whether every handle is
bit-equal at the end; and the card name and power limit.

    python benchmarks/bench_active_submaps3d.py --scans 100
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks import synthetic  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402

F = np.float32


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def host_library(tmp):
    """tests/submap_insert3d_oracle.cc, the single-thread host restatement of the transform,
    the filter and the cells, built into a temporary directory."""
    so = os.path.join(tmp, "libsubmap_insert3d_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared",
                           os.path.join(ROOT, "tests", "submap_insert3d_oracle.cc"), "-o", so])
    return C.CDLL(so)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    import torch
    rng = np.random.RandomState(0)
    occ, cell, origin = synthetic.make_building(5, size_m=40.0)
    world = (occ, cell, origin)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng) for _ in range(4)]
    clouds = [synthetic.cast_lidar_3d(occ, cell, origin, p, rings=64, azimuths=1024,
                                      max_range=20.0, seed=i) for i, p in enumerate(poses)]
    opts = sm.RangeDataInserterOptions3D(hit_probability=0.55, miss_probability=0.49,
                                         num_free_space_voxels=2, intensity_threshold=40.0)
    new_ins, old_ins = sm.RangeDataInserter3D(opts), sm.RangeDataInserter3D(opts)
    m0, m1 = poses[0], poses[1]
    submap_poses = [[m0[0], m0[1], m0[2], math.cos(m0[3] / 2), 0.0, 0.0, math.sin(m0[3] / 2)],
                    [m1[0], m1[1], m1[2], math.cos(m1[3] / 2), 0.01, -0.02,
                     math.sin(m1[3] / 2)]]
    submap_poses[1][3:] = list(np.asarray(submap_poses[1][3:]) /
                               np.linalg.norm(submap_poses[1][3:]))

    def handles():
        return [(sm.DeviceHybridGrid.empty(0.10), sm.DeviceHybridGrid.empty(0.45),
                 sm.DeviceIntensityGrid.empty(0.10)) for _ in submap_poses]

    new_h, old_h = handles(), handles()
    tmp = tempfile.mkdtemp(prefix="bench_active_submaps3d_")
    host = host_library(tmp)
    rec = {k: [] for k in ("new_dev", "new_wall", "old_dev", "old_wall", "old_transform",
                           "old_cells", "old_upload")}
    for k in range(args.warmup + args.scans):
        base = poses[k % len(poses)]
        pose = base + np.array([rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5), 0.0,
                                rng.uniform(-0.5, 0.5)])
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (clouds[k % len(clouds)].astype(np.float64) @
               np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T + pose[:3]).astype(F)
        far = rng.rand(len(pts)) < 0.05
        pts[far] = (pose[:3] + (pts[far] - pose[:3]) * 1.6).astype(F)
        inten = synthetic.surface_intensity(world, pts, seed=k)
        org = pose[:3].astype(F)
        keep = k >= args.warmup
        # ---- new: one call for both submaps ----
        t0 = time.perf_counter()
        new_ins.insert_submaps([(p, *h) for p, h in zip(submap_poses, new_h)], org, pts, inten,
                               20.0)
        if keep:
            rec["new_wall"].append((time.perf_counter() - t0) * 1e3)
            rec["new_dev"].append(new_ins.last_stats["device_ms"])
        # ---- old: per submap, host transform and filter, then two calls ----
        wall = dev = tr = 0.0
        transformed = []
        for p, (hi, lo, ig) in zip(submap_poses, old_h):
            t0 = time.perf_counter()
            out_o, out_p = np.zeros(3, F), np.zeros_like(pts)
            kept = np.zeros(len(pts), np.uint8)
            host.submap_transform(_p(np.asarray(p, np.float64), C.c_double), _p(org, C.c_float),
                                  _p(pts, C.c_float), len(pts), C.c_float(20.0),
                                  _p(out_o, C.c_float), _p(out_p, C.c_float),
                                  _p(kept, C.c_uint8))
            kept = kept.astype(bool)
            near, near_i = np.ascontiguousarray(out_p[kept]), np.ascontiguousarray(inten[kept])
            t1 = time.perf_counter()
            old_ins.Insert(out_o, near, near_i, hi, ig)
            dev += old_ins.last_stats["device_ms"]
            old_ins.Insert(out_o, out_p, None, lo)
            dev += old_ins.last_stats["device_ms"]
            t2 = time.perf_counter()
            tr += (t1 - t0) * 1e3
            wall += (t2 - t0) * 1e3
            transformed.append((near, out_p))
        if not keep:
            continue
        rec["old_wall"].append(wall)
        rec["old_dev"].append(dev)
        rec["old_transform"].append(tr)
        # the single-grid calls' host cell loop, restated: the same points, the same grids
        t0 = time.perf_counter()
        nbytes = 0
        for near, all_p in transformed:
            for pts_r, res in ((near, 0.10), (near, 0.10), (all_p, 0.45)):
                cells = np.zeros(pts_r.shape, np.int32)
                ok = np.zeros(len(pts_r), np.uint8)
                host.submap_cells(_p(pts_r, C.c_float), len(pts_r), C.c_float(res),
                                  _p(cells, C.c_int32), _p(ok, C.c_uint8))
                nbytes += cells.nbytes
        rec["old_cells"].append((time.perf_counter() - t0) * 1e3)
        # ... and their uploads: the same bytes, pinned host to device, synchronised
        src = torch.empty(nbytes // 4, dtype=torch.int32).pin_memory()
        dst = torch.empty(nbytes // 4, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        rec["old_upload"].append((time.perf_counter() - t0) * 1e3)
    # ---- every handle bit-equal ----
    equal = True
    for (a_hi, a_lo, a_ig), (b_hi, b_lo, b_ig) in zip(new_h, old_h):
        for a, b in ((a_hi, b_hi), (a_lo, b_lo)):
            (la, va), (lb, vb) = a.read(), b.read()
            equal &= bool(np.array_equal(la, lb) and np.array_equal(va, vb))
        for x, y in zip(a_ig.read(), b_ig.read()):
            equal &= bool(x.shape == y.shape and x.tobytes() == y.tobytes())
    med = {k: float(np.median(v)) for k, v in rec.items()}
    result = {
        "bench": "active_submaps3d", "scans": args.scans, "submaps": len(submap_poses),
        "points_per_scan": int(np.mean([len(c) for c in clouds])),
        "new_device_ms": med["new_dev"], "new_wall_ms": med["new_wall"],
        "old_device_ms": med["old_dev"], "old_wall_ms": med["old_wall"],
        "old_split_ms": {
            "host_transform_and_filter": med["old_transform"],
            "host_cells_restated": med["old_cells"],
            "upload_of_cells_restated": med["old_upload"],
            "rest_device_sync_host": med["old_wall"] - med["old_transform"] - med["old_cells"]
            - med["old_upload"],
        },
        "speedup_wall": med["old_wall"] / med["new_wall"],
        "bit_equal": equal, "card": card(),
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
