"""Saving device-resident submap grids: the serialised proto::HybridGrid / proto::Grid2D straight
from the handles (csm_grid3d_to_proto, csm_rt_grid2d_to_proto) versus the route they replace —
reading the grid back (csm_grid3d_read / csm_rt_grid2d_read and _read_weights), extracting the
voxels on the host in HybridGrid's iteration order, and encoding with tests/protowire.py's
writers (tests/grid_proto_ref.py for Grid2D).

Workloads: the config-5-like submap of benchmarks/bench_matcher3d_from_grid.py (`--scans` scans
of 64 rings x 1024 azimuths inserted into empty 0.10 m and 0.45 m grids), and 1600 x 1600 2D
grids, a ProbabilityGrid and a TSDF2D, filled by `--scans2d` inserted scans.  The two routes run
alternately, `--reps` times each after `--warmup` rounds.  Prints one JSON line: the median wall
ms of each route per grid, the message sizes, whether the two routes' bytes are equal, and the
card name and power limit.

    python benchmarks/bench_grid_to_proto.py --scans 20
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
from tests import grid_proto_ref as R  # noqa: E402
from tests import protowire as pw  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def host_hybrid(grid):
    """The replaced 3D route: the dense box to the host, the non-zero voxels sorted into
    HybridGrid's blocked iteration order, protowire encoding."""
    lo, vol = grid.read()
    z, y, x = np.nonzero(vol)
    idx = np.stack([x, y, z], 1).astype(np.int64) + lo
    xs, ys, zs = idx[:, 0], idx[:, 1], idx[:, 2]
    order = np.lexsort([xs & 7, ys & 7, zs & 7, (xs >> 3) & 7, (ys >> 3) & 7, (zs >> 3) & 7,
                        xs >> 6, ys >> 6, zs >> 6])
    return pw.hybrid_grid(grid.resolution, idx[order], vol[z, y, x][order])


def host_grid2d(grid, tsdf):
    """The replaced 2D route: cells (and weights) to the host, Grid2D encoding."""
    st = grid.read()
    if tsdf is None:
        return R.grid2d_message(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box)
    return R.grid2d_message(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box,
                            st.weight_cells, *tsdf)


def submap3d(scans):
    rng = np.random.RandomState(0)
    occ, cell, origin = synthetic.make_building(5, size_m=40.0)
    poses = [synthetic.random_free_pose_3d(occ, cell, origin, rng) for _ in range(4)]
    clouds = [synthetic.cast_lidar_3d(occ, cell, origin, p, rings=64, azimuths=1024,
                                      max_range=20.0, seed=i) for i, p in enumerate(poses)]
    ins = sm.RangeDataInserter3D(sm.RangeDataInserterOptions3D(0.55, 0.49, 2, 40.0))
    hi, lo = sm.DeviceHybridGrid.empty(0.10), sm.DeviceHybridGrid.empty(0.45)
    for k in range(scans):
        pose = poses[k % len(poses)] + np.array([rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5),
                                                 0.0, rng.uniform(-0.5, 0.5)])
        c, s = math.cos(pose[3]), math.sin(pose[3])
        pts = (clouds[k % len(clouds)].astype(np.float64) @
               np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]).T + pose[:3]).astype(np.float32)
        org = pose[:3].astype(np.float32)
        ins.Insert(org, pts, None, hi)
        ins.Insert(org, pts, None, lo)
    ins.close()
    return hi, lo


def grids2d(scans):
    spec, occ = synthetic.make_grid2d(7, size_cells=1600)
    rng = np.random.RandomState(1)
    prob = sm.RealTimeGrid2D.empty(spec.resolution, spec.max_x, spec.max_y, 1600, 1600)
    topts = sm.TSDFRangeDataInserterOptions2D()
    tsdf = sm.RealTimeGrid2D.empty_tsdf(spec.resolution, spec.max_x, spec.max_y,
                                        topts.truncation_distance, topts.maximum_weight,
                                        1600, 1600)
    pins, tins = sm.ProbabilityGridRangeDataInserter2D(), sm.TSDFRangeDataInserter2D(topts)
    for k in range(scans):
        pose = synthetic.random_free_pose(occ, spec, rng, margin_cells=60)
        pts = synthetic.cast_scan(occ, spec, pose, beams=1081, max_range=30.0, seed=k)
        c, s = math.cos(pose[2]), math.sin(pose[2])
        w = np.stack([c * pts[:, 0] - s * pts[:, 1] + pose[0],
                      s * pts[:, 0] + c * pts[:, 1] + pose[1], np.zeros(len(pts))],
                     1).astype(np.float32)
        far = np.hypot(pts[:, 0], pts[:, 1]) >= 30.0 - 0.05
        origin = np.float32([pose[0], pose[1], 0])
        pins.Insert(origin, w[~far], prob, w[far])
        tins.Insert(origin, w[~far], tsdf)
    pins.close()
    tins.close()
    return prob, tsdf, (topts.truncation_distance, topts.maximum_weight)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--scans2d", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    hi, lo = submap3d(args.scans)
    prob, tsdf, tsdf_params = grids2d(args.scans2d)
    cases = {
        "hybrid_high": (hi.to_proto, lambda: host_hybrid(hi)),
        "hybrid_low": (lo.to_proto, lambda: host_hybrid(lo)),
        "probability_grid_1600": (prob.to_proto, lambda: host_grid2d(prob, None)),
        "tsdf_1600": (tsdf.to_proto, lambda: host_grid2d(tsdf, tsdf_params)),
    }
    result = {"metric": "grid_to_proto", "scans": args.scans, "scans2d": args.scans2d,
              "reps": args.reps}
    equal = True
    for name, (device, host) in cases.items():
        wall_d, wall_h = [], []
        for r in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            a = device()
            td = (time.perf_counter() - t0) * 1e3
            t0 = time.perf_counter()
            b = host()
            th = (time.perf_counter() - t0) * 1e3
            if r >= args.warmup:
                wall_d.append(td)
                wall_h.append(th)
        equal &= a == b
        result[name] = {"device_route_wall_ms": float(np.median(wall_d)),
                        "host_route_wall_ms": float(np.median(wall_h)),
                        "bytes": len(a), "byte_equal": a == b}
    result["voxels"] = {"high": int(len(hi.voxels()[1])), "low": int(len(lo.voxels()[1]))}
    result["byte_equal"] = bool(equal)
    result["card"] = card()
    print(json.dumps(result))
    for h in (hi, lo, prob, tsdf):
        h.close()
    if not equal:
        raise SystemExit("the two routes wrote different bytes")


if __name__ == "__main__":
    main()
