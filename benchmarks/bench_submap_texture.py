"""Drawing submaps for display: the serialised proto::SubmapQuery::Response::SubmapTexture
straight from the device handles (csm_grid3d_to_texture, csm_rt_grid2d_to_texture) versus the
route they replace — reading the grid back, drawing it with the host restatement
(tests/submap_texture_oracle.cc, one thread, the reference's sequential loops) and gzip'ing and
framing the cells (tests/submap_texture_oracle.py, zlib level 1).

Workloads: the config-5-like submap of benchmarks/bench_matcher3d_from_grid.py (`--scans` scans
of 64 rings x 1024 azimuths inserted into empty 0.10 m and 0.45 m grids) under a yawed and
slightly tilted global pose, and a 1600 x 1600 active 2D ProbabilityGrid filled by `--scans2d`
1081-beam scans, its cropped (finished) form, and a 1600 x 1600 TSDF2D.  The two routes run
alternately, `--reps` times each after `--warmup` rounds.  Both include gzip on the host; the
gzip time of the cells alone is measured separately, and the device route's remainder (wall
minus gzip: kernels, copies and synchronisations) is reported as device_ms.  Prints one JSON
line with median ms per texture, whether the routes' decompressed cells, sizes and slice poses
are equal, and the card name and power limit.

    python benchmarks/bench_submap_texture.py --scans 20
"""
import argparse
import json
import math
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_grid_to_proto import card, grids2d, submap3d  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402
from tests import submap_texture_oracle as T  # noqa: E402

YAW, ROLL, PITCH = math.radians(37.0), 0.02, -0.015


def global_pose():
    """(tx, ty, tz, qw, qx, qy, qz) of yaw * pitch * roll and a translation."""
    cr, sr = math.cos(ROLL / 2), math.sin(ROLL / 2)
    cp, sp = math.cos(PITCH / 2), math.sin(PITCH / 2)
    cy, sy = math.cos(YAW / 2), math.sin(YAW / 2)
    return (12.3, -4.56, 0.78, cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy,
            cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy)


def host_texture3d(grid, pose):
    """The replaced 3D route: the dense box to the host, the non-zero voxels sorted into
    HybridGrid's blocked iteration order, the restatement, gzip and framing."""
    lo, vol = grid.read()
    z, y, x = np.nonzero(vol)
    idx = np.stack([x, y, z], 1).astype(np.int64) + lo
    xs, ys, zs = idx[:, 0], idx[:, 1], idx[:, 2]
    order = np.lexsort([xs & 7, ys & 7, zs & 7, (xs >> 3) & 7, (ys >> 3) & 7, (zs >> 3) & 7,
                        xs >> 6, ys >> 6, zs >> 6])
    t = T.texture3d(idx[order], vol[z, y, x][order], grid.resolution, pose)
    return T.message(t), t


def host_texture2d(grid, pose, tsdf):
    """The replaced 2D route: cells (and weights) to the host, the restatement, gzip, framing."""
    st = grid.read()
    if tsdf is None:
        t = T.texture2d(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box, pose)
    else:
        t = T.texture2d(st.cells, st.resolution, st.max_x, st.max_y, st.known_cells_box, pose,
                        st.weight_cells, *tsdf)
    return T.message(t), t


def same(msg, t):
    got = T.parse(msg)
    return (got["cells"] == t["cells"] and (got["width"], got["height"]) == (t["width"],
                                                                             t["height"]) and
            T.same_bits(got["slice_pose"], t["slice_pose"]))


def gzip_ms(cells, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        T.gzip_member(cells)
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


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
    crop = prob.ComputeCroppedGrid()
    pose3 = global_pose()
    pose2 = (1.5, -2.5, 0.0, math.cos(YAW / 2), 0.0, 0.0, math.sin(YAW / 2))
    cases = {
        "hybrid_high": (lambda: hi.to_texture(pose3), lambda: host_texture3d(hi, pose3)),
        "hybrid_low": (lambda: lo.to_texture(pose3), lambda: host_texture3d(lo, pose3)),
        "probability_grid_1600": (lambda: prob.to_texture(pose2),
                                  lambda: host_texture2d(prob, pose2, None)),
        "probability_grid_cropped": (lambda: crop.to_texture(pose2),
                                     lambda: host_texture2d(crop, pose2, None)),
        "tsdf_1600": (lambda: tsdf.to_texture(pose2),
                      lambda: host_texture2d(tsdf, pose2, tsdf_params)),
    }
    result = {"metric": "submap_texture", "scans": args.scans, "scans2d": args.scans2d,
              "reps": args.reps, "zlib": zlib.ZLIB_RUNTIME_VERSION}
    equal = True
    for name, (device, host) in cases.items():
        wall_d, wall_h = [], []
        for r in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            a = device()
            td = (time.perf_counter() - t0) * 1e3
            t0 = time.perf_counter()
            b, t = host()
            th = (time.perf_counter() - t0) * 1e3
            if r >= args.warmup:
                wall_d.append(td)
                wall_h.append(th)
        ok = same(a, t)
        equal &= ok
        gz = gzip_ms(t["cells"], args.reps)
        result[name] = {"device_route_wall_ms": float(np.median(wall_d)),
                        "device_ms": float(np.median(wall_d)) - gz,
                        "host_route_wall_ms": float(np.median(wall_h)),
                        "gzip_ms": gz, "pixels": t["width"] * t["height"],
                        "message_bytes": len(a), "cells_equal": ok}
    result["voxels"] = {"high": int(len(hi.voxels()[1])), "low": int(len(lo.voxels()[1]))}
    result["cells_equal"] = bool(equal)
    result["card"] = card()
    print(json.dumps(result))
    for h in (hi, lo, prob, crop, tsdf):
        h.close()
    if not equal:
        raise SystemExit("the two routes drew different textures")


if __name__ == "__main__":
    main()
