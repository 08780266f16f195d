"""The assets writer's X-ray images on the device (csm_xray_*) versus the host restatement of
XRayPointsProcessor on one thread (tests/xray_oracle.cc, std::map, g++ -O2).

Workload: config-5-like coloured scans (64 rings x 1024 azimuths, 65,536 points each, of
synthetic.moving_box_scans with seeded colours), `--scans` batches cycled over `--distinct`
distinct scans at --voxel-size (0.05 m default), streamed into `--views` processors with
different view transforms (the assets writer's XY, XZ and YZ cuts, then tilted ones), as a
pipeline that runs write_xray_image once per view.  The device takes --per-call batches per
insert call and draws each view once at the end.  Prints one JSON line: the device ms (CUDA
events of all calls) and wall ms (host clock around all calls: checks, staging, kernels,
read-back) of the inserts and of the draws; points per second of insert device time; the most
syncs any call made; the restatement's ms for the same views; whether every pixel, voxel and
column equals the restatement's; the card's name, power limit and clocks.

    python benchmarks/bench_xray.py --scans 100 --views 3
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks import synthetic  # noqa: E402
from benchmarks.bench_insert2d import card  # noqa: E402
from cartographer_b200 import points_processing as pp  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402
from tests import xray_oracle as O  # noqa: E402

S = math.sqrt(0.5)


def views(k):
    """k view transforms (t x, y, z, q w, x, y, z): XY (pitch -pi/2), XZ (yaw -pi/2), YZ
    (identity), then rotations about a tilted axis."""
    out = [(0.0, 0.0, 0.0, S, 0.0, -S, 0.0), (0.0, 0.0, 0.0, S, 0.0, 0.0, -S),
           (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)]
    j = 0
    while len(out) < k:
        j += 1
        a = 0.4 * j
        axis = np.array([0.3, -0.5, 0.81]) / np.linalg.norm([0.3, -0.5, 0.81])
        q = [math.cos(a / 2)] + list(math.sin(a / 2) * axis)
        out.append((0.2 * j, -0.1 * j, 0.05 * j) + tuple(q))
    return out[:k]


def device_stream(batches, voxel_size, transforms, per_call):
    groups = [batches[i:i + per_call] for i in range(0, len(batches), per_call)]
    xs = [pp.XRay(voxel_size, t) for t in transforms]
    out = {"device_ms": [0.0, 0.0], "wall_ms": [0.0, 0.0], "syncs": 0}
    for g in groups:
        for x in xs:
            t0 = time.perf_counter()
            st = x.insert([p for p, _ in g], [c for _, c in g])
            out["wall_ms"][0] += (time.perf_counter() - t0) * 1e3
            out["device_ms"][0] += st["device_ms"]
            out["syncs"] = max(out["syncs"], st["host_syncs"])
    images = []
    for x in xs:
        t0 = time.perf_counter()
        px, st = x.draw()
        out["wall_ms"][1] += (time.perf_counter() - t0) * 1e3
        out["device_ms"][1] += st["device_ms"]
        out["syncs"] = max(out["syncs"], st["host_syncs"])
        images.append(px)
    return xs, images, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--per-call", type=int, default=20)
    ap.add_argument("--voxel-size", type=float, default=0.05)
    ap.add_argument("--views", type=int, default=3)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    base = synthetic.moving_box_scans(5, args.distinct, rings=64, azimuths=1024, max_range=8.0)
    rng = np.random.RandomState(17)
    batches = [(np.resize(base[k % len(base)][1], (65536, 3)),
                rng.uniform(0, 1, (65536, 3)).astype(np.float32)) for k in range(args.scans)]
    transforms = views(args.views)
    device_stream(batches[:args.per_call], args.voxel_size, transforms[:1], args.per_call)
    xs, images, dev = device_stream(batches, args.voxel_size, transforms, args.per_call)
    host_ms = 0.0
    parity = True
    for x, px, t in zip(xs, images, transforms):
        t0 = time.perf_counter()
        o = O.Processor(args.voxel_size, transform=t)
        for p, c in batches:
            assert o.insert(p, c)
        want = o.draw()
        host_ms += (time.perf_counter() - t0) * 1e3
        parity = parity and np.array_equal(px, want) and np.array_equal(x.voxels(), o.voxels())
        for a, b in zip(x.columns(), o.columns()):
            parity = parity and np.array_equal(a.view(np.uint32), b.view(np.uint32))
    points = sum(len(p) for p, _ in batches)
    result = {
        "bench": "xray", "card": card(), "batches": len(batches), "points": int(points),
        "views": len(transforms), "voxel_size": args.voxel_size,
        "batches_per_call": args.per_call,
        "voxels": [int(len(x.voxels())) for x in xs],
        "image_pixels": [int(px.size) for px in images],
        "device_ms": {"insert": round(dev["device_ms"][0], 3), "draw": round(dev["device_ms"][1], 3)},
        "wall_ms": {"insert": round(dev["wall_ms"][0], 3), "draw": round(dev["wall_ms"][1], 3)},
        "wall_ms_total": round(sum(dev["wall_ms"]), 3),
        "insert_points_per_s": round(points * len(transforms) / (dev["device_ms"][0] * 1e-3), 1),
        "host_syncs_per_call": dev["syncs"],
        "host_restatement_ms": round(host_ms, 1),
        "speedup_wall_vs_host": round(host_ms / sum(dev["wall_ms"]), 1),
        "parity": bool(parity),
    }
    for x in xs:
        x.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
