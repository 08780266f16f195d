"""The assets writer's outlier removal on the device (csm_outlier_remover_*) versus the host
restatement of OutlierRemovingPointsProcessor on one thread (tests/outlier_removal_oracle.cc,
std::map, g++ -O2).

Workload: a trajectory of config-5-like scans (64 rings x 1024 azimuths, 65,536 points each,
of synthetic.moving_box_scans: a 16 m building with a box crossing it, ranges up to 8 m),
`--scans` batches cycled over `--distinct` distinct scans, at --voxel-size (0.1 m default)
and miss_per_hit_limit 3.  The device takes --per-call batches per call.  Prints one JSON line:
per phase the device ms (CUDA events of all its calls) and the wall ms (host clock around all
its calls: checks, upload, kernels, read-back); the syncs per call; phase 2's samples (one hash
probe each) and samples per second of device time; the restatement's ms for the whole stream;
whether every voxel count and kept index equals the restatement's; the card's name, power limit
and clocks.

    python benchmarks/bench_outlier_removal.py --scans 100
"""
import argparse
import json
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
from tests import outlier_removal_oracle as O  # noqa: E402


def device_stream(batches, voxel_size, limit, per_call):
    groups = [batches[i:i + per_call] for i in range(0, len(batches), per_call)]
    r = pp.OutlierRemover(voxel_size, limit)
    out = {"device_ms": [0.0] * 3, "wall_ms": [0.0] * 3, "syncs": 0}
    kept = []

    def phase(k, fn):
        for g in groups:
            t0 = time.perf_counter()
            res = fn(g)
            out["wall_ms"][k] += (time.perf_counter() - t0) * 1e3
            st = res[1] if isinstance(res, tuple) else res
            out["device_ms"][k] += st["device_ms"]
            out["syncs"] = max(out["syncs"], st["host_syncs"])
            if isinstance(res, tuple):
                kept.extend(res[0])
    phase(0, lambda g: r.add_hits([p for _, p in g]))
    hits = r.voxels()
    phase(1, lambda g: r.count_rays([o for o, _ in g], [p for _, p in g]))
    rays = r.voxels()
    phase(2, lambda g: r.filter([p for _, p in g]))
    r.close()
    return hits, rays, kept, out


def samples(batches, voxel_size):
    """Phase 2's sample count: per ray the x_k below its length."""
    xs = O.ray_samples(voxel_size, 1e3, cap=1 << 24)
    total = 0
    for o, p in batches:
        d = p - o
        length = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        total += int(np.searchsorted(xs, length, side="left").sum())
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=100)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--per-call", type=int, default=20)
    ap.add_argument("--voxel-size", type=float, default=0.1)
    ap.add_argument("--limit", type=float, default=3.0)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    base = synthetic.moving_box_scans(5, args.distinct, rings=64, azimuths=1024, max_range=8.0)
    batches = [(o, np.resize(p, (65536, 3))) for o, p in
               (base[k % len(base)] for k in range(args.scans))]
    device_stream(batches[:args.per_call], args.voxel_size, args.limit, args.per_call)  # warm-up
    hits, rays, kept, dev = device_stream(batches, args.voxel_size, args.limit, args.per_call)
    t0 = time.perf_counter()
    want = O.run(batches, args.voxel_size, args.limit)
    host_ms = (time.perf_counter() - t0) * 1e3
    parity = all(np.array_equal(a, b) for a, b in zip(hits, want[0])) and \
        all(np.array_equal(a, b) for a, b in zip(rays, want[1])) and \
        len(kept) == len(want[2]) and all(np.array_equal(a, b) for a, b in zip(kept, want[2]))
    n_samples = samples(batches, args.voxel_size)
    result = {
        "bench": "outlier_removal", "card": card(), "batches": len(batches),
        "points": int(sum(len(p) for _, p in batches)), "voxel_size": args.voxel_size,
        "miss_per_hit_limit": args.limit, "batches_per_call": args.per_call,
        "voxels": int(len(hits[1])),
        "kept": int(sum(len(k) for k in kept)),
        "device_ms": {k: round(v, 3) for k, v in zip(("hits", "rays", "filter"),
                                                    dev["device_ms"])},
        "wall_ms": {k: round(v, 3) for k, v in zip(("hits", "rays", "filter"), dev["wall_ms"])},
        "wall_ms_total": round(sum(dev["wall_ms"]), 3),
        "host_syncs_per_call": dev["syncs"],
        "phase2_samples": n_samples,
        "phase2_samples_per_s": round(n_samples / (dev["device_ms"][1] * 1e-3), 1),
        "host_restatement_ms": round(host_ms, 1),
        "speedup_wall_vs_host": round(host_ms / sum(dev["wall_ms"]), 1),
        "parity": bool(parity),
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
