"""ConstraintBuilder2D on device-resident submaps versus the route a device submap had to take
before: for each finished submap, read the cropped cells back (csm_rt_grid2d_read), make a host
grid record, and let the builder upload it twice (csm_stack2d_create for the stack and
csm_rt_grid2d_create for the refinement).

Workload: `--submaps` submaps, each grown on the device by ProbabilityGridRangeDataInserter2D
from `--scans` 1081-beam scans (30 m range) in the 50 m synthetic world and cropped on the
device; `--nodes` 361-beam node scans taken within 1.5 m of the submaps' centres; one drain
of all submaps x nodes local pairs with the config-4 search (7 m / 30°, depth 7, min score 0.55) and the Ceres refinement on.  The two
paths run alternately, `--reps` times each after `--warmup` rounds.  Prints one JSON line:

* crop_to_stack_ms: median wall ms per finished submap from the crop to a ready stack (and,
  for (b), the refinement's upload): (a) crop + stack from the handle, (b) crop + read-back +
  host record + both uploads;
* constraints_per_s: the drain's constraints per second of wall time, stacks built inside the
  drain (for (b) including the read-backs);
* identical: whether (a) and (b) gave the same constraints, bit for bit;
* the card name and power limit.

    python benchmarks/bench_cb2d_device_submaps.py --submaps 4 --nodes 25
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
from cartographer_b200 import constraint_builder as cb  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def world_scan(occ, spec, pose, seed, max_range=30.0):
    """A 1081-beam scan in the world frame: origin, returns, and the beams that reached
    max_range as misses."""
    pts = synthetic.cast_scan(occ, spec, pose, beams=1081, max_range=max_range, seed=seed)
    c, s = math.cos(pose[2]), math.sin(pose[2])
    w = np.stack([c * pts[:, 0] - s * pts[:, 1] + pose[0], s * pts[:, 0] + c * pts[:, 1] + pose[1],
                  np.zeros(len(pts))], 1).astype(np.float32)
    far = np.hypot(pts[:, 0], pts[:, 1]) >= max_range - 0.05
    return np.float32([pose[0], pose[1], 0]), w[~far], w[far]


def grow(occ, spec, poses, seed):
    """An active submap's grid after its scans, before Finish."""
    ins = sm.ProbabilityGridRangeDataInserter2D()
    grid = sm.RealTimeGrid2D.empty(0.05, poses[0][0] + 2.5, poses[0][1] + 2.5)
    for k, pose in enumerate(poses):
        origin, returns, misses = world_scan(occ, spec, pose, seed + k)
        ins.Insert(origin, returns, grid, misses)
    ins.close()
    return grid


def options():
    return cb.ConstraintBuilderOptions(
        sampling_ratio=1.0, max_constraint_distance=100.0, min_score=0.55,
        linear_search_window=7.0, angular_search_window=math.radians(30.0),
        branch_and_bound_depth=7, ceres_scan_matcher_options=sm.CeresScanMatcherOptions2D())


def finish(active, device_path):
    """Crop to ready stack for one submap; returns the closeable handles it made."""
    opts = options()
    fo = sm.FastCorrelativeScanMatcherOptions2D(opts.linear_search_window,
                                                opts.angular_search_window,
                                                opts.branch_and_bound_depth)
    crop = active.ComputeCroppedGrid()
    if device_path:
        return [crop, sm.FastCorrelativeScanMatcher2D.from_device_grid(crop, fo)]
    host = crop.read()
    return [crop, sm.FastCorrelativeScanMatcher2D(host, fo), sm.RealTimeGrid2D(host)]


def drain(crops, local_poses, nodes, device_path):
    """One builder, one drain of every (submap, node) pair; stacks built inside it."""
    b = cb.ConstraintBuilder2D(options())
    submaps = {(0, s): cb.Submap2D(c if device_path else c.read(), local_poses[s])
               for s, c in enumerate(crops)}
    for n, (cloud, pose) in enumerate(nodes):
        start = (pose[0] + 0.1, pose[1] - 0.1, pose[2] + 0.02)
        for sid, sub in submaps.items():
            b.MaybeAddConstraint(sid, sub, (0, n), cloud,
                                 cb._compose(cb._inverse(sub.local_pose), start))
        b.NotifyEndOfNode()
    result = b.WhenDone(lambda r: None)
    for sid in submaps:
        b.DeleteScanMatcher(sid)
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--submaps", type=int, default=4)
    ap.add_argument("--nodes", type=int, default=25)
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    spec, occ = synthetic.make_grid2d(4, size_cells=1000)
    rng = np.random.RandomState(0)
    centres = [synthetic.random_free_pose(occ, spec, rng, margin_cells=100)
               for _ in range(args.submaps)]
    active = [grow(occ, spec, [c + np.array([0.2 * k, -0.1 * k, 0.03 * k])
                               for k in range(args.scans)], seed=1000 * s)
              for s, c in enumerate(centres)]
    crops = [a.ComputeCroppedGrid() for a in active]
    local_poses = [(float(c[0]), float(c[1]), 0.0) for c in centres]
    # nodes near the submaps' centres, as the scans a trajectory revisits
    node_poses = [centres[n % args.submaps] + rng.uniform([-1.5, -1.5, -0.3], [1.5, 1.5, 0.3])
                  for n in range(args.nodes)]
    nodes = [(synthetic.cast_scan(occ, spec, p, beams=361, max_range=30.0, seed=5000 + n),
              tuple(float(v) for v in p)) for n, p in enumerate(node_poses)]

    finish_ms = {True: [], False: []}
    drain_s = {True: [], False: []}
    results = {}
    for r in range(args.warmup + args.reps):
        for device_path in (True, False):
            t0 = time.perf_counter()
            made = [finish(a, device_path) for a in active]
            t = (time.perf_counter() - t0) * 1e3 / len(active)
            for handles in made:
                for h in handles:
                    h.close()
            t0 = time.perf_counter()
            res = drain(crops, local_poses, nodes, device_path)
            d = time.perf_counter() - t0
            if r >= args.warmup:
                finish_ms[device_path].append(t)
                drain_s[device_path].append(d)
            results[device_path] = res
    bits = {k: [(c.submap_id, c.node_id, np.float32(c.score).tobytes(),
                 np.array(c.zbar_ij, np.float64).tobytes()) for c in v]
            for k, v in results.items()}
    identical = bits[True] == bits[False]
    n_constraints = len(results[True])
    print(json.dumps({
        "metric": "cb2d_device_submaps", "submaps": args.submaps, "nodes": args.nodes,
        "pairs": args.submaps * args.nodes, "constraints": n_constraints, "reps": args.reps,
        "cropped_cells": [list(c.read().cells.shape[::-1]) for c in crops],
        "crop_to_stack_ms": {"device_submaps": float(np.median(finish_ms[True])),
                             "host_roundtrip": float(np.median(finish_ms[False]))},
        "constraints_per_s": {"device_submaps": n_constraints / float(np.median(drain_s[True])),
                              "host_roundtrip": n_constraints / float(np.median(drain_s[False]))},
        "drain_ms": {"device_submaps": 1e3 * float(np.median(drain_s[True])),
                     "host_roundtrip": 1e3 * float(np.median(drain_s[False]))},
        "identical": identical, "card": card()}))
    for h in active + crops:
        h.close()
    if not identical:
        raise SystemExit("the two paths gave different constraints")


if __name__ == "__main__":
    main()
