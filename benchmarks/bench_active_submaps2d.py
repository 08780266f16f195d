"""Inserting each scan into the active 2D submaps with one call
(csm_range_inserter2d_insert_submaps) versus one single-grid call per submap
(csm_range_inserter2d_insert), as ActiveSubmaps2D::InsertRangeData does with num_range_data = 90:
a new submap every 90 scans, every scan into the (up to) two active submaps, a submap done after
its 180th scan.

Two workloads over bench_insert2d.py's world and trajectory (30 m range, misses 5 m along the
beam): 1081-beam scans, and scans of 17 296 returns, the size of a multi-ring scan accumulated
over num_accumulated_range_data > 1 (the 1081-beam returns repeated with seeded 2 cm jitter).
Both paths keep their own grids and run in the same process, alternating which goes first
scan by scan, after a warm-up; the grids of the two paths are compared bit for bit whenever a
submap is done and at the end.

Prints one JSON line: per workload, per scan median device ms (CUDA events, summed over the
single calls) and wall ms of each path; whether every grid was bit-equal; the card's name,
power limit and clocks.

    python benchmarks/bench_active_submaps2d.py --scans 360
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
from benchmarks.bench_insert2d import card, range_data, trajectory  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402

NUM_RANGE_DATA = 90
ACCUMULATED_RETURNS = 17296
WARMUP_SCANS = 20


def scans(occ, spec, poses, accumulated):
    out = []
    for k, pose in enumerate(poses):
        origin, returns, misses = range_data(occ, spec, pose, seed=k)
        if accumulated:
            rng = np.random.RandomState(1000 + k)
            returns = np.resize(returns, (ACCUMULATED_RETURNS, 3)).copy()
            returns[:, :2] += rng.uniform(-0.02, 0.02, (ACCUMULATED_RETURNS, 2)).astype(np.float32)
        out.append((origin, returns, misses))
    return out


def same(a, b):
    x, y = a.read(), b.read()
    return bool(np.array_equal(x.cells, y.cells) and x.known_cells_box == y.known_cells_box and
                (x.resolution, x.max_x, x.max_y) == (y.resolution, y.max_x, y.max_y))


def run(data, ins):
    """Both paths over `data`; returns per-scan (device ms, wall ms) of each and bit-equality."""
    active = []   # [one-call grid, single-call grid, scans inserted]
    times = {"one_call": ([], []), "single_calls": ([], [])}
    ok = True
    for k, (origin, returns, misses) in enumerate(data):
        if not active or active[-1][2] == NUM_RANGE_DATA:
            if len(active) == 2:
                done = active.pop(0)
                ok &= same(done[0], done[1])
                done[0].close()
                done[1].close()
            lim = sm.create_grid_limits(origin[:2], 0.05)
            active.append([sm.RealTimeGrid2D.empty(*lim), sm.RealTimeGrid2D.empty(*lim), 0])

        def one_call():
            t0 = time.perf_counter()
            ins.insert_submaps([a[0] for a in active], origin, returns, misses)
            return ins.last_stats["device_ms"], (time.perf_counter() - t0) * 1e3

        def single_calls():
            d, t0 = 0.0, time.perf_counter()
            for a in active:
                ins.Insert(origin, returns, a[1], misses)
                d += ins.last_stats["device_ms"]
            return d, (time.perf_counter() - t0) * 1e3

        order = (("one_call", one_call), ("single_calls", single_calls))
        for name, fn in (order if k % 2 == 0 else order[::-1]):
            d, w = fn()
            if k >= WARMUP_SCANS:
                times[name][0].append(d)
                times[name][1].append(w)
        for a in active:
            a[2] += 1
    for a in active:
        ok &= same(a[0], a[1])
        a[0].close()
        a[1].close()
    med = lambda v: float(np.median(v))  # noqa: E731
    return {name: {"device_ms_per_scan": med(d), "wall_ms_per_scan": med(w),
                   "device_ms_p90": float(np.percentile(d, 90)),
                   "wall_ms_p90": float(np.percentile(w, 90))}
            for name, (d, w) in times.items()}, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=360)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    spec, occ = synthetic.make_grid2d(3, size_cells=1000)
    poses = trajectory(occ, spec, np.random.RandomState(11), args.scans)
    ins = sm.ProbabilityGridRangeDataInserter2D(
        sm.ProbabilityGridRangeDataInserterOptions2D(0.55, 0.49, True))   # trajectory_builder_2d.lua
    result = {"metric": "active_submaps2d", "scans": args.scans, "warmup_scans": WARMUP_SCANS,
              "num_range_data": NUM_RANGE_DATA}
    ok = True
    for name, accumulated in (("beams_1081", False), ("returns_17296", True)):
        data = scans(occ, spec, poses, accumulated)
        r, equal = run(data, ins)
        r["mean_returns"] = float(np.mean([len(d[1]) for d in data]))
        r["mean_misses"] = float(np.mean([len(d[2]) for d in data]))
        r["bit_equal"] = equal
        result[name] = r
        ok &= equal
    result["bit_equal"] = ok
    result["card"] = card()
    print(json.dumps(result))
    ins.close()
    if not ok:
        raise SystemExit("the one call and the single calls left different grids")


if __name__ == "__main__":
    main()
