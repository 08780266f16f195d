"""Lifelong mapping in 2D: OverlappingSubmapsTrimmer2D's coverage pass over device-resident submap
grids (csm_trim_overlapping_submaps2d) versus the single-threaded CPU restatement of the
reference's std::map pass (tests/trimmer2d_oracle.cc).

Workload: a synthetic lifelong map of `--submaps` finished submaps (default 200 and 1000), each a
320 x 320 ProbabilityGrid at 5 cm made from cells (a disc of known cells with scattered holes),
placed along a looping trajectory that passes the same places again and again, with random yaw
and a small pose-graph correction between local and global pose, so that coverage overlaps
heavily; a few submaps share a freshness.  The device call is timed with a host clock around it
(the call ends in a stream synchronisation), `--reps` times after one warm-up; the restatement
runs once per map.  Prints one JSON line per map size with median device ms, CPU ms, entries,
coverage cells, whether trim flags and counts are equal, and the card's name and power limit.

    python benchmarks/bench_trimmer2d.py --submaps 200 1000
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

from benchmarks.bench_grid_to_proto import card  # noqa: E402

SIZE, RESOLUTION = 320, 0.05


def _pose(x, y, yaw):
    return [x, y, 0.0, math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)]


def lifelong_map(num_submaps, seed=0, size=SIZE, resolution=RESOLUTION):
    """Per submap (cells, (max_x, max_y, resolution), global pose, local pose, freshness): grids
    centred on their local pose along a loop of 12 m radius, 24 submaps per lap, so that every
    place is revisited num_submaps / 24 times."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:size, 0:size]
    disc = (xx - size / 2 + 0.5) ** 2 + (yy - size / 2 + 0.5) ** 2 < (0.45 * size) ** 2
    out = []
    for i in range(num_submaps):
        a = 2 * math.pi * i / 24 + rng.uniform(-0.1, 0.1)
        x, y = 12.0 * math.cos(a) + rng.uniform(-0.5, 0.5), 12.0 * math.sin(a) + rng.uniform(-0.5, 0.5)
        local = _pose(x, y, rng.uniform(-math.pi, math.pi))
        glob = _pose(x + rng.uniform(-0.3, 0.3), y + rng.uniform(-0.3, 0.3),
                     2 * math.atan2(local[6], local[3]) + rng.uniform(-0.05, 0.05))
        cells = np.where(disc & (rng.rand(size, size) > 0.05),
                         rng.randint(1, 32768, (size, size)), 0).astype(np.uint16)
        limits = (x + size / 2 * resolution, y + size / 2 * resolution, resolution)
        t = 1000 * i
        if i % 50 == 7:
            t = 1000 * (i - 1)   # shares its freshness with the previous submap
        out.append((cells, limits, glob, local, t))
    return out


def run(num_submaps, reps, fresh, min_area):
    from cartographer_b200 import pose_graph as P
    from cartographer_b200 import scan_matching as sm
    from benchmarks.synthetic import GridSpec
    from tests import trimmer2d_oracle as O

    m = lifelong_map(num_submaps)
    grids = [sm.RealTimeGrid2D(GridSpec(c, lim[2], lim[0], lim[1])) for c, lim, _, _, _ in m]
    poses = [P.global_frame_from_local_frame(g, loc) for _, _, g, loc, _ in m]
    first = m[0][1]
    min_cells = P.double_to_uint16(min_area / (first[2] * first[2]))
    records = [(g, p, t) for g, p, (_, _, _, _, t) in zip(grids, poses, m)]
    P.trim_overlapping_submaps2d(records, first, fresh, min_cells)   # warm-up
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        trim, counts, stats = P.trim_overlapping_submaps2d(records, first, fresh, min_cells)
        times.append((time.perf_counter() - t0) * 1e3)
    subs = []
    for (c, lim, _, _, t), p in zip(m, poses):
        ys, xs = np.nonzero(c)
        box = (int(xs.min()), int(ys.min()), int(xs.max()), int(ys.max())) if len(xs) else None
        subs.append((c, box, lim, p, t))
    t0 = time.perf_counter()
    want_trim, want_counts, want_stats = O.trim(subs, first, fresh, min_cells)
    cpu_ms = (time.perf_counter() - t0) * 1e3
    for g in grids:
        g.close()
    return {
        "submaps": num_submaps, "fresh_submaps_count": fresh, "min_covered_cells_count": min_cells,
        "device_ms": float(np.median(times)), "device_ms_min": float(np.min(times)),
        "cpu_restatement_ms": cpu_ms, "speedup": cpu_ms / float(np.median(times)),
        "entries": stats["entries"], "coverage_cells": stats["coverage_cells"],
        "device_tie_cells": stats["device_tie_cells"],
        "host_sorted_cells": stats["host_sorted_cells"], "host_syncs": stats["host_syncs"],
        "trimmed": int(trim.sum()),
        "equal": bool(np.array_equal(trim, want_trim) and np.array_equal(counts, want_counts)
                      and stats["entries"] == want_stats["entries"]
                      and stats["coverage_cells"] == want_stats["coverage_cells"]),
        "card": card(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--submaps", type=int, nargs="+", default=[200, 1000])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--fresh", type=int, default=3)
    ap.add_argument("--min-area", type=float, default=10.0)
    a = ap.parse_args()
    for n in a.submaps:
        print(json.dumps(run(n, a.reps, a.fresh, a.min_area)), flush=True)


if __name__ == "__main__":
    main()
