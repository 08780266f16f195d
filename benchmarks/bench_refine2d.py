"""Post-match refinement throughput (CeresScanMatcher2D, constraint_builder_2d.cc:245-249):
`jobs` found matches of 1081-beam node scans refined against 1000 x 1000 submap grids in ONE
csm_ceres_match2d_batch launch (host clouds: their H2D is inside the timed call), beside the
oracle's CPU restatement on the host threads.  Prints one JSON line.

  python -m benchmarks.bench_refine2d [--jobs 2000] [--submaps 4] [--iterations 10]
                                      [--grid {probability,tsdf}]

--grid tsdf refines against TSDF2D submaps (synthetic.make_tsdf2d, TSDFMatchCostFunction2D);
its CPU baseline is the numpy restatement tests/tsdf2d_oracle.py on a smaller sample.
"""
import argparse
import json
import os
import time

import numpy as np

from benchmarks import synthetic


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=2000)
    ap.add_argument("--submaps", type=int, default=4)
    ap.add_argument("--iterations", type=int, default=10)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--grid", choices=("probability", "tsdf"), default="probability")
    args = ap.parse_args()
    from cartographer_b200 import scan_matching as sm
    worlds = []
    for s in range(args.submaps):
        if args.grid == "tsdf":
            grid, occ = synthetic.make_tsdf2d(900 + s, size_cells=1000)
        else:
            grid, occ = synthetic.make_grid2d(900 + s, size_cells=1000)
        rng = np.random.RandomState(900 + s)
        scans = []
        for k in range(4):
            pose = np.asarray(synthetic.random_free_pose(occ, grid, rng, margin_cells=40))
            scans.append((pose, synthetic.cast_scan(occ, grid, pose, beams=1081, seed=k)))
        worlds.append((grid, sm.RealTimeGrid2D(grid), scans))
    rng = np.random.RandomState(1)
    targets, inits, clouds, grids, cpu_jobs = [], [], [], [], []
    for j in range(args.jobs):
        grid, dev, scans = worlds[j % args.submaps]
        pose, scan = scans[(j // args.submaps) % len(scans)]
        init = pose + np.array([rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05),
                                rng.uniform(-0.01, 0.01)])
        targets.append(init[:2])
        inits.append(init)
        clouds.append(scan)
        grids.append(dev)
        cpu_jobs.append((grid, scan, init))
    opts = sm.CeresScanMatcherOptions2D(max_num_iterations=args.iterations)
    m = sm.CeresScanMatcher2D(opts)
    m.MatchBatch(targets[:8], inits[:8], clouds[:8], grids[:8])   # warm-up
    wall, dev_ms = [], []
    for _ in range(args.repeat):
        t0 = time.perf_counter()
        poses, sums = m.MatchBatch(targets, inits, clouds, grids)
        wall.append(time.perf_counter() - t0)
        dev_ms.append(m.last_stats["device_ms"])
    out = {"metric": "refinements_per_sec", "jobs": args.jobs, "points_per_scan": 1081,
           "grid": "1000x1000", "grid_type": args.grid, "max_num_iterations": args.iterations,
           "value": args.jobs / float(np.median(wall)), "wall_ms": 1e3 * float(np.median(wall)),
           "device_ms": float(np.median(dev_ms)),
           "mean_iterations": float(np.mean([s["iterations"] for s in sums])),
           "h2d_bytes": int(sum(c.nbytes for c in clouds))}
    if not args.no_cpu_baseline and args.grid == "tsdf":
        from tests import tsdf2d_oracle
        ogs = {id(g): tsdf2d_oracle.TSDF2D.from_spec(g) for g, _, _ in worlds}
        sample = cpu_jobs[:64]
        t0 = time.perf_counter()
        want = [tsdf2d_oracle.match(ogs[id(g)], scan, init[:2], init,
                                    max_num_iterations=args.iterations)
                for g, scan, init in sample]
        secs = time.perf_counter() - t0
        worst = max(float(np.abs(poses[i] - w["pose"]).max()) for i, w in enumerate(want))
        out["cpu_baseline"] = {"value": len(sample) / secs, "unit": "refinements/s", "cores": 1,
                               "kind": "numpy restatement (test oracle), not a port",
                               "sample": "%d of the jobs, %.2f s wall" % (len(sample), secs)}
        out["parity_checked"] = sum(float(np.abs(poses[i] - w["pose"]).max()) <= 1e-7
                                    for i, w in enumerate(want))
        out["max_abs_pose_difference"] = worst
    elif not args.no_cpu_baseline:
        from concurrent.futures import ThreadPoolExecutor
        from oracle import pyoracle as oracle
        oracle.build()
        threads = max(1, min(os.cpu_count() or 1, 64))
        # ~2 ms per refinement and thread: enough jobs for a wall time well above thread start-up
        sample = (cpu_jobs * (1 + 4096 // max(1, len(cpu_jobs))))[:4096]
        ogs = {id(g): oracle.Grid2D(g.cells, g.resolution, g.max_x, g.max_y) for g, _, _ in worlds}

        def one(job):
            g, scan, init = job
            return oracle.ceres2d_match(ogs[id(g)], scan, init[:2], init,
                                        max_num_iterations=args.iterations)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(threads) as ex:
            want = list(ex.map(one, sample))
        secs = time.perf_counter() - t0
        worst = max(float(np.abs(poses[i % args.jobs] - w["pose"]).max())
                    for i, w in enumerate(want))
        out["cpu_baseline"] = {"value": len(sample) / secs, "unit": "refinements/s",
                               "cores": threads, "kind": "port",
                               "sample": "%d of the jobs, %.2f s wall" % (len(sample), secs)}
        out["parity_checked"] = len(sample)
        out["max_abs_pose_difference"] = worst
    print(json.dumps(out))


if __name__ == "__main__":
    main()
