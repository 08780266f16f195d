"""3D post-match refinement throughput (CeresScanMatcher3D, constraint_builder_3d.cc:265-275)
at BASELINE config-5 size: node scans of 64 rings x 1024 azimuths (~64 k points + the
low-resolution cloud) refined against a submap's 10 cm / 45 cm hybrid grids, `jobs` matches in
ONE csm_ceres_match3d_batch launch (host clouds: their H2D is inside the timed call), beside
the oracle's CPU restatement on the host threads.  Prints one JSON line.

  python -m benchmarks.bench_refine3d [--jobs 128] [--rings 64] [--az 1024] [--intensity]

--intensity gives the high-resolution cloud per-point intensities and the submap an intensity
grid over its 10 cm voxels (seeded per-surface intensities, benchmarks/synthetic.py), and
refines with the high-resolution pair's IntensityCostFunction3D block under HuberLoss, with
trajectory_builder_3d.lua's intensity_cost_function_options_0 (weight 0.5, huber_scale 0.3)
and an intensity threshold of 100.
"""
import argparse
import json
import math
import os
import time

import numpy as np

from benchmarks import synthetic


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=128)
    ap.add_argument("--rings", type=int, default=64)
    ap.add_argument("--az", type=int, default=1024)
    ap.add_argument("--nodes", type=int, default=3)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--intensity", action="store_true")
    args = ap.parse_args()
    from cartographer_b200 import scan_matching as sm
    t0 = time.perf_counter()
    hi, lo, _, world = synthetic.make_submap3d(40, 40.0, args.rings, args.az, 20.0)
    rng = np.random.RandomState(540)
    nodes = [synthetic.make_node3d(world, rng, args.rings, args.az, 20.0, seed=7000 + k, jitter=0.15)
             for k in range(args.nodes)]
    gen_s = time.perf_counter() - t0
    dhi, dlo = sm.DeviceHybridGrid(hi), sm.DeviceHybridGrid(lo)
    intensity_options = (0.5, 0.3, 100.0)
    if args.intensity:
        ispec = synthetic.make_intensity_grid3d(hi, world, 40)
        dint = sm.DeviceIntensityGrid(ispec)
        for k, n in enumerate(nodes):
            n["intensities"] = synthetic.node_intensities(world, n, 7000 + k)
    rng = np.random.RandomState(2)
    targets, inits, pairs, cpu_jobs = [], [], [], []
    for j in range(args.jobs):
        n = nodes[j % len(nodes)]
        init = n["pose"].copy()
        init[:3] += rng.uniform(-0.05, 0.05, 3)
        yaw = 2 * math.atan2(n["pose"][6], n["pose"][3]) + rng.uniform(-0.01, 0.01)
        init[3:] = [math.cos(yaw / 2), 0, 0, math.sin(yaw / 2)]
        targets.append(init[:3])
        inits.append(init)
        if args.intensity:
            pairs.append([(n["cloud"], dhi, dint, n["intensities"]), (n["low"], dlo)])
        else:
            pairs.append([(n["cloud"], dhi), (n["low"], dlo)])
        cpu_jobs.append((n, init))
    opts = sm.CeresScanMatcherOptions3D()
    if args.intensity:
        opts.intensity_cost_function_options_0 = sm.IntensityCostFunctionOptions(*intensity_options)
    m = sm.CeresScanMatcher3D(opts)
    m.MatchBatch(targets[:2], inits[:2], pairs[:2])   # warm-up
    wall, dev_ms = [], []
    for _ in range(args.repeat):
        t0 = time.perf_counter()
        poses, sums = m.MatchBatch(targets, inits, pairs)
        wall.append(time.perf_counter() - t0)
        dev_ms.append(m.last_stats["device_ms"])
    npts = int(np.mean([len(n["cloud"]) + len(n["low"]) for n in nodes]))
    out = {"metric": "refinements_per_sec", "jobs": args.jobs, "points_per_job": npts,
           "grids": "hybrid 0.10 m + 0.45 m, 40 m building" +
                    (" + intensity 0.10 m" if args.intensity else ""),
           "max_num_iterations": 10,
           "value": args.jobs / float(np.median(wall)), "wall_ms": 1e3 * float(np.median(wall)),
           "device_ms": float(np.median(dev_ms)),
           "mean_iterations": float(np.mean([s["iterations"] for s in sums])),
           "h2d_bytes": int(sum(12 * (len(n["cloud"]) + len(n["low"])) +
                                (4 * len(n["cloud"]) if args.intensity else 0)
                                for n, _ in cpu_jobs)),
           "host_generation_s": gen_s}
    if not args.no_cpu_baseline:
        from concurrent.futures import ThreadPoolExecutor
        from oracle import pyoracle as oracle
        oracle.build()
        threads = max(1, min(os.cpu_count() or 1, 64))
        ohi = oracle.HybridGrid(hi.resolution, hi.indices, hi.values)
        olo = oracle.HybridGrid(lo.resolution, lo.indices, lo.values)
        sample = cpu_jobs[:max(threads, min(args.jobs, 128))]

        if args.intensity:   # the intensity block's restatement lives with the tests
            from tests import intensity3d_oracle
            oint = intensity3d_oracle.IntensityHybridGrid(ispec.resolution, ispec.indices,
                                                          ispec.sums, ispec.counts)

        def one(job):
            n, init = job
            if args.intensity:
                return intensity3d_oracle.match(
                    [(n["cloud"], ohi, oint, n["intensities"]), (n["low"], olo)], init[:3], init,
                    [intensity_options, None])
            return oracle.ceres3d_match([(n["cloud"], ohi), (n["low"], olo)], init[:3], init)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(threads) as ex:
            want = list(ex.map(one, sample))
        secs = time.perf_counter() - t0
        worst = max(float(np.abs(poses[i] - w["pose"]).max()) for i, w in enumerate(want))
        same_iterations = sum(int(sums[i]["iterations"] == w["iterations"]) for i, w in enumerate(want))
        out["cpu_baseline"] = {"value": len(sample) / secs, "unit": "refinements/s",
                               "cores": threads,
                               "kind": "numpy restatement" if args.intensity else "port",
                               "sample": "%d of the jobs, %.2f s wall" % (len(sample), secs)}
        out["parity_checked"] = len(sample)
        out["max_abs_pose_difference"] = worst
        out["same_iteration_count"] = same_iterations
    print(json.dumps(out))


if __name__ == "__main__":
    main()
