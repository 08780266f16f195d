"""2D local SLAM per scan: the one-call device path (local_slam.LocalTrajectoryBuilder2D over
csm_local_slam2d) against the recipe (the same scans through the single-stage public calls,
benchmarks/local_slam2d_recipe.py), over bench_insert2d.py's world and trajectory.

For each configuration (scan size x online matching) both builders take the same scans; which
one runs first alternates scan by scan.  Reported per path: median and p99 wall ms per scan
(host clock around a call that ends in a stream synchronisation), the one-call path's median
device ms (CUDA events inside the calls) and host syncs per matched scan.  At the end every
active submap's cells, limits and box and every pose are compared bit for bit.

The recipe's per-point transforms are vectorised numpy (float32); its wall time is what a caller
pays today for the glue.  Usage: python benchmarks/bench_local_slam2d.py [--scans N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks import local_slam2d_recipe as R  # noqa: E402
from cartographer_b200 import local_slam as L  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def dense(hw, factor):
    """A denser scan: every beam repeated `factor` times at slightly shifted angles."""
    if factor == 1:
        return hw
    out = []
    for k in range(factor):
        a = 1e-4 * k
        c, s = np.cos(a), np.sin(a)
        p = hw.copy()
        p[:, 0], p[:, 1] = c * hw[:, 0] - s * hw[:, 1], s * hw[:, 0] + c * hw[:, 1]
        out.append(p)
    r = np.concatenate(out).astype(np.float32)
    r[:, 3] = np.linspace(-0.05, 0.0, len(r), dtype=np.float32)
    return r


def one(options, scans, factor, warmup):
    spec, occ, traj = R.world(scans + warmup)
    ex_a, ex_b = R.FakeExtrapolator(traj), R.FakeExtrapolator(traj)
    b = L.LocalTrajectoryBuilder2D(options, ex_a)
    rec = R.Recipe(options, ex_b)
    origins = np.zeros((1, 3), np.float32)
    wall_a, wall_b, dev, syncs = [], [], [], []
    poses_equal = True
    for k in range(scans + warmup):
        time_s = (k + 1) * 0.1
        hw = dense(R.scan_at(spec, occ, traj[k + 1], seed=k), factor)
        oi = np.zeros(len(hw), np.int32)
        order = (0, 1) if k % 2 == 0 else (1, 0)
        res = [None, None]
        ms = [0.0, 0.0]
        for which in order:
            t0 = time.perf_counter()
            if which == 0:
                res[0] = b.AddRangeData(time_s, hw, origins, oi)
            else:
                res[1] = rec.add(time_s, hw, origins, oi)
            ms[which] = 1e3 * (time.perf_counter() - t0)
        if k < warmup:
            continue
        wall_a.append(ms[0])
        wall_b.append(ms[1])
        if res[0] is not None:
            st = b.last_stats
            dev.append(st["match"]["device_ms"] + st.get("insert", {}).get("device_ms", 0.0))
            syncs.append(st["match"]["host_syncs"] + st.get("insert", {}).get("host_syncs", 0))
            poses_equal &= bool(np.array_equal(res[0].pose_estimate_2d, res[1]["pose2d"]))
    try:
        R.grids_equal(b.active_submaps, rec.submaps)
        grids_equal = True
    except AssertionError:
        grids_equal = False
    b.close()
    pct = lambda v, q: float(np.percentile(v, q))  # noqa: E731
    return dict(one_call_median_ms=pct(wall_a, 50), one_call_p99_ms=pct(wall_a, 99),
                recipe_median_ms=pct(wall_b, 50), recipe_p99_ms=pct(wall_b, 99),
                one_call_device_median_ms=pct(dev, 50) if dev else None,
                one_call_host_syncs_median=pct(syncs, 50) if syncs else None,
                poses_equal=poses_equal, grids_equal=grids_equal)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    out = {"card": card(), "scans": args.scans, "configs": []}
    for factor, label in ((1, "1081 beams"), (16, "17296 beams")):
        for online in (False, True):
            o = L.LocalTrajectoryBuilderOptions2D(min_range=0.2,
                                                  use_online_correlative_scan_matching=online)
            o.submaps_options = sm.SubmapsOptions2D(num_range_data=90)
            r = one(o, args.scans, factor, args.warmup)
            r.update(scan=label, online=online)
            out["configs"].append(r)
            print(json.dumps(r), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
