"""Where the time of one config-2 step goes (bench.py --config 2: 64 MatchFullSubmap
searches in one batch, the same seeds and the same call as the timed leg of bench.py).

  python -m benchmarks.step_breakdown2d --out DIR [--steps 3 --warmup 3]

Three passes, each in its own process so that none of them perturbs another:
  1. `CSM_TIMING` host phases of the engine (every phase ends in a stream synchronise,
     so the phases add up to more than an untimed step);
  2. untimed steps with a host clock, for the reference step time;
  3. a torch.profiler trace with CUDA activities (DIR/trace_step2d.json), from which it
     derives per-kernel device time, the device-idle gaps between activities, grouped
     by the pair of activities around them, and the host time before the first and
     after the last device activity of each step.
Prints one JSON line (also written to DIR/step_breakdown2d.json).
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _setup(total_steps):
    import bench
    from cartographer_b200 import scan_matching as sm
    grid, scans = bench.make_world(0, total_steps * bench.MATCHES_PER_STEP)
    opts = sm.FastCorrelativeScanMatcherOptions2D(bench.LIN, bench.ANG, bench.DEPTH)
    matcher = sm.FastCorrelativeScanMatcher2D(grid, opts, device=0)
    clouds = [sm.DeviceCloud(s, device=0) for s in scans]
    ctx = sm.MultiGpuContext(1, 0, 0, None)
    n = bench.MATCHES_PER_STEP
    jobs = np.zeros(n, sm.JOB2D_DTYPE)
    jobs["cloud_index"] = np.arange(n)
    jobs["full_submap"] = 1
    jobs["min_score"] = bench.MIN_SCORE

    def step(it):
        return sm.match_batch_sharded(ctx, [matcher], clouds[it * n:(it + 1) * n], jobs,
                                      bench.LIN, bench.ANG, np.zeros(1, np.int32))
    return step


def _child(mode, warmup, steps, out):
    import torch
    step = _setup(warmup + steps)
    for it in range(warmup):
        step(it)
    torch.cuda.synchronize()
    if mode == "timing":     # CSM_TIMING is set: the engine prints its phases to stderr
        print("----- timed -----", file=sys.stderr, flush=True)
        for it in range(warmup, warmup + steps):
            step(it)
        return
    if mode == "plain":
        ms, stats = [], []
        for it in range(warmup, warmup + steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, st = step(it)
            ms.append(1e3 * (time.perf_counter() - t0))
            stats.append(st)
        print(json.dumps({"step_ms": ms, "device_ms": [s["device_ms"] for s in stats],
                          "host_syncs": [s["host_syncs"] for s in stats],
                          "candidates_scored": [s["candidates_scored"] for s in stats]}))
        return
    from torch.profiler import ProfilerActivity, profile, record_function
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for it in range(warmup, warmup + steps):
            torch.cuda.synchronize()
            with record_function("step2d_%d" % it):
                step(it)
    prof.export_chrome_trace(os.path.join(out, "trace_step2d.json"))


def _run_child(mode, args, env_extra=None):
    env = dict(os.environ)
    env.update(env_extra or {})
    cmd = [sys.executable, "-m", "benchmarks.step_breakdown2d", "--child", mode,
           "--warmup", str(args.warmup), "--steps", str(args.steps), "--out", args.out]
    p = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-4000:] + p.stderr[-4000:])
        raise RuntimeError("step_breakdown2d: the %s pass failed" % mode)
    return p


def _timing_phases(stderr):
    tail = stderr.split("----- timed -----", 1)[-1]
    per = defaultdict(list)
    for m in re.finditer(r"\[csm timing\] (.+?)\s+([0-9.]+) ms", tail):
        per[m.group(1).strip()].append(float(m.group(2)))
    return {k: {"median_ms": float(np.median(v)), "calls": len(v)} for k, v in per.items()}


def _trace_summary(path):
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    dev_cats = {"kernel", "gpu_memcpy", "gpu_memset"}
    steps = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") == "user_annotation"
                    and str(e.get("name", "")).startswith("step2d_")), key=lambda e: e["ts"])
    dev = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") in dev_cats),
                 key=lambda e: e["ts"])
    out = []
    for s in steps:
        t0, t1 = s["ts"], s["ts"] + s["dur"]
        acts = [e for e in dev if t0 <= e["ts"] < t1]
        if not acts:
            continue
        per_kernel = defaultdict(lambda: [0, 0.0])
        for e in acts:
            nm = re.sub(r"\(.*", "", e["name"]).replace("void ", "").replace("csm::", "")
            per_kernel[nm][0] += 1
            per_kernel[nm][1] += e["dur"] / 1e3
            e["_n"] = nm
        gaps = defaultdict(lambda: [0, 0.0])
        busy_end = acts[0]["ts"] + acts[0]["dur"]
        prev = acts[0]["_n"]
        busy = acts[0]["dur"]
        for e in acts[1:]:
            g = e["ts"] - busy_end
            if g > 0:
                key = "%s -> %s" % (prev, e["_n"])
                gaps[key][0] += 1
                gaps[key][1] += g / 1e3
                busy += e["dur"]
            else:
                busy += max(0.0, e["ts"] + e["dur"] - busy_end)
            if e["ts"] + e["dur"] >= busy_end:
                busy_end = e["ts"] + e["dur"]
                prev = e["_n"]
        top_gaps = sorted(gaps.items(), key=lambda kv: -kv[1][1])[:12]
        out.append({
            "step_ms": s["dur"] / 1e3,
            "host_before_first_device_ms": (acts[0]["ts"] - t0) / 1e3,
            "host_after_last_device_ms": (t1 - busy_end) / 1e3,
            "device_span_ms": (busy_end - acts[0]["ts"]) / 1e3,
            "device_busy_ms": busy / 1e3,
            "device_idle_in_span_ms": (busy_end - acts[0]["ts"] - busy) / 1e3,
            "activities": len(acts),
            "kernels_ms": {k: {"n": v[0], "ms": round(v[1], 4)}
                           for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1][1])},
            "largest_idle_gaps_ms": {k: {"n": v[0], "ms": round(v[1], 4)} for k, v in top_gaps},
        })
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--child", default=None)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.child:
        _child(args.child, args.warmup, args.steps, args.out)
        return
    phases = _timing_phases(_run_child("timing", args, {"CSM_TIMING": "1"}).stderr)
    plain = json.loads(_run_child("plain", args).stdout.strip().splitlines()[-1])
    _run_child("trace", args)
    steps = _trace_summary(os.path.join(args.out, "trace_step2d.json"))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    line = {"gpu": q.stdout.strip(), "phases": phases, "plain": plain, "trace_steps": steps}
    with open(os.path.join(args.out, "step_breakdown2d.json"), "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
