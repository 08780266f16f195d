"""Inserting scans into device-resident 2D submap grids (ProbabilityGridRangeDataInserter2D on
the device, growth and cropping included) versus what it replaces: inserting on the host and
re-uploading the grids, then cropping on the host and uploading the crop into a new stack.

Workload: a local-SLAM sequence of `--scans` 1081-beam / 270 degree scans (30 m max range,
synthetic 50 m floor plan at 5 cm from benchmarks/synthetic.py, a seeded trajectory through
its free space).  Beams that reach the maximum range become misses 5 m along the beam
(missing_data_ray_length).  As ActiveSubmaps2D does with num_range_data = 90, a new submap
starts every 90 scans, every scan goes into the (up to) two active submaps, and a submap
finishes after its 180th scan: it is cropped (Submap2D::Finish) and turned into a depth-7
precomputation stack (ConstraintBuilder2D's FastCorrelativeScanMatcher2D).  Submap grids start
as ActiveSubmaps2D::CreateGrid's 100 x 100 cells and grow.

Prints one JSON line: per scan, the device inserts' device and wall ms, and the host path's
ms (the C++ restatement's two inserts, and csm_rt_grid2d_update of both grids, or their
re-creation when a grid grew); per finished submap, crop + stack from the device handle
against the host crop + csm_stack2d_create; whether every grid and crop is bit-equal to the
restatement's; and the card's name, power limit and clocks.

    python benchmarks/bench_insert2d.py --scans 360
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
from cartographer_b200 import scan_matching as sm  # noqa: E402
from tests import insert2d_oracle as O  # noqa: E402

NUM_RANGE_DATA = 90
MAX_RANGE = 30.0
MISSING_DATA_RAY_LENGTH = 5.0


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.mem,"
                          "clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def trajectory(occ, spec, rng, n):
    """Seeded poses along a walk through free space (0.1 m and a few degrees per scan)."""
    pose = synthetic.random_free_pose(occ, spec, rng, margin_cells=60)
    poses = []
    heading = pose[2]
    ny, nx = occ.shape
    while len(poses) < n:
        step = np.array([0.1 * math.cos(heading), 0.1 * math.sin(heading)])
        nxt = pose[:2] + step
        cx = int((spec.max_y - nxt[1]) / spec.resolution)
        cy = int((spec.max_x - nxt[0]) / spec.resolution)
        blocked = not (20 <= cx < nx - 20 and 20 <= cy < ny - 20) or \
            occ[max(0, cy - 8):cy + 9, max(0, cx - 8):cx + 9].any()
        if blocked:
            heading += rng.uniform(0.6, 2.5)
            continue
        heading += rng.normal(0.0, 0.05)
        pose = np.array([nxt[0], nxt[1], heading])
        poses.append(pose)
    return poses


def range_data(occ, spec, pose, seed):
    pts = synthetic.cast_scan(occ, spec, pose, beams=1081, max_range=MAX_RANGE, seed=seed)
    rng_ = np.hypot(pts[:, 0], pts[:, 1])
    far = rng_ >= MAX_RANGE - 1e-3
    local = pts.astype(np.float64)
    local[far, :2] *= (MISSING_DATA_RAY_LENGTH / rng_[far])[:, None]
    c, s = math.cos(pose[2]), math.sin(pose[2])
    w = np.stack([c * local[:, 0] - s * local[:, 1] + pose[0],
                  s * local[:, 0] + c * local[:, 1] + pose[1], np.zeros(len(local))],
                 1).astype(np.float32)
    return np.float32([pose[0], pose[1], 0.0]), w[~far], w[far]


class Submap:
    def __init__(self, origin, ins):
        self.ora = O.Grid.create_grid(origin[:2], 0.05)
        res, max_x, max_y, nx, ny = self.ora.limits
        self.dev = sm.RealTimeGrid2D.empty(res, max_x, max_y, nx, ny)
        self.twin = None   # the host path's handle, refreshed from the restatement's cells
        self.count = 0


def equal(dev, ora):
    st = dev.read()
    return bool(np.array_equal(st.cells, ora.cells) and
                (st.resolution, st.max_x, st.max_y) == ora.limits[:3] and
                st.known_cells_box == ora.known_box)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=360)
    ap.add_argument("--depth", type=int, default=7)
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    spec, occ = synthetic.make_grid2d(3, size_cells=1000)
    rng = np.random.RandomState(11)
    poses = trajectory(occ, spec, rng, args.scans)
    opts = sm.ProbabilityGridRangeDataInserterOptions2D(0.55, 0.49, True)   # trajectory_builder_2d.lua
    dev_ins = sm.ProbabilityGridRangeDataInserter2D(opts)
    ora_ins = O.Inserter(0.55, 0.49, True)
    fast = sm.FastCorrelativeScanMatcherOptions2D(7.0, math.radians(30.0), args.depth)
    active, finished = [], []
    dev_ms, wall_ms, host_ms, upload_ms, n_returns, regrown = [], [], [], [], [], 0
    finish = {"device_crop_stack_ms": [], "host_crop_stack_ms": [], "crop_cells": []}
    ok = True
    for k, pose in enumerate(poses):
        origin, returns, misses = range_data(occ, spec, pose, seed=k)
        n_returns.append(len(returns))
        if not active or active[-1].count == NUM_RANGE_DATA:   # ActiveSubmaps2D::InsertRangeData
            if len(active) == 2:
                done = active.pop(0)
                # Submap2D::Finish + the constraint builder's matcher, both ways
                t0 = time.perf_counter()
                crop = done.dev.ComputeCroppedGrid()
                m_dev = sm.FastCorrelativeScanMatcher2D.from_device_grid(crop, fast)
                finish["device_crop_stack_ms"].append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                ocrop = done.ora.crop()
                r, mx, my, nx, ny = ocrop.limits
                m_host = sm.FastCorrelativeScanMatcher2D(
                    synthetic.GridSpec(ocrop.cells, r, mx, my), fast)
                finish["host_crop_stack_ms"].append((time.perf_counter() - t0) * 1e3)
                finish["crop_cells"].append([nx, ny])
                ok &= equal(crop, ocrop)
                ok &= all(np.array_equal(m_dev.precomputation_grid(lv), m_host.precomputation_grid(lv))
                          for lv in (0, args.depth - 1))
                finished.append(done)
                for h in (crop, m_dev, m_host, done.dev):
                    h.close()
                if done.twin is not None:
                    done.twin.close()
            active.append(Submap(origin, dev_ins))
        t0 = time.perf_counter()
        d = 0.0
        for s in active:
            dev_ins.Insert(origin, returns, s.dev, misses)
            d += dev_ins.last_stats["device_ms"]
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        dev_ms.append(d)
        t0 = time.perf_counter()
        for s in active:
            ora_ins.insert(origin, returns, s.ora, misses)
        host_ms.append((time.perf_counter() - t0) * 1e3)
        cells = [(s, s.ora.cells, s.ora.limits) for s in active]   # the host owns them anyway
        t0 = time.perf_counter()
        for s, c, (r, mx, my, nx, ny) in cells:
            if s.twin is not None and s.twin.shape == c.shape:
                s.twin.update(c)
            else:
                if s.twin is not None:
                    s.twin.close()
                    regrown += 1
                s.twin = sm.RealTimeGrid2D(synthetic.GridSpec(c, r, mx, my))
        upload_ms.append((time.perf_counter() - t0) * 1e3)
        for s in active:
            s.count += 1
    for s in active:
        ok &= equal(s.dev, s.ora)
    med = lambda v: float(np.median(v)) if len(v) else None  # noqa: E731
    total = lambda v: float(np.sum(v))  # noqa: E731
    print(json.dumps({
        "metric": "insert2d", "scans": args.scans, "beams": 1081,
        "mean_returns": float(np.mean(n_returns)), "submaps_finished": len(finish["crop_cells"]),
        "device_ms_per_scan": med(dev_ms), "wall_ms_per_scan": med(wall_ms),
        "host_insert_ms_per_scan": med(host_ms), "host_upload_ms_per_scan": med(upload_ms),
        "host_path_ms_per_scan": med(np.add(host_ms, upload_ms)),
        "totals_ms": {"device": total(dev_ms), "device_wall": total(wall_ms),
                      "host_insert": total(host_ms), "host_upload": total(upload_ms)},
        "host_handle_recreations": regrown,
        "finish_device_crop_stack_ms": med(finish["device_crop_stack_ms"]),
        "finish_host_crop_stack_ms": med(finish["host_crop_stack_ms"]),
        "finish_crop_cells": finish["crop_cells"],
        "final_active_cells": [list(s.dev.shape[::-1]) for s in active],
        "bit_equal_to_restatement": ok, "card": card()}))
    for s in active:
        s.dev.close()
        if s.twin is not None:
            s.twin.close()
    dev_ins.close()
    if not ok:
        raise SystemExit("device grids differ from the CPU restatement")


if __name__ == "__main__":
    main()
