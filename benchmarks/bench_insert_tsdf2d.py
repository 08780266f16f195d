"""Inserting scans into device-resident 2D TSDF submap grids (TSDFRangeDataInserter2D on the
device, normal estimation and growth included) versus what it replaces: inserting on the host and
re-uploading both arrays of both grids.

Workload: the local-SLAM sequence of bench_insert2d.py (`--scans` seeded 1081-beam / 270 degree
scans in the synthetic 50 m floor plan at 5 cm), with trajectory_builder_2d.lua's
tsdf_range_data_inserter options (truncation 0.3 m, maximum weight 10, normals from 4 samples
within 0.5 m, projection onto the normal, both kernel bandwidths 0.5; `--free-space` turns
update_free_space on).  The TSDF inserter reads the returns only.  As ActiveSubmaps2D does with
num_range_data = 90, a new submap starts every 90 scans and every scan goes into the (up to) two
active submaps; grids start as CreateGrid's 100 x 100 cells and grow.

Prints one JSON line: per scan, the device inserts' device and wall ms and the share of the wall
time the device time does not cover (host preparation: growth, sort, normals, ray records,
launches and the synchronisation); the host path's ms (the C++ restatement's two inserts, and
csm_rt_grid2d_update_tsdf of both grids, or their re-creation when a grid grew); whether every
grid is bit-equal to the restatement's; and the card's name, power limit and clocks.

    python benchmarks/bench_insert_tsdf2d.py --scans 360 [--free-space]
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
from benchmarks.bench_insert2d import NUM_RANGE_DATA, card, range_data, trajectory  # noqa: E402
from cartographer_b200 import scan_matching as sm  # noqa: E402
from tests import insert_tsdf2d_oracle as O  # noqa: E402

TRUNCATION, MAX_WEIGHT = 0.3, 10.0


class Submap:
    def __init__(self, origin):
        self.ora = O.TsdfGrid.create_grid(origin[:2], 0.05, TRUNCATION, MAX_WEIGHT)
        res, max_x, max_y, nx, ny = self.ora.limits
        self.dev = sm.RealTimeGrid2D.empty_tsdf(res, max_x, max_y, TRUNCATION, MAX_WEIGHT, nx, ny)
        self.twin = None   # the host path's handle, refreshed from the restatement's cells
        self.count = 0


def equal(dev, ora):
    st = dev.read()
    tsd, weight = ora.arrays()
    return bool(np.array_equal(st.cells, tsd) and np.array_equal(st.weight_cells, weight) and
                (st.resolution, st.max_x, st.max_y) == ora.limits[:3] and
                st.known_cells_box == ora.known_box)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=360)
    ap.add_argument("--free-space", action="store_true")
    args = ap.parse_args()
    if sm.device_count() < 1:
        raise SystemExit("no CUDA device: nothing to measure")
    spec, occ = synthetic.make_grid2d(3, size_cells=1000)
    rng = np.random.RandomState(11)
    poses = trajectory(occ, spec, rng, args.scans)
    opts = sm.TSDFRangeDataInserterOptions2D(update_free_space=args.free_space)
    dev_ins = sm.TSDFRangeDataInserter2D(opts)
    ora_ins = O.TsdfInserter(opts)
    active = []
    dev_ms, wall_ms, host_ms, upload_ms, n_returns, regrown = [], [], [], [], [], 0
    ok = True
    for k, pose in enumerate(poses):
        origin, returns, _ = range_data(occ, spec, pose, seed=k)
        n_returns.append(len(returns))
        if not active or active[-1].count == NUM_RANGE_DATA:   # ActiveSubmaps2D::InsertRangeData
            if len(active) == 2:
                done = active.pop(0)
                ok &= equal(done.dev, done.ora)
                done.dev.close()
                if done.twin is not None:
                    done.twin.close()
            active.append(Submap(origin))
        t0 = time.perf_counter()
        d = 0.0
        for s in active:
            dev_ins.Insert(origin, returns, s.dev)
            d += dev_ins.last_stats["device_ms"]
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        dev_ms.append(d)
        t0 = time.perf_counter()
        for s in active:
            ok &= ora_ins.insert(origin, returns, s.ora)
        host_ms.append((time.perf_counter() - t0) * 1e3)
        arrays = [(s, s.ora.arrays(), s.ora.limits) for s in active]   # the host owns them anyway
        t0 = time.perf_counter()
        for s, (tsd, weight), (r, mx, my, nx, ny) in arrays:
            if s.twin is not None and s.twin.shape == tsd.shape:
                s.twin.update(tsd, weight)
            else:
                if s.twin is not None:
                    s.twin.close()
                    regrown += 1
                s.twin = sm.RealTimeGrid2D(sm.TSDF2DSpec(tsd, weight, r, mx, my, TRUNCATION,
                                                         MAX_WEIGHT))
        upload_ms.append((time.perf_counter() - t0) * 1e3)
        for s in active:
            s.count += 1
    for s in active:
        ok &= equal(s.dev, s.ora)
    med = lambda v: float(np.median(v)) if len(v) else None  # noqa: E731
    total = lambda v: float(np.sum(v))  # noqa: E731
    print(json.dumps({
        "metric": "insert_tsdf2d", "scans": args.scans, "beams": 1081,
        "update_free_space": bool(args.free_space), "mean_returns": float(np.mean(n_returns)),
        "device_ms_per_scan": med(dev_ms), "wall_ms_per_scan": med(wall_ms),
        "host_prep_share_of_wall": 1.0 - total(dev_ms) / total(wall_ms),
        "host_insert_ms_per_scan": med(host_ms), "host_upload_ms_per_scan": med(upload_ms),
        "host_path_ms_per_scan": med(np.add(host_ms, upload_ms)),
        "totals_ms": {"device": total(dev_ms), "device_wall": total(wall_ms),
                      "host_insert": total(host_ms), "host_upload": total(upload_ms)},
        "host_handle_recreations": regrown,
        "final_active_cells": [list(s.dev.shape[::-1]) for s in active],
        "bit_equal_to_restatement": bool(ok), "card": card()}))
    for s in active:
        s.dev.close()
        if s.twin is not None:
            s.twin.close()
    dev_ins.close()
    if not ok:
        raise SystemExit("device grids differ from the CPU restatement")


if __name__ == "__main__":
    main()
