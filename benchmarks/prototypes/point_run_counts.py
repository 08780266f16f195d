#!/usr/bin/env python
"""CPU study (no product code): how many scan entries the 2D matcher's kernels would walk
if every run of consecutive points with the same cell were scored once, weighted by its
length, and how many child-window words the branch step (k_expand_lattice) would then read.

Scores are sums of uint8 cells, so summing weight x value over runs gives the points' sum
exactly.  Runs are taken in beam order over the oracle's discrete scans (DiscretizeScans of
the rotated scans), and a run longer than the weight cap C is cut every C points, because
the kernels add weight x byte into packed u16 sums that hold 257 x 255 at most.

Words of the branch step are counted as in early_exit_counts.py: the expanded parents are
those of the tree with the optimum S* known; a parent stops reading once the bound rules out
all its children at an early-exit test (T from S*, "opt", or from min_score alone, "pess").
"points" tests every 128 points and reads one word per point; "entries" tests every 64
entries (a weight of at most 256 per lane between flushes with C = 4) and reads one word
per entry.

  python benchmarks/prototypes/point_run_counts.py [seed ...]     (default: seeds 0 1)
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                      # noqa: E402  (workload generator)
from early_exit_counts import BATCH, level_grid, to_score, values  # noqa: E402
from oracle import pyoracle as oracle  # noqa: E402

CAPS = (1, 2, 4, 8, None)
CAP = 4                 # the engine's kMaxWeight
POINT_CHUNK = 128       # early-exit spacing over points (the parent)
ENTRY_CHUNK = 64        # early-exit spacing over entries


def entries(scan, cap):
    """Per point of one discrete scan (n, 2): its entry index; and the number of entries."""
    n = len(scan)
    head = np.ones(n, bool)
    head[1:] = (scan[1:] != scan[:-1]).any(1)
    run_start = np.maximum.accumulate(np.where(head, np.arange(n), 0))
    pos = np.arange(n) - run_start
    ent_head = head if cap is None else head | (pos % cap == 0)
    eid = np.cumsum(ent_head) - 1
    return eid, int(eid[-1]) + 1


def first_exit(csum, msum, P, valid, T, test_at, n_units):
    """Units read per parent: the first test index (in units) at which every valid child's
    bound c_t + P - m is below T, or n_units.  csum (4, m, B), msum (m, B) at the tests."""
    if len(test_at) == 0:
        return np.full(P.shape, n_units)
    ub = csum + (P[None, :, None] - msum[None])
    dead = np.where(valid[:, :, None], ub < T, True).all(0)
    return np.where(dead.any(1), test_at[np.argmax(dead, 1)], n_units)


def study(seed):
    grid, scans = bench.make_world(seed, 1)
    cloud = scans[0]
    og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
    om = oracle.FastCorrelativeScanMatcher2D(og, bench.LIN, bench.ANG, bench.DEPTH)
    want = om.match_full_submap(cloud, bench.MIN_SCORE)
    assert want["found"]
    fe = oracle.frontend2d(og, cloud, (0, 0, 0), full=True, lin=bench.LIN, ang=bench.ANG)
    ds = fe["discrete_scans"].astype(np.int64)     # (S, n, 2)
    bounds = fe["bounds"].astype(np.int64)
    S, n = ds.shape[0], ds.shape[1]
    share = {}
    for cap in CAPS:
        share[cap] = sum(entries(ds[k], cap)[1] for k in range(S)) / float(S * n)
    print("seed %d: scans %d, points %d; entries / points: %s" % (
        seed, S, n, ", ".join("cap %s %.1f %%" % (c or "none", 100 * share[c]) for c in CAPS)))

    depth = bench.DEPTH
    levels = [level_grid(grid.cells, h) for h in range(depth)]
    k, bx, by = want["best_scan_index"], want["best_x_offset"], want["best_y_offset"]
    s_star = int(values(levels[0][0], levels[0][1], ds[k], np.array([bx]), np.array([by])).sum())
    min_s, max_s = np.float32(1.0 - og.max_cost), np.float32(1.0 - og.min_cost)
    k255 = np.float32((max_s - min_s) / np.float32(255.0))
    all_sc = to_score(np.arange(255 * n + 1), n, min_s, k255)
    t_pess = int(np.argmax(all_sc > np.float32(bench.MIN_SCORE)))
    t_opt = max(t_pess, s_star)
    ent = [entries(ds[kk], CAP) for kk in range(S)]

    top = depth - 1
    fk, fx, fy = [], [], []
    for kk in range(S):
        mnx, mxx, mny, mxy = bounds[kk]
        X, Y = np.meshgrid(np.arange(mnx, mxx + 1, 1 << top), np.arange(mny, mxy + 1, 1 << top),
                           indexing="ij")
        xo, yo = X.ravel(), Y.ravel()
        keep = np.zeros(len(xo), bool)
        for a in range(0, len(xo), BATCH):
            keep[a:a + BATCH] = values(levels[top][0], levels[top][1], ds[kk], xo[a:a + BATCH],
                                       yo[a:a + BATCH]).sum(1) >= s_star
        fk.append(np.full(keep.sum(), kk))
        fx.append(xo[keep])
        fy.append(yo[keep])
    fk, fx, fy = np.concatenate(fk), np.concatenate(fx), np.concatenate(fy)

    rows = []
    for h in range(top, 0, -1):
        half = 1 << (h - 1)
        words = {(u, name): 0 for u in ("points", "entries") for name in ("all", "opt", "pess")}
        nk, nx, ny = [], [], []
        for kk in np.unique(fk):
            sel = fk == kk
            px, py = fx[sel], fy[sel]
            mnx, mxx, mny, mxy = bounds[kk]
            eid, m = ent[kk]
            last = np.flatnonzero(np.r_[eid[1:] != eid[:-1], True])   # last point of each entry
            p_tests = np.arange(POINT_CHUNK, n, POINT_CHUNK)
            e_tests = np.arange(ENTRY_CHUNK, m, ENTRY_CHUNK)
            for a in range(0, len(px), BATCH):
                bxo, byo = px[a:a + BATCH], py[a:a + BATCH]
                P = values(levels[h][0], levels[h][1], ds[kk], bxo, byo).sum(1)
                vc, valid = [], []
                for dx in (0, half):
                    for dy in (0, half):
                        vc.append(values(levels[h - 1][0], levels[h - 1][1], ds[kk], bxo + dx,
                                         byo + dy))
                        valid.append((bxo + dx <= mxx) & (byo + dy <= mxy))
                vc, valid = np.stack(vc), np.stack(valid)
                csum = np.cumsum(vc, axis=2)
                msum = np.cumsum(vc.max(0), axis=1)
                final = csum[:, :, -1]
                words[("points", "all")] += len(bxo) * n
                words[("entries", "all")] += len(bxo) * m
                for name, T in (("opt", t_opt), ("pess", t_pess)):
                    words[("points", name)] += int(first_exit(
                        csum[:, :, p_tests - 1], msum[:, p_tests - 1], P, valid, T, p_tests,
                        n).sum())
                    # sums after entry e are the points' sums at the entry's last point
                    at = last[e_tests - 1]
                    words[("entries", name)] += int(first_exit(
                        csum[:, :, at], msum[:, at], P, valid, T, e_tests, m).sum())
                for t, (dx, dy) in enumerate(((0, 0), (0, half), (half, 0), (half, half))):
                    keep = valid[t] & (final[t] >= s_star)
                    nk.append(np.full(keep.sum(), kk))
                    nx.append(bxo[keep] + dx)
                    ny.append(byo[keep] + dy)
        rows.append((h, len(fk), words))
        fk, fx, fy = np.concatenate(nk), np.concatenate(nx), np.concatenate(ny)
    return rows


def main():
    seeds = [int(a) for a in sys.argv[1:]] or [0, 1]
    for seed in seeds:
        t0 = time.time()
        rows = study(seed)
        print("branch-step words (cap %d): per point / per entry, and the entries' share" % CAP)
        print("  h  parents   %-28s %-28s %-28s" % ("no early exit", "early exit, opt",
                                                    "early exit, pess"))
        tot = {}
        for h, parents, w in rows:
            cells = ""
            for name in ("all", "opt", "pess"):
                a, b = w[("points", name)], w[("entries", name)]
                tot[name] = (tot.get(name, (0, 0))[0] + a, tot.get(name, (0, 0))[1] + b)
                cells += " %12d %12d %5.1f%%" % (a, b, 100.0 * b / max(1, a))
            print("  %d  %7d %s" % (h, parents, cells))
        cells = "".join(" %12d %12d %5.1f%%" % (a, b, 100.0 * b / max(1, a))
                        for a, b in (tot[name] for name in ("all", "opt", "pess")))
        print("  all %7s %s   [%.0f s]" % ("", cells, time.time() - t0))


if __name__ == "__main__":
    main()
