#!/usr/bin/env python
"""CPU study (no product code): how many (parent, point) child-window words the branch
step (k_expand_lattice) would still gather if a parent stopped summing its children once
its remaining bound rules all of them out.

For parent level h and scan point p, one 32-bit word holds the four children values of
level h-1.  Every child window lies inside the parent's window, so max4(word) <= the
parent's level-h value at p (asserted below on every sampled point).  After the first b
points, with c_t child t's partial sum, m the partial sum of max4(word) and P the parent's
sum, child t ends at most at c_t + (P - m).  When that is below the integer survival
threshold T for every valid child, the parent's remaining words need not be read.

The expanded parents are those of the tree with the optimum S* known (every node whose
parent's bound is >= S*), as in theta_hierarchy_counts.py.  T is taken twice:
  optimistic  : T from S* (the engine's bound after the dives is <= S*);
  pessimistic : T from min_score alone.
The early exit is tested at chunk boundaries of 64, 128 and 256 points, in the points'
stored (beam) order.  "today" counts n words per expanded parent.

  python benchmarks/prototypes/early_exit_counts.py [seed ...]     (default: seeds 0 1)
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench                      # noqa: E402  (workload generator)
from oracle import pyoracle as oracle  # noqa: E402

CHUNKS = (64, 128, 256)
BATCH = 1024


def level_grid(cells, h):
    """PrecomputationGrid2D of width 2^h as int array with its offset (wide grid)."""
    w = 1 << h
    pg = oracle.precompute_grid2d(cells, oracle.constant(2), oracle.constant(3), w)
    return pg.astype(np.int32), w - 1   # value(x, y) = pg[y + off, x + off], 0 outside


def values(pg, off, pts, xo, yo):
    """(m, n) per-point GetValue(p + (xo, yo)); pts: (n, 2) cells; xo, yo: (m,) offsets."""
    wy, wx = pg.shape
    x = pts[None, :, 0] + xo[:, None] + off
    y = pts[None, :, 1] + yo[:, None] + off
    ok = (x >= 0) & (x < wx) & (y >= 0) & (y < wy)
    return pg[np.clip(y, 0, wy - 1), np.clip(x, 0, wx - 1)] * ok


def to_score(sums, n, min_s, k255):
    """PrecomputationGrid2D::ToScore(sum / float(n)) in float32 round-to-nearest."""
    mean = sums.astype(np.float32) / np.float32(n)
    return np.float32(min_s) + mean * np.float32(k255)


def study(seed):
    grid, scans = bench.make_world(seed, 1)
    cloud = scans[0]
    og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
    om = oracle.FastCorrelativeScanMatcher2D(og, bench.LIN, bench.ANG, bench.DEPTH)
    want = om.match_full_submap(cloud, bench.MIN_SCORE)
    assert want["found"]
    fe = oracle.frontend2d(og, cloud, (0, 0, 0), full=True, lin=bench.LIN, ang=bench.ANG)
    ds = fe["discrete_scans"].astype(np.int64)     # (S, n, 2)
    bounds = fe["bounds"].astype(np.int64)         # (S, 4) min_x max_x min_y max_y
    S, n = ds.shape[0], ds.shape[1]
    depth = bench.DEPTH
    levels = [level_grid(grid.cells, h) for h in range(depth)]
    k, bx, by = want["best_scan_index"], want["best_x_offset"], want["best_y_offset"]
    s_star = int(values(levels[0][0], levels[0][1], ds[k], np.array([bx]), np.array([by])).sum())
    # integer thresholds: smallest sum whose score passes "> min_score" (and ">= S*")
    min_s, max_s = np.float32(1.0 - og.max_cost), np.float32(1.0 - og.min_cost)
    k255 = np.float32((max_s - min_s) / np.float32(255.0))
    all_sc = to_score(np.arange(255 * n + 1), n, min_s, k255)
    t_pess = int(np.argmax(all_sc > np.float32(bench.MIN_SCORE)))
    t_opt = max(t_pess, s_star)
    print("seed %d: scans %d, points %d, S* sum %d (score %.4f), T optimistic %d, "
          "T pessimistic %d" % (seed, S, n, s_star, want["score"], t_opt, t_pess))

    top = depth - 1
    fr = []
    for kk in range(S):
        mnx, mxx, mny, mxy = bounds[kk]
        X, Y = np.meshgrid(np.arange(mnx, mxx + 1, 1 << top), np.arange(mny, mxy + 1, 1 << top),
                           indexing="ij")
        xo, yo = X.ravel(), Y.ravel()
        keep = np.zeros(len(xo), bool)
        for a in range(0, len(xo), BATCH):
            keep[a:a + BATCH] = values(levels[top][0], levels[top][1], ds[kk], xo[a:a + BATCH],
                                       yo[a:a + BATCH]).sum(1) >= s_star
        fr.append((np.full(keep.sum(), kk), xo[keep], yo[keep]))
    fk = np.concatenate([f[0] for f in fr])
    fx = np.concatenate([f[1] for f in fr])
    fy = np.concatenate([f[2] for f in fr])

    rows = []
    for h in range(top, 0, -1):
        half = 1 << (h - 1)
        today = 0
        kept = {(name, c): 0 for name in ("opt", "pess") for c in CHUNKS}
        nk, nx, ny = [], [], []
        for kk in np.unique(fk):
            sel = fk == kk
            px, py = fx[sel], fy[sel]
            mnx, mxx, mny, mxy = bounds[kk]
            for a in range(0, len(px), BATCH):
                bxo, byo = px[a:a + BATCH], py[a:a + BATCH]
                vp = values(levels[h][0], levels[h][1], ds[kk], bxo, byo)
                P = vp.sum(1)
                vc, valid = [], []
                for dx in (0, half):        # slot t = 2*ix + iy, as in the kernel
                    for dy in (0, half):
                        vc.append(values(levels[h - 1][0], levels[h - 1][1], ds[kk], bxo + dx,
                                         byo + dy))
                        valid.append((bxo + dx <= mxx) & (byo + dy <= mxy))
                vc = np.stack(vc)                     # (4, m, n)
                valid = np.stack(valid)               # (4, m)
                mx = vc.max(0)
                assert (mx <= vp).all(), "a child value exceeds its parent's at some point"
                today += len(bxo) * n
                csum = np.cumsum(vc, axis=2)          # (4, m, n)
                msum = np.cumsum(mx, axis=1)          # (m, n)
                final = csum[:, :, -1]
                for name, T in (("opt", t_opt), ("pess", t_pess)):
                    for c in CHUNKS:
                        ends = np.arange(c, n, c)     # boundaries strictly inside the scan
                        if len(ends) == 0:
                            kept[(name, c)] += len(bxo) * n
                            continue
                        ub = csum[:, :, ends - 1] + (P[None, :, None] - msum[None, :, ends - 1])
                        dead = np.where(valid[:, :, None], ub < T, True).all(0)   # (m, B)
                        first = np.where(dead.any(1), ends[np.argmax(dead, 1)], n)
                        # a parent ruled out early has no child that would have survived
                        gone = first < n
                        assert not (valid[:, gone] & (final[:, gone] >= T)).any()
                        kept[(name, c)] += int(first.sum())
                # next frontier: children with sum >= S* (the tree with S* known)
                for t, (dx, dy) in enumerate(((0, 0), (0, half), (half, 0), (half, half))):
                    keep = valid[t] & (final[t] >= s_star)
                    nk.append(np.full(keep.sum(), kk))
                    nx.append(bxo[keep] + dx)
                    ny.append(byo[keep] + dy)
        rows.append((h, int(len(fk)), today, kept))
        fk, fx, fy = np.concatenate(nk), np.concatenate(nx), np.concatenate(ny)
    return rows


def main():
    seeds = [int(a) for a in sys.argv[1:]] or [0, 1]
    hdr = "  h  parents      words today" + "".join(
        "  %s/%-3d" % (name, c) for name in ("opt", "pess") for c in CHUNKS)
    for seed in seeds:
        t0 = time.time()
        rows = study(seed)
        print("words saved by the early exit, per parent level h (share of today's words):")
        print(hdr)
        tot_today = 0
        tot = {key: 0 for key in rows[0][3]}
        for h, parents, today, kept in rows:
            tot_today += today
            cells = ""
            for name in ("opt", "pess"):
                for c in CHUNKS:
                    tot[(name, c)] += kept[(name, c)]
                    cells += "  %7.1f%%" % (100.0 * (1 - kept[(name, c)] / today))
            print("  %d  %7d  %15d%s" % (h, parents, today, cells))
        cells = "".join("  %7.1f%%" % (100.0 * (1 - tot[(name, c)] / tot_today))
                        for name in ("opt", "pess") for c in CHUNKS)
        print("  all %7s  %15d%s   [%.0f s]" % ("", tot_today, cells, time.time() - t0))


if __name__ == "__main__":
    main()
