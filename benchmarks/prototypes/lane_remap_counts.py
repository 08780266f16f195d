#!/usr/bin/env python
"""CPU study (no product code): warp trips of the branch step (k_expand_lattice) with the
early exit, when a warp keeps its sub-lane count G fixed for the whole item ("today") and
when it re-chooses G from the parents still running at every early-exit test ("re-map").

The tree and the per-parent early exit are those of early_exit_counts.py, with the
survival threshold T from the optimum S* (the engine's bound after the dives).  A work
item is <= 32 parents of one scan, taken in lattice order (y, then x).  G starts as the
largest power of two with count * G <= 32.  A trip is one warp pass over one 128-point
chunk divided by G (a 64-point segment is half a trip).  Today a warp passes over a chunk
while any parent of its item runs.  With the re-map, after a test that leaves L parents
running, G becomes the largest power of two with L * G <= 32 whenever that is larger
(G can only grow: L only falls).  Words read are the same under both rules.

  python benchmarks/prototypes/lane_remap_counts.py [seed ...]     (default: seeds 0 1)
"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import early_exit_counts as eec   # noqa: E402  (workload, tree and bound helpers)

bench, oracle = eec.bench, eec.oracle
SPACINGS = (128, 64)
BATCH = eec.BATCH


def first_point(csum, msum, P, valid, T, n, c):
    """Points a parent reads with tests every c points: the first test boundary where all
    valid children's upper bounds are below T, else n."""
    ends = np.arange(c, n, c)
    ub = csum[:, :, ends - 1] + (P[None, :, None] - msum[None, :, ends - 1])
    dead = np.where(valid[:, :, None], ub < T, True).all(0)
    return np.where(dead.any(1), ends[np.argmax(dead, 1)], n)


def item_trips(first, n, c):
    """(no exit, today, re-map, re-maps, tests) trips of one item whose parents read
    `first` points each."""
    cnt = len(first)
    lg = 0
    while (cnt << (lg + 1)) <= 32:
        lg += 1
    g0 = 1 << lg
    seg = c / 128.0
    nseg = -(-n // c)
    no_exit = nseg * seg / g0
    last = -(-int(first.max()) // c)         # segments the warp passes over
    today = last * seg / g0
    remap, remaps, g = 0.0, 0, g0
    for k in range(last):
        if k:
            live = int((first > k * c).sum())
            gl = g
            while live * 2 * gl <= 32:
                gl *= 2
            if gl > g:
                g, remaps = gl, remaps + 1
        remap += seg / g
    return no_exit, today, remap, remaps, max(last - 1, 0)


def study(seed):
    grid, scans = bench.make_world(seed, 1)
    cloud = scans[0]
    og = oracle.Grid2D(grid.cells, grid.resolution, grid.max_x, grid.max_y)
    om = oracle.FastCorrelativeScanMatcher2D(og, bench.LIN, bench.ANG, bench.DEPTH)
    want = om.match_full_submap(cloud, bench.MIN_SCORE)
    assert want["found"]
    fe = oracle.frontend2d(og, cloud, (0, 0, 0), full=True, lin=bench.LIN, ang=bench.ANG)
    ds = fe["discrete_scans"].astype(np.int64)
    bounds = fe["bounds"].astype(np.int64)
    S, n = ds.shape[0], ds.shape[1]
    depth = bench.DEPTH
    levels = [eec.level_grid(grid.cells, h) for h in range(depth)]
    k, bx, by = want["best_scan_index"], want["best_x_offset"], want["best_y_offset"]
    s_star = int(eec.values(levels[0][0], levels[0][1], ds[k], np.array([bx]),
                            np.array([by])).sum())
    min_s, max_s = np.float32(1.0 - og.max_cost), np.float32(1.0 - og.min_cost)
    k255 = np.float32((max_s - min_s) / np.float32(255.0))
    all_sc = eec.to_score(np.arange(255 * n + 1), n, min_s, k255)
    T = max(int(np.argmax(all_sc > np.float32(bench.MIN_SCORE))), s_star)
    print("seed %d: scans %d, points %d, S* sum %d, T %d" % (seed, S, n, s_star, T))

    top = depth - 1
    fr = []
    for kk in range(S):
        mnx, mxx, mny, mxy = bounds[kk]
        X, Y = np.meshgrid(np.arange(mnx, mxx + 1, 1 << top), np.arange(mny, mxy + 1, 1 << top),
                           indexing="ij")
        xo, yo = X.ravel(), Y.ravel()
        keep = np.zeros(len(xo), bool)
        for a in range(0, len(xo), BATCH):
            keep[a:a + BATCH] = eec.values(levels[top][0], levels[top][1], ds[kk], xo[a:a + BATCH],
                                           yo[a:a + BATCH]).sum(1) >= s_star
        fr.append((np.full(keep.sum(), kk), xo[keep], yo[keep]))
    fk = np.concatenate([f[0] for f in fr])
    fx = np.concatenate([f[1] for f in fr])
    fy = np.concatenate([f[2] for f in fr])

    rows = []
    for h in range(top, 0, -1):
        half = 1 << (h - 1)
        tot = {c: np.zeros(5) for c in SPACINGS}
        nk, nx, ny = [], [], []
        for kk in np.unique(fk):
            sel = fk == kk
            order = np.lexsort((fx[sel], fy[sel]))      # lattice order: y, then x
            px, py = fx[sel][order], fy[sel][order]
            mnx, mxx, mny, mxy = bounds[kk]
            first = {c: [] for c in SPACINGS}
            for a in range(0, len(px), BATCH):
                bxo, byo = px[a:a + BATCH], py[a:a + BATCH]
                P = eec.values(levels[h][0], levels[h][1], ds[kk], bxo, byo).sum(1)
                vc, valid = [], []
                for dx in (0, half):
                    for dy in (0, half):
                        vc.append(eec.values(levels[h - 1][0], levels[h - 1][1], ds[kk],
                                             bxo + dx, byo + dy))
                        valid.append((bxo + dx <= mxx) & (byo + dy <= mxy))
                vc, valid = np.stack(vc), np.stack(valid)
                csum = np.cumsum(vc, axis=2)
                msum = np.cumsum(vc.max(0), axis=1)
                for c in SPACINGS:
                    first[c].append(first_point(csum, msum, P, valid, T, n, c))
                final = csum[:, :, -1]
                for t, (dx, dy) in enumerate(((0, 0), (0, half), (half, 0), (half, half))):
                    keep = valid[t] & (final[t] >= s_star)
                    nk.append(np.full(keep.sum(), kk))
                    nx.append(bxo[keep] + dx)
                    ny.append(byo[keep] + dy)
            for c in SPACINGS:
                fc = np.concatenate(first[c])
                for a in range(0, len(fc), 32):
                    tot[c] += item_trips(fc[a:a + 32], n, c)
        rows.append((h, int(len(fk)), tot))
        fk, fx, fy = np.concatenate(nk), np.concatenate(nx), np.concatenate(ny)
    return rows


def main():
    seeds = [int(a) for a in sys.argv[1:]] or [0, 1]
    for seed in seeds:
        t0 = time.time()
        rows = study(seed)
        for c in SPACINGS:
            print("tests every %d points: trips per parent level h" % c)
            print("  h  parents   no exit     today    re-map  (vs today)  re-maps     tests")
            tot = np.zeros(5)
            for h, parents, t in rows:
                tc = t[c]
                tot += tc
                print("  %d  %7d  %8.0f  %8.0f  %8.0f  (%+5.1f %%)  %7d  %8d" % (
                    h, parents, tc[0], tc[1], tc[2], 100.0 * (tc[2] / tc[1] - 1), tc[3], tc[4]))
            print("  all %7s %8.0f  %8.0f  %8.0f  (%+5.1f %%)  %7d  %8d" % (
                "", tot[0], tot[1], tot[2], 100.0 * (tot[2] / tot[1] - 1), tot[3], tot[4]))
        print("[%.0f s]" % (time.time() - t0))


if __name__ == "__main__":
    main()
