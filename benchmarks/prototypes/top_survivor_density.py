#!/usr/bin/env python
"""CPU study (no product code): how the surviving parents at the top level (h = 6 at depth
7) are spread over the rotated scans, and how many 128-byte lines of the child-window table
(StackDev::win[6]) the branch step would touch per scan in two forms:

  sparse : today's k_expand_lattice.  Items of up to 32 parents of one scan in row-major
           lattice order; per point one load of the running parents' words.  Lines are the
           distinct 128-byte lines of one such load, summed over the points each parent
           reads before the early exit (tests every 128 points, as in early_exit_counts.py).
  dense  : a tile form that walks the scan's run-merged entries (cap 4, as k_discretize
           writes them) and, per entry, reads the whole valid lattice of the scan shifted
           by the entry's cell: the words of the window table inside [0, ids) x [0, jd).

Survivors at the top are lattice cells whose sum passes min_score and is >= the bound.
The bound is taken twice: from the optimum S* ("opt"), and from min_score alone ("pess");
the engine's bound after the dives lies between the two.  Words are (parent, point) pairs,
one 32-bit table word each, counted before the early exit.

  python benchmarks/prototypes/top_survivor_density.py [seed ...]     (default: seeds 0 1)
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench                      # noqa: E402  (workload generator only)
from early_exit_counts import BATCH, level_grid, to_score, values  # noqa: E402
from point_run_counts import entries, first_exit  # noqa: E402
from oracle import pyoracle as oracle  # noqa: E402

TAUS = (0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8)
HIST = np.linspace(0.0, 1.0, 11)
CAP = 4                 # the engine's kMaxWeight
CHUNK = 128             # early-exit spacing over points (kLatChunk)
ITEM = 32               # parents per work item of the sparse form
LINE_WORDS = 32         # 128-byte lines of 32-bit words


def window_addr(pts, min_x, min_y, h, jd, ids):
    """Per point: the window word of lattice cell (0, 0), and its (qx, qy) in the phase,
    as k_expand_lattice stages them (the word of cell (i, j) is addr + j * ids + i)."""
    s = 1 << (h - 1)
    bx = pts[:, 0] + min_x + s - 1
    by = pts[:, 1] + min_y + s - 1
    qx, qy = (bx >> h) + 1, (by >> h) + 1
    phase = ((by & ((1 << h) - 1)) << h) | (bx & ((1 << h) - 1))
    return (phase * jd + qy) * ids + qx, qx, qy


def distinct_per_column(lines):
    """Distinct non-negative values per column of an (r, n) array (-1 = no load)."""
    srt = np.sort(lines, axis=0)
    new = np.ones_like(srt, bool)
    new[1:] = srt[1:] != srt[:-1]
    return ((srt >= 0) & new).sum(0)


def sparse_lines(addr, qx, qy, pi, pj, run_pts, jd, ids):
    """Lines of the sparse form for parents (pi, pj) in row-major lattice order, each
    reading its first run_pts[k] points."""
    n = len(addr)
    total = 0
    for a in range(0, len(pi), ITEM):
        i, j, r = pi[a:a + ITEM, None], pj[a:a + ITEM, None], run_pts[a:a + ITEM, None]
        ok = ((qx[None] + i >= 0) & (qx[None] + i < ids) & (qy[None] + j >= 0) &
              (qy[None] + j < jd) & (np.arange(n)[None] < r))
        words = addr[None] + j * ids + i
        total += int(distinct_per_column(np.where(ok, words // LINE_WORDS, -1)).sum())
    return total


def dense_lines(addr, qx, qy, ent_pts, nxc, nyc, jd, ids):
    """Lines of the dense form: per entry, the valid lattice window shifted by its cell."""
    a, x, y = addr[ent_pts], qx[ent_pts], qy[ent_pts]
    c0, c1 = np.maximum(x, 0), np.minimum(x + nxc, ids) - 1          # table columns
    j = np.arange(nyc)[None]
    r = y[:, None] + j                                              # table rows
    ok = (r >= 0) & (r < jd) & (c1 >= c0)[:, None]
    lo = (a[:, None] + j * ids + (c0 - x)[:, None]) // LINE_WORDS
    hi = (a[:, None] + j * ids + (c1 - x)[:, None]) // LINE_WORDS
    per_row = np.where(ok, hi - lo + 1, 0).sum()
    # rows ascend in memory and never overlap, so neighbouring valid rows share at most
    # one line: the last line of a row and the first of the next
    shared = (ok[:, 1:] & ok[:, :-1] & (lo[:, 1:] == hi[:, :-1])).sum()
    return int(per_row - shared)


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
    h = depth - 1
    levels = [level_grid(grid.cells, l) for l in range(depth)]
    k, bx, by = want["best_scan_index"], want["best_x_offset"], want["best_y_offset"]
    s_star = int(values(levels[0][0], levels[0][1], ds[k], np.array([bx]), np.array([by])).sum())
    min_s, max_s = np.float32(1.0 - og.max_cost), np.float32(1.0 - og.min_cost)
    k255 = np.float32((max_s - min_s) / np.float32(255.0))
    all_sc = to_score(np.arange(255 * n + 1), n, min_s, k255)
    t_pess = int(np.argmax(all_sc > np.float32(bench.MIN_SCORE)))
    t_opt = max(t_pess, s_star)
    # the window table of parent level h: one phase is jd x ids words (k_stack_window)
    wy, wx = levels[h - 1][0].shape
    ids = (wx + (1 << h) - 1) // (1 << h) + 1
    jd = (wy + (1 << h) - 1) // (1 << h) + 1
    print("seed %d: scans %d, points %d, S* sum %d, T opt %d, T pess %d; win[%d] phase %d x %d "
          "words" % (seed, S, n, s_star, t_opt, t_pess, h, jd, ids))

    rows = {name: [] for name in ("opt", "pess")}   # per scan: density, parents, words, lines
    half = 1 << (h - 1)
    for kk in range(S):
        mnx, mxx, mny, mxy = bounds[kk]
        nxc, nyc = ((mxx - mnx) >> h) + 1, ((mxy - mny) >> h) + 1
        J, I = np.meshgrid(np.arange(nyc), np.arange(nxc), indexing="ij")
        pi, pj = I.ravel(), J.ravel()                # row-major lattice order (k_filter_top)
        xo, yo = mnx + (pi << h), mny + (pj << h)
        top = np.concatenate([values(levels[h][0], levels[h][1], ds[kk], xo[a:a + BATCH],
                                     yo[a:a + BATCH]).sum(1) for a in range(0, len(xo), BATCH)])
        addr, qx, qy = window_addr(ds[kk], mnx, mny, h, jd, ids)
        eid, m = entries(ds[kk], CAP)
        ent_pts = np.flatnonzero(np.r_[True, eid[1:] != eid[:-1]])  # first point of each entry
        dense = dense_lines(addr, qx, qy, ent_pts, nxc, nyc, jd, ids)
        for name, T in (("opt", t_opt), ("pess", t_pess)):
            keep = top >= T
            P = int(keep.sum())
            if P == 0:
                rows[name].append((0.0, 0, 0, 0, dense))
                continue
            kx, ky = xo[keep], yo[keep]
            vc, valid = [], []
            for dx in (0, half):
                for dy in (0, half):
                    vc.append(values(levels[h - 1][0], levels[h - 1][1], ds[kk], kx + dx, ky + dy))
                    valid.append((kx + dx <= mxx) & (ky + dy <= mxy))
            vc, valid = np.stack(vc), np.stack(valid)
            tests = np.arange(CHUNK, n, CHUNK)
            run_pts = first_exit(np.cumsum(vc, axis=2)[:, :, tests - 1],
                                 np.cumsum(vc.max(0), axis=1)[:, tests - 1], top[keep], valid,
                                 T, tests, n)
            sparse = sparse_lines(addr, qx, qy, pi[keep], pj[keep], run_pts, jd, ids)
            rows[name].append((P / float(nxc * nyc), P, P * n, sparse, dense))
    return {name: np.array(r, dtype=np.float64) for name, r in rows.items()}


def report(seed, res):
    for name, r in res.items():
        dens, parents, words, sparse, dense = r.T
        live = parents > 0
        print("  bound %s: %d parents in %d of %d scans; sparse lines %d, dense lines (every "
              "scan) %d" % (name, parents.sum(), live.sum(), len(r), sparse.sum(), dense.sum()))
        hist, _ = np.histogram(dens[live], HIST)
        print("    scans by survivor density: " + "  ".join(
            "%.1f-%.1f: %d" % (HIST[i], HIST[i + 1], hist[i]) for i in range(len(hist))))
        print("    tau  scans  parents  words   dense<sparse words  lines sparse -> mixed")
        for tau in TAUS:
            sel = live & (dens >= tau)
            win = sel & (dense < sparse)
            mixed = sparse.sum() - sparse[sel].sum() + dense[sel].sum()
            print("    %.1f  %5d  %6.1f%%  %6.1f%%  %6.1f%%             %d -> %d (%+.1f%%)" % (
                tau, sel.sum(), 100 * parents[sel].sum() / parents.sum(),
                100 * words[sel].sum() / words.sum(), 100 * words[win].sum() / words.sum(),
                sparse.sum(), mixed, 100 * (mixed / sparse.sum() - 1)))


def main():
    seeds = [int(a) for a in sys.argv[1:]] or [0, 1]
    for seed in seeds:
        t0 = time.time()
        res = study(seed)
        report(seed, res)
        print("  [%.0f s]" % (time.time() - t0))


if __name__ == "__main__":
    main()
