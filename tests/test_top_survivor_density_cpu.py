"""The line-counting helpers of benchmarks/prototypes/top_survivor_density.py against
brute-force sets of 128-byte lines, on random window tables and scans."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                "benchmarks", "prototypes"))
tsd = pytest.importorskip("top_survivor_density")


def _case(seed):
    rng = np.random.RandomState(seed)
    h = int(rng.randint(2, 5))
    jd, ids = int(rng.randint(3, 20)), int(rng.randint(3, 40))
    n = int(rng.randint(1, 300))
    pts = rng.randint(-(jd << h), (ids + 2) << h, size=(n, 2)).astype(np.int64)
    min_x, min_y = int(rng.randint(-40, 40)), int(rng.randint(-40, 40))
    addr, qx, qy = tsd.window_addr(pts, min_x, min_y, h, jd, ids)
    return rng, h, jd, ids, n, addr, qx, qy


def _word_ok(qx, qy, i, j, jd, ids):
    return 0 <= qx + i < ids and 0 <= qy + j < jd


@pytest.mark.parametrize("seed", range(12))
def test_dense_lines(seed):
    rng, h, jd, ids, n, addr, qx, qy = _case(seed)
    nxc, nyc = int(rng.randint(1, ids + 6)), int(rng.randint(1, jd + 6))
    ent = np.sort(rng.choice(n, int(rng.randint(1, n + 1)), replace=False))
    want = 0
    for p in ent:
        lines = {(addr[p] + j * ids + i) // tsd.LINE_WORDS for j in range(nyc) for i in range(nxc)
                 if _word_ok(qx[p], qy[p], i, j, jd, ids)}
        want += len(lines)
    assert tsd.dense_lines(addr, qx, qy, ent, nxc, nyc, jd, ids) == want


@pytest.mark.parametrize("seed", range(12))
def test_sparse_lines(seed):
    rng, h, jd, ids, n, addr, qx, qy = _case(100 + seed)
    nxc, nyc = int(rng.randint(1, ids + 6)), int(rng.randint(1, jd + 6))
    cells = [(i, j) for j in range(nyc) for i in range(nxc)]
    pick = np.sort(rng.choice(len(cells), int(rng.randint(1, min(len(cells), 80) + 1)),
                              replace=False))
    pi = np.array([cells[c][0] for c in pick])
    pj = np.array([cells[c][1] for c in pick])
    run_pts = rng.randint(0, n + 1, size=len(pi))
    want = 0
    for a in range(0, len(pi), tsd.ITEM):
        for p in range(n):
            lines = {(addr[p] + pj[k] * ids + pi[k]) // tsd.LINE_WORDS
                     for k in range(a, min(a + tsd.ITEM, len(pi)))
                     if p < run_pts[k] and _word_ok(qx[p], qy[p], pi[k], pj[k], jd, ids)}
            want += len(lines)
    assert tsd.sparse_lines(addr, qx, qy, pi, pj, run_pts, jd, ids) == want
