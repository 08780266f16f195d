"""The C++ adapter's RangeDataInserter3D (adapter_selftest.cc, `insert3d` RESULT lines) against
the CPU restatement: the reference's InsertPointCloudWithIntensities, inserted twice into empty
1 m device grids, bit for bit."""
import os
import subprocess

import numpy as np
import pytest

from tests import insert3d_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


@pytest.mark.gpu
def test_adapter_insert3d_matches_oracle():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT insert3d")}
    ins = O.RangeDataInserter3D(0.7, 0.4, 1000, 100.0)
    g, ig = O.HybridGrid(1.0), O.IntensityHybridGrid(1.0)
    returns = np.float32([[-3, -1, 4], [-2, 0, 4], [-1, 1, 4], [0, 2, 4]])
    for _ in range(2):
        ins.insert([0, 0, -4], returns, np.float32([7, 8, 9, 10]), g, ig)
    got = [int(v) for v in res["insert3d"]]
    lo, dims = got[:3], got[3:6]
    np.testing.assert_array_equal(np.array(got[6:], np.uint16), g.dense(lo, dims).reshape(-1))
    assert int((g.values != 0).sum()) == int((np.array(got[6:]) != 0).sum())
    got = res["insert3d_intensity"]
    lo, dims = [int(v) for v in got[:3]], [int(v) for v in got[3:6]]
    cells = [v.split(":") for v in got[6:]]
    mean = np.array([int(c[0], 16) for c in cells], np.uint32)
    sums = np.array([int(c[1], 16) for c in cells], np.uint32)
    counts = np.array([int(c[2]) for c in cells], np.int32)
    np.testing.assert_array_equal(counts, ig.dense(lo, dims, 1).reshape(-1))
    np.testing.assert_array_equal(sums, ig.dense(lo, dims, 0).view(np.uint32).reshape(-1))
    np.testing.assert_array_equal(mean, ig.dense_mean(lo, dims).view(np.uint32).reshape(-1))
    assert counts.sum() == 8
