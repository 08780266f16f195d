"""The C++ adapter's ProbabilityGridRangeDataInserter2D, DeviceGrid2D::ComputeCroppedGrid and
FastCorrelativeScanMatcher2D(DeviceGrid2D) (adapter_selftest.cc, `insert2d` / `crop2d` /
`stack2d` RESULT lines) against the CPU restatement and the host-built stack."""
import os
import subprocess

import numpy as np
import pytest

from tests import insert2d_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


def _grid_line(fields):
    res, max_x, max_y = (float(v) for v in fields[:3])
    nx, ny, empty, x0, y0, x1, y1 = (int(v) for v in fields[3:10])
    cells = np.array([int(v) for v in fields[10:]], np.uint16).reshape(ny, nx)
    return (res, max_x, max_y, nx, ny), None if empty else (x0, y0, x1, y1), cells


@pytest.mark.gpu
def test_adapter_insert2d_matches_oracle():
    from benchmarks import synthetic
    from cartographer_b200 import scan_matching as sm
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT ") and ln.split()[1] in ("insert2d", "crop2d", "stack2d")}
    ins = O.Inserter(0.7, 0.4, True)
    g = O.Grid(1.0, 1.0, 5.0, 5, 5)
    ins.insert([-0.5, 0.5, 0], np.float32([[-3.5, 0.5, 0], [-2.5, 1.5, 0], [-1.5, 2.5, 0],
                                           [-0.5, 3.5, 0]]), g, np.float32([[0.5, 4.5, 0]]))
    ins.insert([-0.5, 0.5, 0], np.float32([[-6.5, 0.5, 0]]), g)
    crop = g.crop()
    for name, ora in (("insert2d", g), ("crop2d", crop)):
        limits, box, cells = _grid_line(res[name])
        assert limits == ora.limits and box == ora.known_box, name
        np.testing.assert_array_equal(cells, ora.cells)
    assert g.limits[3] == 10   # the second insert grew the grid
    r, max_x, max_y, nx, ny = crop.limits
    m = sm.FastCorrelativeScanMatcher2D(synthetic.GridSpec(crop.cells, r, max_x, max_y),
                                        sm.FastCorrelativeScanMatcherOptions2D(3.0, 0.5, 2))
    want = m.precomputation_grid(1)
    got = [int(v) for v in res["stack2d"]]
    assert got[:2] == [want.shape[1], want.shape[0]]
    np.testing.assert_array_equal(np.array(got[2:], np.uint8).reshape(want.shape), want)
    m.close()
