"""The C++ adapter's DeviceHybridGrid::ToProto and DeviceGrid2D::ToProto (adapter_selftest.cc,
`grid_to_proto_*` RESULT lines) against the test-side reference encoders applied to the same
grids, which the self-test prints beside them: byte for byte."""
import os
import subprocess

import numpy as np
import pytest

from tests import grid_proto_ref as R

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


def _grid2d(fields, tsdf=None):
    res, max_x, max_y = (float(v) for v in fields[:3])
    nx, ny, empty, mn_x, mn_y, mx_x, mx_y = (int(v) for v in fields[3:10])
    values = np.array([int(v) for v in fields[10:]], np.uint16)
    cells = values[:nx * ny].reshape(ny, nx)
    box = None if empty else (mn_x, mn_y, mx_x, mx_y)
    if tsdf is None:
        return R.grid2d_message(cells, res, max_x, max_y, box)
    return R.grid2d_message(cells, res, max_x, max_y, box, values[nx * ny:].reshape(ny, nx), *tsdf)


@pytest.mark.gpu
def test_adapter_grid_to_proto_matches_reference_encoders():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT ")}
    got = {k[len("grid_to_proto_"):]: bytes.fromhex(v[0]) for k, v in res.items()
           if k.startswith("grid_to_proto_")}
    assert sorted(got) == ["crop2d", "insert2d", "insert3d", "insert_tsdf2d"]
    # 3D: the dense box of the 1 m grid, its non-zero voxels in the walk's order
    box = [int(v) for v in res["insert3d"]]
    lo, dims = np.array(box[:3]), box[3:6]
    vol = np.array(box[6:], np.uint16).reshape(dims[::-1])
    z, y, x = np.nonzero(vol)
    idx, val, _ = R.walk((np.stack([x, y, z], 1) + lo, vol[z, y, x]))
    assert len(val) > 0
    assert got["insert3d"] == R.hybrid_grid_message(1.0, idx, val)
    # 2D: the ProbabilityGrid, its crop, and the TSDF2D (truncation 2, max weight 10)
    assert got["insert2d"] == _grid2d(res["insert2d"])
    assert got["crop2d"] == _grid2d(res["crop2d"])
    assert got["insert_tsdf2d"] == _grid2d(res["insert_tsdf2d"], (2.0, 10.0))
