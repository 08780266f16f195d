"""The C++ adapter's TSDFRangeDataInserter2D over a DeviceGrid2D(limits, truncation, max_weight)
(adapter_selftest.cc, `insert_tsdf2d` RESULT line) against the CPU restatement."""
import os
import subprocess

import numpy as np
import pytest

from tests import insert_tsdf2d_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


class _Opts:
    def __init__(self, **kw):
        self.truncation_distance = 2.0
        self.maximum_weight = 10.0
        self.update_free_space = False
        self.num_normal_samples = 2
        self.sample_radius = 10.0
        self.project_sdf_distance_to_scan_normal = False
        self.update_weight_range_exponent = 0
        self.update_weight_angle_scan_normal_to_ray_kernel_bandwidth = 0.0
        self.update_weight_distance_cell_to_hit_kernel_bandwidth = 0.0
        self.__dict__.update(kw)


@pytest.mark.gpu
def test_adapter_insert_tsdf2d_matches_oracle():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    line = [ln.split()[2:] for ln in out.stdout.splitlines()
            if ln.startswith("RESULT insert_tsdf2d ")]
    assert len(line) == 1
    fields = line[0]
    g = O.TsdfGrid(1.0, 1.0, 7.0, 8, 1, 2.0, 10.0)
    origin = np.float32([-0.5, -0.5, 0])
    assert O.TsdfInserter(_Opts()).insert(origin, np.float32([[-0.5, 3.5, 0]]), g)
    weighted = _Opts(project_sdf_distance_to_scan_normal=True,
                     update_weight_angle_scan_normal_to_ray_kernel_bandwidth=0.5,
                     update_weight_distance_cell_to_hit_kernel_bandwidth=0.5)
    assert O.TsdfInserter(weighted).insert(origin, np.float32([[-0.5, 3.5, 0], [5.5, 3.5, 0]]), g)
    res, max_x, max_y = (float(v) for v in fields[:3])
    nx, ny, empty, x0, y0, x1, y1 = (int(v) for v in fields[3:10])
    assert (res, max_x, max_y, nx, ny) == g.limits
    assert (None if empty else (x0, y0, x1, y1)) == g.known_box
    cells = np.array([int(v) for v in fields[10:]], np.uint16)
    tsd, weight = g.arrays()
    np.testing.assert_array_equal(cells[:nx * ny].reshape(ny, nx), tsd)
    np.testing.assert_array_equal(cells[nx * ny:].reshape(ny, nx), weight)
    assert nx > 8   # the first insert grew the grid
