"""The C++ adapter's CeresScanMatcher3D with an intensity grid (DeviceIntensityGrid,
PointCloudAndDeviceGrid::intensity_hybrid_grid) on the device: the self-test's
`RESULT ceres3d_intensity` line against the oracle on the same inputs (rebuilt here from the
self-test's formulas, tests/intensity3d_oracle.py; doubles, 1e-7)."""
import os
import subprocess

import numpy as np
import pytest

from tests import intensity3d_oracle as iorc
from tests.test_gpu_adapter import ADAPTER, lround


def _selftest_cloud3():
    """adapter_selftest.cc's 12-point axis cloud and the cells of its HybridGrid."""
    cloud3, idx = [], []
    tx, ty, tz = np.float32(0.2), np.float32(-0.15), np.float32(0.1)
    for axis in range(3):
        d = np.float32(4.0)
        while d <= 5.5:
            p = [np.float32(0), np.float32(0), np.float32(0)]
            p[axis] = d
            cloud3.append(p)
            idx.append([lround(np.float32(p[0] + tx) / np.float32(0.05)),
                        lround(np.float32(p[1] + ty) / np.float32(0.05)),
                        lround(np.float32(p[2] + tz) / np.float32(0.05))])
            d = np.float32(d + np.float32(0.5))
    return np.array(cloud3, np.float32), np.array(idx, np.int32)


@pytest.mark.gpu
def test_adapter_ceres3d_intensity_equals_the_oracle(oracle):
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [ln.split()[2:] for ln in out.stdout.splitlines()
             if ln.startswith("RESULT ceres3d_intensity ")]
    assert len(lines) == 1, out.stdout
    got = lines[0]
    cloud3, idx = _selftest_cloud3()
    ohi = oracle.HybridGrid(0.05, idx, np.full(len(idx), 24575, np.uint16))
    oint = iorc.IntensityHybridGrid(0.05, idx, np.full(len(idx), 50.0, np.float32),
                                      np.ones(len(idx), np.int32))
    intensities = np.full(len(cloud3), 50.0, np.float32)
    intensities[3] = 150.0
    start = [0.22, -0.13, 0.08, 1, 0, 0, 0]
    want = iorc.match([(cloud3, ohi, oint, intensities)], start[:3], start, [(0.5, 0.3, 100.0)],
                      occupied_space_weights=[5.0])
    np.testing.assert_allclose([float(v) for v in got[0:7]], want["pose"], rtol=0, atol=1e-7)
    assert float(got[7]) == pytest.approx(want["initial_cost"], rel=1e-12)
    assert float(got[8]) == pytest.approx(want["final_cost"], rel=1e-9)
    assert [int(got[9]), int(got[10])] == [want["iterations"], want["num_successful_steps"]]
    assert oracle.CERES_TERMINATION[int(got[11])] == want["termination"]
