"""The C++ adapter's FastCorrelativeScanMatcher3D(const DeviceHybridGrid&, ...) and
ConstraintBuilder3D on a DeviceSubmap3D, on grids filled by RangeDataInserter3D: every RESULT
line the self-test prints for them equals, character for character (float bit patterns,
doubles to 17 digits), the line of the same call on host HybridGrids of the grids' non-zero
voxels."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAPTER = os.path.join(ROOT, "cartographer_b200", "adapter")

NAMES = ("fast3d_grid", "fast3d_grid_full", "cb3d_grid", "cb3d_grid_refined")


@pytest.mark.gpu
def test_device_grid_results_equal_host_grid_results():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "link check only" not in out.stdout, "no CUDA device seen by the adapter"
    lines = {}
    for ln in out.stdout.splitlines():
        if ln.startswith("RESULT "):
            name, rest = ln.split(" ", 2)[1:]
            lines.setdefault(name, []).append(rest)
    for name in NAMES:
        dev, host = lines.get(name + "_dev"), lines.get(name + "_host")
        assert dev and host, name
        assert dev == host, (name, dev, host)
    # the local match found the pose the cloud was inserted at (within a voxel)
    fields = lines["fast3d_grid_dev"][0].split()
    assert fields[0] == "1"
    for got, want in zip(fields[2:5], (0.2, -0.15, 0.1)):
        assert abs(float(got) - want) <= 0.051
    assert len(lines["cb3d_grid_dev"]) == 2 and len(lines["cb3d_grid_refined_dev"]) == 2
