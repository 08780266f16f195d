"""The C++ adapter's ConstraintBuilder2D on DeviceSubmap2Ds (adapter_selftest.cc, the
`cb2d_device_submaps*` RESULT lines): two submaps grown by ProbabilityGridRangeDataInserter2D
and cropped on the device give, through two rounds of the reference's call cycle with a
DeleteScanMatcher in between, unrefined and refined, the constraints and candidate counts of the
same queues on host Submap2Ds made from the cells read back, bit for bit."""
import os
import subprocess

import pytest

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


@pytest.mark.gpu
def test_adapter_cb2d_on_device_submaps_equals_host_submaps():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = {}
    for ln in out.stdout.splitlines():
        f = ln.split()
        if ln.startswith("RESULT cb2d_device_submaps"):
            lines.setdefault(f[1], []).append(f[2:])
    for refined in ("", "_refined"):
        dev = lines["cb2d_device_submaps%s_dev" % refined]
        host = lines["cb2d_device_submaps%s_host" % refined]
        assert dev == host
        assert {row[0] for row in dev} == {"0", "1"}       # both rounds found constraints
        assert {row[1] for row in dev} == {"0", "1"}       # on both submaps
    # the refinement moved the poses and left the searches as they were
    plain, refined = lines["cb2d_device_submaps_dev"], lines["cb2d_device_submaps_refined_dev"]
    assert [r[:3] + r[-1:] for r in plain] == [r[:3] + r[-1:] for r in refined]
    assert [r[3:7] for r in plain] != [r[3:7] for r in refined]
