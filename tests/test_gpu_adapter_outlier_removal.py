"""The C++ adapter's io::OutlierRemovingPointsProcessor (adapter_selftest.cc, `or_*` RESULT
lines) against the CPU restatement: intensities carry each point's input index and colors its
index and batch, so the lines list the kept indices and show that the payloads follow them."""
import os
import subprocess

import numpy as np
import pytest

from tests import outlier_removal_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


def _fixture():
    """The self-test's three batches: a wall at x = 5 and a patch in front of it per batch."""
    f = np.float32
    i = np.arange(600)
    batches = []
    for b in range(3):
        wall = np.stack([np.full(400, f(5.0)), f(i[:400] % 20) * f(0.1) - f(1.0),
                         f(i[:400] // 20) * f(0.1)], 1)
        j = i[400:]
        patch = np.stack([np.full(200, f(2.0) + f(b)), f(j % 10) * f(0.1) - f(0.5),
                          f((j // 10) % 10) * f(0.1)], 1)
        origin = np.array([f(b) * f(0.3), f(b) * f(-0.2), f(1.0)], np.float32)
        batches.append((origin, np.concatenate([wall, patch]).astype(np.float32)))
    return batches


@pytest.mark.gpu
def test_adapter_outlier_removal_matches_oracle():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT or_")}
    assert res["or_action"] == ["voxel_filter_and_remove_moving_objects"]
    assert res["or_flush"] == ["0", "0", "1"]        # kRestartStream twice, then kFinished
    _, _, kept = O.run(_fixture(), 0.1, 3.0)
    assert sum(len(k) for k in kept) < 3 * 600       # the patches the other rays cross go
    for b, k in enumerate(kept):
        assert [int(v) for v in res["or_kept_%d" % b]] == k.tolist()
        assert [int(v) for v in res["or_colors_%d" % b]] == k.tolist()
        assert res["or_points_%d" % b] == ["1"] * len(k)
