"""The C++ adapter's sensor::VoxelFilter overloads and AdaptiveVoxelFilter
(adapter_selftest.cc, `vf_*` RESULT lines) against the CPU restatement: each payload carries its
point's input index, so the lines list the kept indices."""
import os
import subprocess

import numpy as np
import pytest

from tests import voxel_filter_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


def _fixture():
    i = np.arange(2000)
    return np.stack([((i * 37) % 101).astype(np.float32) * np.float32(0.05),
                     ((i * 53) % 89).astype(np.float32) * np.float32(0.05),
                     (i % 13).astype(np.float32) * np.float32(0.1)], 1).astype(np.float32)


@pytest.mark.gpu
def test_adapter_voxel_filter_matches_oracle():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: [int(v) for v in ln.split()[2:]] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT vf_")}
    pts = _fixture()
    assert res["vf_cloud"] == list(O.voxel_filter(pts, 0.3)[0])
    assert res["vf_points"] == [len(res["vf_cloud"])]
    assert res["vf_timed"] == list(O.voxel_filter(pts, 0.2)[0])
    assert res["vf_range"] == list(O.voxel_filter(pts, 0.5)[0])
    assert res["vf_adaptive"] == list(O.adaptive_voxel_filter(pts, 2.0, 150.0, 4.0)[0])
