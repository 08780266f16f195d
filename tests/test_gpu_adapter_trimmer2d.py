"""The C++ adapter's OverlappingSubmapsTrimmer2D (pose_graph_trimmer_b200.h) on device grids:
the reference's seven overlapping_submaps_trimmer_2d_test.cc cases (adapter_selftest.cc,
`trimmer2d_*` RESULT lines), and one random map whose inputs the self-test prints beside its
trimmed submaps, checked here against the CPU restatement (tests/trimmer2d_oracle.cc)."""
import os
import subprocess

import numpy as np
import pytest

from tests import trimmer2d_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")
CASES = ["EmptyPoseGraph", "TrimOneOfTwoOverlappingSubmaps", "TestMinAddedSubmapsCountParam_first",
         "TestMinAddedSubmapsCountParam", "DoNotTrimUnfinishedSubmap",
         "UseOnlyIntraSubmapsToComputeFreshness", "TrimSubmapWithLowCoveredCellsCount",
         "TestTransformations"]


def _submap(fields):
    fresh = int(fields[1])
    mx, my, res = (float(v) for v in fields[2:5])
    pose = [float(v) for v in fields[5:12]]
    size = int(fields[12])
    hexcells = fields[13]
    cells = np.array([int(hexcells[4 * k:4 * k + 4], 16) for k in range(size * size)],
                     np.uint16).reshape(size, size)
    ys, xs = np.nonzero(cells)
    box = (int(xs.min()), int(ys.min()), int(xs.max()), int(ys.max())) if len(xs) else None
    return (cells, box, (mx, my, res), pose, fresh)


@pytest.mark.gpu
def test_adapter_trimmer_cases():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr
    lines = [ln.split() for ln in out.stdout.splitlines() if ln.startswith("RESULT trimmer2d_")]
    res = {ln[1]: ln[2:] for ln in lines}
    for name in CASES:
        assert res["trimmer2d_" + name][0] == "ok", (name, res.get("trimmer2d_" + name))
    subs = [_submap(ln[2:]) for ln in lines if ln[1] == "trimmer2d_random_submap"]
    assert len(subs) == 40
    first = subs[0][2]
    # Trimmer(2, 0.5, 0): min_covered_cells_count = uint16(0.5 / resolution^2)
    trim, _, want = O.trim(subs, first, 2, int(0.5 / (first[2] * first[2])))
    trimmed = res["trimmer2d_random_map"][0] if res["trimmer2d_random_map"] else ""
    assert trimmed == "".join("%d," % i for i in np.nonzero(trim)[0])
    assert 0 < trim.sum() < len(trim)
    entries, cells = (int(v) for v in res["trimmer2d_random_map_stats"])
    assert (entries, cells) == (want["entries"], want["coverage_cells"])
