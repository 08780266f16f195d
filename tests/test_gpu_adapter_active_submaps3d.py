"""The C++ adapter's ActiveSubmaps3D (adapter_selftest.cc, `active0` / `active1` / `evicted`
RESULT lines) against scan_matching.ActiveSubmaps3D driven with the same seven scans: every
handle's box and voxels, the intensity sums, counts and means, num_range_data,
insertion_finished and the histograms, bit for bit."""
import math
import os
import subprocess

import numpy as np
import pytest

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")
F = np.float32


def _python_side():
    from cartographer_b200 import scan_matching as sm
    options = sm.SubmapsOptions3D(
        high_resolution=0.1, high_resolution_max_range=4.0, low_resolution=0.45,
        num_range_data=2, range_data_inserter_options=sm.RangeDataInserterOptions3D(
            hit_probability=0.55, miss_probability=0.49, num_free_space_voxels=2,
            intensity_threshold=40.0))
    active = sm.ActiveSubmaps3D(options)
    first = None
    i = np.arange(240)
    for k in range(7):
        pts = np.stack([F(-3) + F(0.125) * (i % 48).astype(F) + F(0.25) * F(k),
                        F(2) - F(0.5) * (i // 48).astype(F),
                        F(1.5) - F(0.25) * (i % 5).astype(F)], 1).astype(F)
        q = [math.cos(0.05 * k), 0.0, 0.0, math.sin(0.05 * k)]
        subs = active.InsertData(F([0.25 * k, -0.125 * k, 0.5]), pts, (i % 60).astype(F), q,
                                 np.arange(8, dtype=F) + F(k))
        first = first or subs[0]
    return subs + [first]


@pytest.mark.gpu
def test_adapter_active_submaps3d_matches_python():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT ")}
    subs = _python_side()
    assert subs[2] not in subs[:2] and subs[2].high_resolution_intensity_hybrid_grid is None
    for name, sub in zip(("active0", "active1", "evicted"), subs):
        for side, grid in (("high", sub.high_resolution_hybrid_grid),
                           ("low", sub.low_resolution_hybrid_grid)):
            lo, vol = grid.read()
            got = [int(v) for v in res["%s_%s" % (name, side)]]
            assert got[:3] == lo.tolist() and got[3:6] == list(vol.shape[::-1])
            np.testing.assert_array_equal(np.array(got[6:], np.uint16), vol.reshape(-1))
        state = res[name + "_state"]
        assert int(state[0]) == sub.num_range_data
        assert int(state[1]) == int(sub.insertion_finished)
        np.testing.assert_array_equal(np.array([int(h, 16) for h in state[2:]], np.uint32),
                                      sub.rotational_scan_matcher_histogram.view(np.uint32))
        got = res[name + "_intensity"]
        ig = sub.high_resolution_intensity_hybrid_grid
        assert (ig is None) == (got == ["forgotten"])
        if ig is None:
            continue
        lo, mean, sums, counts = ig.read()
        assert [int(v) for v in got[:3]] == lo.tolist()
        assert [int(v) for v in got[3:6]] == list(mean.shape[::-1])
        cells = [v.split(":") for v in got[6:]]
        np.testing.assert_array_equal(np.array([int(c[0], 16) for c in cells], np.uint32),
                                      mean.reshape(-1).view(np.uint32))
        np.testing.assert_array_equal(np.array([int(c[1], 16) for c in cells], np.uint32),
                                      sums.reshape(-1).view(np.uint32))
        np.testing.assert_array_equal(np.array([int(c[2]) for c in cells], np.int32),
                                      counts.reshape(-1))
    assert subs[0].insertion_finished is False or subs[0].num_range_data == 4
    assert subs[2].insertion_finished and subs[2].num_range_data == 4
