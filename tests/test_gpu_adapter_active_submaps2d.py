"""The C++ adapter's ActiveSubmaps2D (adapter_selftest.cc, `active2d0` / `active2d1` /
`evicted2d` RESULT lines) against scan_matching.ActiveSubmaps2D driven with the same seven
scans: every grid's cells, limits and known-cells box, num_range_data, insertion_finished and
the local poses, bit for bit."""
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
    active = sm.ActiveSubmaps2D(sm.SubmapsOptions2D(num_range_data=2, resolution=0.05))
    first = None
    for k in range(7):
        origin = F([F(0.3) * F(k), F(-0.2) * F(k), 0])
        returns, misses = [], []
        for i in range(180):
            a = 0.035 * i + 0.1 * k
            r = F(5.0) if i % 7 == 3 else F(2.0) + F(0.01) * F(i % 40)
            p = [origin[0] + r * F(math.cos(a)), origin[1] + r * F(math.sin(a)), F(0)]
            (misses if i % 7 == 3 else returns).append(p)
        subs = active.InsertRangeData(origin, np.array(returns, F), np.array(misses, F))
        first = first or subs[0]
    return subs + [first]


@pytest.mark.gpu
def test_adapter_active_submaps2d_matches_python():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT ")}
    subs = _python_side()
    assert subs[2] not in subs[:2] and subs[2].insertion_finished
    for name, sub in zip(("active2d0", "active2d1", "evicted2d"), subs):
        got = res[name + "_grid"]
        st = sub.grid.read()
        assert [int(v) for v in got[:2]] == [st.cells.shape[1], st.cells.shape[0]]
        assert [float(v) for v in got[2:5]] == [st.resolution, st.max_x, st.max_y]
        box = None if int(got[5]) else tuple(int(v) for v in got[6:10])
        assert box == st.known_cells_box
        np.testing.assert_array_equal(np.array([int(v) for v in got[10:]], np.uint16),
                                      st.cells.reshape(-1))
        state = res[name + "_state"]
        assert int(state[0]) == sub.num_range_data
        assert int(state[1]) == int(sub.insertion_finished)
        assert tuple(float(v) for v in state[2:]) == sub.local_pose
    assert subs[2].num_range_data == 4
