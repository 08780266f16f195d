"""The C++ adapter's io::XRayPointsProcessor (adapter_selftest.cc, `xr_*` RESULT lines) against
the CPU restatement: three batches in three floors, one floor without points; the stand-in
Image writes its cairo words, so the lines list every floor's pixels."""
import os
import subprocess

import numpy as np
import pytest

from tests import xray_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")
TRANSFORM = (0.5, -0.25, 0.125, 0.8, 0.0, 0.6, 0.0)
FLOORS = [[(0, 1)], [(1, 2)], [(5, 6)]]


def _fixture():
    """The self-test's batches: (start_time, points, colours or None)."""
    f = np.float32
    i = np.arange(300)
    out = []
    for b in range(3):
        pts = np.stack([f((i * 7) % 23) * f(0.1), f((i * 11) % 17) * f(0.1) - f(0.8),
                        f(i % 9) * f(0.15) + f(b) * f(0.2)], 1).astype(np.float32)
        cols = None if b == 1 else np.stack(
            [f(i % 10) * f(0.1), np.full(300, f(b) * f(0.3)), f((i * 3) % 7) / f(7.0)],
            1).astype(np.float32)
        out.append((b, pts, cols))
    return out


@pytest.mark.gpu
def test_adapter_xray_matches_oracle():
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT xr_")}
    assert res["xr_action"] == ["write_xray_image"]
    assert res["xr_flush"] == ["1", "3"]              # kFinished; every batch passed on
    o = O.Processor(0.25, 1.5, TRANSFORM, num_aggregations=3)
    for t, pts, cols in _fixture():
        for k, spans in enumerate(FLOORS):
            if any(a <= t <= b for a, b in spans):
                assert o.insert(pts, cols, aggregation=k)
    lo, hi, empty = o.bounding_box()
    assert res["xr_box"] == [str(v) for v in [int(empty)] + lo.tolist() + hi.tolist()]
    assert sorted(k for k in res if k.startswith("xr_file_")) == \
        ["xr_file_xray%d.png" % k for k in range(3)]
    for k in range(3):
        want = o.draw(k)
        assert [int(v) for v in res["xr_file_xray%d.png" % k]] == want.ravel().tolist()
    assert (o.draw(2) == 0xFFFFFFFF).all()
    assert len({int(v) for v in o.draw(0).ravel()}) > 5
