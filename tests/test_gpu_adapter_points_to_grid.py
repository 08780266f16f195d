"""The C++ adapter's io::ProbabilityGridPointsProcessor (PNG and PB), io::DrawProbabilityGrid and
io::HybridGridPointsProcessor (adapter_selftest.cc, `pg_*` RESULT lines) against the Python
stages on the same three batches, and the image against the DrawProbabilityGrid restatement."""
import os
import subprocess

import numpy as np
import pytest

from tests import probability_grid_draw_oracle as O

ADAPTER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "cartographer_b200", "adapter")


def _fixture(pp):
    """The self-test's batches, with the same float steps."""
    f = np.float32
    i = np.arange(400)
    out = []
    for b in range(3):
        ox, oy = f(b) * f(0.7) - f(0.5), f(b) * f(-0.4) + f(0.2)
        pts = np.stack([f((i * 37) % 161 - 80) * f(0.05) + ox, f((i * 53) % 149 - 74) * f(0.05) + oy,
                        f(i % 5) * f(0.1)], 1).astype(np.float32)
        out.append(pp.PointsBatch(pts, origin=(ox, oy, f(0.25))))
    return out


class Files:
    def __init__(self):
        self.data = {}

    def __call__(self, name):
        files = self

        class Writer:
            def write(self, b):
                files.data[name] = files.data.get(name, b"") + bytes(b)

            def close(self):
                pass
        files.data[name] = b""
        return Writer()


@pytest.mark.gpu
def test_adapter_map_writers_match_the_python_stages():
    from cartographer_b200 import points_processing as pp
    from cartographer_b200 import scan_matching as sm
    exe = os.path.join(ADAPTER, "adapter_selftest")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", ADAPTER, "-s"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    res = {ln.split()[1]: ln.split()[2:] for ln in out.stdout.splitlines()
           if ln.startswith("RESULT pg_")}
    assert res["pg_action"] == ["write_probability_grid", "write_hybrid_grid"]
    assert res["pg_flush"] == ["3", "9"]           # kFinished thrice; every batch passed on
    assert res["pg_files"] == ["3"]
    files = Files()
    o2 = sm.ProbabilityGridRangeDataInserterOptions2D(0.55, 0.49, True)
    o3 = sm.RangeDataInserterOptions3D(0.55, 0.49, 2, 40.0)
    stages = [pp.ProbabilityGridPointsProcessor(0.05, o2, "map", "png", files),
              pp.ProbabilityGridPointsProcessor(0.05, o2, "map", "pb", files),
              pp.HybridGridPointsProcessor(0.1, o3, "map_3d", files)]
    for batch in _fixture(pp):
        for stage in stages:
            stage.Process(batch)
    pixels, offset = stages[0].grid.draw()
    st = stages[0].grid.read()
    want, want_offset = O.draw(st.cells, st.known_cells_box)
    np.testing.assert_array_equal(pixels, want)
    assert st.cells.shape[1] > 100                 # the batches grew the grid
    h, w = pixels.shape
    assert res["pg_image"] == [str(v) for v in (w, h, offset[0], offset[1])]
    assert offset == want_offset
    for stage in stages:
        assert stage.Flush() == pp.FlushResult.kFinished
    assert [int(v) for v in res["pg_file_map.png"]] == pixels.ravel().tolist()
    np.testing.assert_array_equal(pp.decode_png(files.data["map.png"]), pp.cairo_to_rgb(pixels))
    assert bytes.fromhex(res["pg_file_map.pb"][0]) == files.data["map.pb"]
    assert bytes.fromhex(res["pg_file_map_3d"][0]) == files.data["map_3d"]
    assert len(files.data["map_3d"]) > 100
