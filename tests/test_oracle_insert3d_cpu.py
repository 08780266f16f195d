"""The CPU restatement of RangeDataInserter3D (tests/insert3d_oracle.py) against the
reference's range_data_inserter_3d_test.cc and an independent C++ build of its lookup tables;
the inserter's C ABI records and status codes without a device."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import insert3d_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = dict(hit_probability=0.7, miss_probability=0.4, num_free_space_voxels=1000,
           intensity_threshold=100.0)   # range_data_inserter_3d_test.cc:33-38
REF_RETURNS = np.array([[-3, -1, 4], [-2, 0, 4], [-1, 1, 4], [0, 2, 4]], np.float32)


def _insert_point_cloud(ins, g, ig=None, intensities=None):
    ins.insert([0.0, 0.0, -4.0], REF_RETURNS, intensities, g, ig)


def _check_ray_and_hits(g, ig=None):
    for c in ([0, 0, -4], [0, 0, -3], [0, 0, -2]):
        assert abs(g.get_probability([c])[0] - 0.4) < 1e-4
    for x in range(-4, 5):
        for y in range(-4, 5):
            if x < -3 or x > 0 or y != x + 2:
                assert g.value([[x, y, 4]])[0] == 0
                if ig is not None:
                    assert abs(ig.get_intensity([[x, y, 4]])[0]) < 1e-6
            else:
                assert abs(g.get_probability([[x, y, 4]])[0] - 0.7) < 1e-4
                if ig is not None:
                    assert abs(ig.get_intensity([[x, y, 4]])[0] - (10 + x)) < 1e-6


def test_insert_point_cloud():
    ins, g = O.RangeDataInserter3D(**REF), O.HybridGrid(1.0)
    _insert_point_cloud(ins, g)
    _check_ray_and_hits(g)


def test_insert_point_cloud_with_intensities():
    ins, g, ig = O.RangeDataInserter3D(**REF), O.HybridGrid(1.0), O.IntensityHybridGrid(1.0)
    _insert_point_cloud(ins, g, ig, np.float32([7, 8, 9, 10]))
    _check_ray_and_hits(g, ig)


def test_probability_progression():
    ins, g = O.RangeDataInserter3D(**REF), O.HybridGrid(1.0)
    _insert_point_cloud(ins, g)
    assert abs(g.get_probability([[-2, 0, 4]])[0] - 0.7) < 1e-4
    assert abs(g.get_probability([[-2, 0, 3]])[0] - 0.4) < 1e-4
    assert abs(g.get_probability([[0, 0, -3]])[0] - 0.4) < 1e-4
    for _ in range(1000):
        _insert_point_cloud(ins, g)
    assert abs(g.get_probability([[-2, 0, 4]])[0] - 0.9) < 1e-3
    assert abs(g.get_probability([[-2, 0, 3]])[0] - 0.1) < 1e-3
    assert abs(g.get_probability([[0, 0, -3]])[0] - 0.1) < 1e-3


def test_lookup_tables_match_a_cpp_build():
    """ComputeLookupTableToApplyOdds compiled from oracle/oracle_common.h's float helpers."""
    src = r'''
#include <cstdio>
#include "oracle/oracle_common.h"
using namespace oracle;
int main(int argc, char** argv) {
  const double probs[4] = {0.7, 0.4, 0.55, 0.49};
  for (double prob : probs) {
    const float odds = Odds(static_cast<float>(prob));
    for (int cell = 0; cell != 32768; ++cell) {
      const float p = cell == 0 ? ProbabilityFromOdds(odds)
          : ProbabilityFromOdds(odds * Odds(SlowValueToBoundedFloat(cell, 0, kMinProbability,
                                                                    kMinProbability, kMaxProbability)));
      std::printf("%d\n", ProbabilityToValue(p) + kUpdateMarker);
    }
  }
}
'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.cc"), "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-I", ROOT,
                               os.path.join(d, "t.cc"), "-o", os.path.join(d, "t")])
        want = np.array(subprocess.check_output([os.path.join(d, "t")]).split(), np.int64)
    got = np.concatenate([O.lookup_table(O.odds(np.float32(p))) for p in (0.7, 0.4, 0.55, 0.49)])
    np.testing.assert_array_equal(got, want.reshape(-1))


def test_hits_win_over_misses_in_either_order():
    """A hit cell that another ray crosses ends at the hit table's value."""
    for order in ([[3, 0, 0], [6, 0, 0]], [[6, 0, 0], [3, 0, 0]]):
        ins, g = O.RangeDataInserter3D(**dict(REF, num_free_space_voxels=2)), O.HybridGrid(1.0)
        ins.insert([0, 0, 0], np.float32(order), None, g)
        assert g.value([[3, 0, 0]])[0] == ins.hit_table[0] - O.K_UPDATE_MARKER
        assert g.value([[5, 0, 0]])[0] == ins.miss_table[0] - O.K_UPDATE_MARKER
        assert g.value([[4, 0, 0]])[0] == ins.miss_table[0] - O.K_UPDATE_MARKER
        assert g.value([[0, 0, 0]])[0] == 0   # before the last two samples of either ray


def test_miss_samples_truncate_towards_zero():
    ins = O.RangeDataInserter3D(**dict(REF, num_free_space_voxels=3))
    cells = ins.miss_cells(np.int64([0, 0, 0]), np.int64([[-7, 3, -2]]))
    # positions 4, 5, 6 of 7: delta * p / 7 with C++ division
    want = [[int(-7 * p / 7), int(3 * p / 7), int(-2 * p / 7)] for p in (4, 5, 6)]
    np.testing.assert_array_equal(cells, want)


def test_intensity_threshold_keeps_equal_values():
    ins = O.RangeDataInserter3D(**REF)
    g, ig = O.HybridGrid(1.0), O.IntensityHybridGrid(0.5)
    ins.insert([0, 0, 0], np.float32([[1, 1, 1], [1, 1, 1], [1, 1, 1]]),
               np.float32([100.0, 100.5, 20.0]), g, ig)
    assert ig.counts.tolist() == [2] and ig.sums.tolist() == [120.0]


def test_cells_outside_the_cube_are_refused():
    ins, g = O.RangeDataInserter3D(**REF), O.HybridGrid(0.1)
    with pytest.raises(ValueError):
        ins.insert([0, 0, 0], np.float32([[900.0, 0, 0]]), None, g)
    assert len(g.keys) == 0


# ---- the C ABI without a device ----
@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def test_inserter_struct_layout(csm):
    from cartographer_b200 import scan_matching as sm
    t = sm.CsmRangeInserterOptions3D
    head = '#include <stdio.h>\n#include <stddef.h>\n#include "include/csm_abi.h"\nint main(){'
    body = 'printf("%zu\\n", sizeof(csm_range_inserter_options3d));' + "".join(
        'printf("%%zu\\n", offsetof(csm_range_inserter_options3d, %s));' % f for f, _ in t._fields_)
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(head + body + "}")
        subprocess.check_call(["gcc", "-I", ROOT, os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        got = [int(v) for v in subprocess.check_output([os.path.join(d, "t")]).split()]
    assert got == [C.sizeof(t)] + [getattr(t, f).offset for f, _ in t._fields_]


def test_invalid_options_and_no_device(csm):
    from cartographer_b200 import scan_matching as sm
    lib = csm.lib()
    out = C.c_void_p()
    for bad in (dict(REF, hit_probability=0.5), dict(REF, miss_probability=0.5),
                dict(REF, num_free_space_voxels=-1)):
        o = sm.RangeDataInserterOptions3D(**bad)._c()
        assert lib.csm_range_inserter3d_create(C.byref(o), 0, C.byref(out)) == 1
    assert lib.csm_range_inserter3d_create(None, 0, C.byref(out)) == 1
    assert lib.csm_range_inserter3d_insert(None, None, None, None, 0, None, None, None) == 1
    assert lib.csm_range_inserter3d_destroy(None) == 0
    lo, dims = (C.c_int32 * 3)(), (C.c_int32 * 3)()
    assert lib.csm_grid3d_read(None, lo, dims, None) == 1
    assert lib.csm_intensity_grid3d_read(None, lo, dims, None, None, None) == 1
    count = C.c_int32(0)
    if lib.csm_device_count(C.byref(count)) == 0 and count.value > 0:
        pytest.skip("GPU present")
    o = sm.RangeDataInserterOptions3D(**REF)._c()
    assert lib.csm_range_inserter3d_create(C.byref(o), 0, C.byref(out)) == 2, "expected CSM_E_CUDA"
