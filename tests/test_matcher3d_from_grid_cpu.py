"""CPU checks of csm_matcher3d_create_from_grid3d: the declaration and export, a refusal that
needs no device, and the premise behind deriving the grid size from a handle's non-zero cells."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import insert3d_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_declared_and_exported():
    with open(os.path.join(ROOT, "include", "csm_abi.h")) as f:
        header = f.read()
    assert re.search(r"csm_status csm_matcher3d_create_from_grid3d\(const csm_grid3d\* hybrid_grid,",
                     header)
    from cartographer_b200._lib import lib
    assert hasattr(lib(), "csm_matcher3d_create_from_grid3d")


def test_null_handle_is_refused_without_a_device():
    from cartographer_b200._lib import lib
    from cartographer_b200.scan_matching import CsmOptions3D
    o = CsmOptions3D(8, 3, 0.77, 0.55, 5.0, 1.0, 0.26)
    out = C.c_void_p(0x1234)
    rc = lib().csm_matcher3d_create_from_grid3d(None, C.c_int32(0), None, None, C.c_int32(0),
                                                C.byref(o), C.byref(out))
    assert rc == 1   # CSM_E_INVALID
    assert out.value == 0x1234


# The box of a handle's non-zero cells is the box of the voxels the reference's DynamicGrid
# allocated for, because ApplyLookupTable never leaves a cell at 0: every entry of the hit and
# miss tables (ComputeLookupTableToApplyOdds), the one for value 0 included, is non-zero in its
# 15 value bits for every option the inserter accepts (hit in (0.5, 1), miss in [0, 0.5)).
@pytest.mark.parametrize("probability", [0.0, 1e-6, 0.1, 0.3, 0.49, 0.4999999, 0.5000001, 0.51,
                                         0.55, 0.7, 0.9, 0.999999])
def test_tables_never_write_zero(probability):
    table = O.lookup_table(O.odds(np.float32(probability)))
    assert len(table) == 32768
    assert np.all(table & 0x7fff != 0)
    assert np.all(table & 0x8000)


def test_inserted_cells_are_non_zero():
    """An insert through the restatement leaves every cell it touched non-zero, with hit and
    miss probabilities at the ends of their ranges."""
    for hit, miss in ((0.5000001, 0.0), (0.999999, 0.4999999), (0.55, 0.49)):
        ins = O.RangeDataInserter3D(hit, miss, 1000, 100.0)
        g = O.HybridGrid(0.1)
        rng = np.random.RandomState(0)
        for _ in range(3):
            ins.insert([0.0, 0.0, 0.0], rng.uniform(-2, 2, size=(50, 3)).astype(np.float32),
                       None, g)
        assert len(g.values) > 50
        assert np.all(g.values != 0)
