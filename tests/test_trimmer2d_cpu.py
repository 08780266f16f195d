"""OverlappingSubmapsTrimmer2D's coverage pass without a device: the CPU restatement on the
reference's seven test cases and on hand-derived edges, the Python trimmer's host logic, and the
C ABI's declaration, export and refusals."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from cartographer_b200 import pose_graph as P
from tests import trimmer2d_cases as K
from tests import trimmer2d_oracle as O

IDENT = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]


@pytest.mark.parametrize("name", sorted(K.REFERENCE_CASES))
def test_reference_cases_on_the_restatement(name):
    K.REFERENCE_CASES[name](K.Builder(lambda g: g), K.OracleTrimmer)


def _one(max_x, max_y, res=1.0, t=0, cells=None, box=None, pose=IDENT):
    cells = np.ones((1, 1), np.uint16) if cells is None else cells
    if box is None:
        box = (0, 0, cells.shape[1] - 1, cells.shape[0] - 1)
    return (cells, box, (max_x, max_y, res), pose, t)


@pytest.mark.parametrize("sign", [1, -1])
def test_keys_round_half_away_from_zero_on_both_signs(sign):
    # first limits max (0, 0), resolution 1: the key is lround(-p).  Submap A's only cell centre
    # is at x = -2.5 sign (key 3 sign, 2 sign under round-half-even), B's at -3 sign (key 3 sign).
    # y: max_y 0.5 puts both centres at 0.
    a = _one(-2.0 if sign > 0 else 3.0, 0.5, t=1)
    b = _one(-2.5 if sign > 0 else 3.5, 0.5, t=2)
    trim, counts, st = O.trim([a, b], (0.0, 0.0, 1.0), 1, 1)
    assert st["coverage_cells"] == 1 and st["entries"] == 2
    assert list(trim) == [True, False] and list(counts) == [0, 1]


def test_duplicates_of_one_submap_each_count():
    # a 2 x 2 submap at resolution 0.5 puts its four cells into the key (0, 0) of resolution 1
    fine = _one(0.45, 0.45, res=0.5, t=1, cells=np.ones((2, 2), np.uint16))
    newer = _one(0.5, 0.5, t=2)
    trim, counts, st = O.trim([fine, newer], (0.0, 0.0, 1.0), 2, 1)
    assert st["coverage_cells"] == 1 and st["entries"] == 5
    assert list(counts) == [1, 1] and list(trim) == [False, False]
    trim, counts, _ = O.trim([fine, newer], (0.0, 0.0, 1.0), 8, 4)
    assert list(counts) == [4, 1] and list(trim) == [False, True]
    trim, counts, _ = O.trim([fine, newer], (0.0, 0.0, 1.0), 1, 0)
    assert list(counts) == [0, 1] and list(trim) == [True, False]   # absent: trimmed at min 0


def test_fresh_submaps_count_zero_trims_everything():
    subs = [_one(0.5, 0.5, t=1), _one(5.5, 5.5, t=2)]
    trim, counts, _ = O.trim(subs, (0.0, 0.0, 1.0), 0, 0)
    assert list(trim) == [True, True] and list(counts) == [0, 0]


@pytest.mark.parametrize("minimum,trimmed", [(0, False), (1, True)])
def test_65536_covered_cells_wrap_to_zero(minimum, trimmed):
    sub = _one(0.0, 0.0, t=1, cells=np.ones((256, 256), np.uint16))
    trim, counts, st = O.trim([sub], (0.0, 0.0, 1.0), 1, minimum)
    assert st["entries"] == 65536 and counts[0] == 65536 and trim[0] == trimmed


def test_empty_box_walks_the_cell_at_the_origin():
    cells = np.zeros((3, 3), np.uint16)
    cells[0, 0] = 5
    cells[1, 1] = 5
    trim, counts, st = O.trim([(cells, None, (0.0, 0.0, 1.0), IDENT, 1)], (0.0, 0.0, 1.0), 1, 0)
    assert st["entries"] == 1 and counts[0] == 1 and not trim[0]


def test_large_ties_are_sorted_like_std_sort():
    # 17 one-cell submaps on one global cell, all with one time: the cut takes std::sort's first
    # entry; the restatement reports the cell as a sort of more than 16 entries
    subs = [_one(0.5, 0.5, t=7) for _ in range(17)]
    trim, counts, st = O.trim(subs, (0.0, 0.0, 1.0), 1, 1)
    assert st["sorted_large"] == 1 and int(counts.sum()) == 1 and int((~trim).sum()) == 1


# ---- the Python trimmer's host logic, without the library ----

class _NoLibrary(P.OverlappingSubmapsTrimmer2D):
    def _limits(self, grid):
        raise AssertionError("the library was reached")

    _coverage = _limits


def test_early_return_in_size_t_arithmetic():
    b = K.Builder(lambda g: g)
    K._two_overlapping(b)
    t = _NoLibrary(1, 0, 2)
    t.Trim(b.pg)   # 2 - 0 <= 2
    assert b.pg.trimmed == []
    t.current_submap_count = 3   # 2 - 3 wraps to 2^64 - 1 in size_t: no early return
    with pytest.raises(AssertionError, match="library"):
        t.Trim(b.pg)


def test_no_participating_submap_does_not_reach_the_library():
    b = K.Builder(lambda g: g)
    K._two_overlapping(b)
    b.pg.constraints = [K.Constraint((0, 0), (0, 0), P.INTER_SUBMAP)]   # no freshness
    t = _NoLibrary(1, 0, 0)
    t.Trim(b.pg)
    assert b.pg.trimmed == [] and t.current_submap_count == 2


def test_freshness_uses_the_largest_intra_submap_node():
    b = K.Builder(lambda g: g)
    K._two_overlapping(b)
    b.node(5, 9000)
    b.node(3, 500)
    b.constraint(0, 5, False)
    b.constraint(0, 3, True)
    b.constraint(1, 7, True)   # a node that does not exist: no freshness for submap 1
    b.constraint(4, 0, True)   # a submap that does not exist
    f = P.compute_submap_freshness(b.pg.submap_data, b.pg.nodes, b.pg.constraints)
    assert f == {(0, 0): 500}


def test_uint16_conversions():
    assert P.double_to_uint16(65535.9) == 65535 and P.double_to_uint16(-0.9) == 0
    for bad in (65536.0, -1.0, math.nan, math.inf):
        with pytest.raises(ValueError):
            P.double_to_uint16(bad)
    with pytest.raises(ValueError):
        P.OverlappingSubmapsTrimmer2D(65536, 0, 0)
    b = K.Builder(lambda g: g)
    K._two_overlapping(b)
    with pytest.raises(ValueError):
        K.OracleTrimmer(1, 65536.0, 0).Trim(b.pg)


def test_composition_is_global_times_local_inverse():
    g = K.embed3d(1.0, 2.0, 0.3)
    loc = K.embed3d(-0.5, 0.25, -0.7)
    p = P.global_frame_from_local_frame(g, loc)
    # applied to the local pose's origin it gives the global pose's origin
    q = P._rotate(p[3:], loc[:3])
    assert np.allclose([q[k] + p[k] for k in range(3)], g[:3], atol=1e-12)
    assert math.isclose(math.atan2(p[6], p[3]) * 2, 1.0, abs_tol=1e-12)


# ---- the C ABI ----

def test_abi_declares_the_entry_point():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "csm_abi.h")) as f:
        h = f.read()
    for s in ("csm_trim_overlapping_submaps2d(", "typedef struct csm_coverage_submap2d",
              "typedef struct csm_coverage_stats2d"):
        assert s in h
    assert C.sizeof(P.CsmCoverageSubmap2D) == 8 + 24 + 32 + 8
    assert C.sizeof(P.CsmCoverageStats2D) == 4 * 8 + 8


@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def _call(csm, recs, n, first=(0.0, 0.0, 1.0), trim=True, counts=True):
    t = np.full(max(n, 1), 7, np.uint8)
    c = np.full(max(n, 1), 7, np.uint32)
    st = csm.lib().csm_trim_overlapping_submaps2d(
        recs, C.c_int32(n), C.c_double(first[0]), C.c_double(first[1]), C.c_double(first[2]),
        C.c_uint16(1), C.c_uint16(0), t.ctypes.data_as(C.c_void_p) if trim else None,
        c.ctypes.data_as(C.c_void_p) if counts else None, None)
    assert np.all(t == 7) and np.all(c == 7)   # nothing written
    return st


def test_symbol_exported_and_refusals(csm):
    L = csm.lib()
    assert hasattr(L, "csm_trim_overlapping_submaps2d")
    recs = (P.CsmCoverageSubmap2D * 1)()
    recs[0].rotation[0] = 1.0
    assert _call(csm, None, 1) == 1                    # null submaps
    assert _call(csm, recs, 1) == 1                    # null grid
    assert _call(csm, recs, 1, trim=False) == 1
    assert _call(csm, recs, 1, counts=False) == 1
    assert _call(csm, recs, -1) == 1
    for bad in ((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), (math.nan, 0.0, 1.0), (0.0, math.inf, 1.0),
                (0.0, 0.0, math.nan)):
        assert _call(csm, recs, 1, first=bad) == 1
    assert _call(csm, recs, 0) == 0                    # n = 0: nothing to do
    d = C.c_double()
    assert L.csm_rt_grid2d_limits(None, C.byref(d), None, None, None, None) == 1


def test_no_handle_exists_without_a_device(csm):
    """Stands for "csm_trim_overlapping_submaps2d returns CSM_E_CUDA without a device", which
    cannot be reached: every submap passes a grid handle, and without a device no handle can be
    made, so the check is on the creation, which returns CSM_E_CUDA.  The trim call itself is
    checked here only for the refusals that come before any device work (above)."""
    n = C.c_int32(0)
    if csm.lib().csm_device_count(C.byref(n)) == 0 and n.value > 0:
        pytest.skip("a device is present")
    h = C.c_void_p()
    st = csm.lib().csm_rt_grid2d_create_empty(C.c_double(0.05), C.c_double(1.0), C.c_double(1.0),
                                              C.c_int32(4), C.c_int32(4), C.c_int32(0),
                                              C.byref(h))
    assert st == 2
