"""CPU checks of saving device grids (csm_grid3d_voxels, csm_grid3d_to_proto,
csm_rt_grid2d_to_proto): declarations and exports, refusals that need no device, the HybridGrid
walk restatement against hand-derived orders, and the reference encoders against hand-written
bytes."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

from tests import grid_proto_ref as R
from tests import protowire as pw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = {
    "csm_grid3d_voxels": r"csm_status csm_grid3d_voxels\(const csm_grid3d\* grid, int32_t\* indices,",
    "csm_grid3d_to_proto": r"csm_status csm_grid3d_to_proto\(const csm_grid3d\* grid, uint8_t\* buf,",
    "csm_rt_grid2d_to_proto":
        r"csm_status csm_rt_grid2d_to_proto\(const csm_rt_grid2d\* grid, uint8_t\* buf,",
}


def test_declared_and_exported():
    with open(os.path.join(ROOT, "include", "csm_abi.h")) as f:
        header = f.read()
    from cartographer_b200._lib import lib
    for name, pattern in ENTRIES.items():
        assert re.search(pattern, header), name
        assert hasattr(lib(), name), name


def test_null_arguments_are_refused_without_a_device():
    from cartographer_b200._lib import lib
    n = C.c_int64(-7)
    assert lib().csm_grid3d_voxels(None, None, None, C.c_int64(0), C.byref(n)) == 1
    assert n.value == -7
    assert lib().csm_grid3d_to_proto(None, None, C.c_int64(0), C.byref(n)) == 1
    assert lib().csm_rt_grid2d_to_proto(None, None, C.c_int64(0), C.byref(n)) == 1
    assert n.value == -7


# ---- the HybridGrid walk restatement against orders derived by hand ----
def test_walk_hand_derived_order():
    # z >> 6 first (j has z = -1), then y >> 6, x >> 6 (f: -2, e and a: -1, h: 1); inside a 64^3
    # block the 8^3 block (a: x >> 3 & 7 = 7 after e's 0; d: 1, g: 7), then z & 7, y & 7, x & 7
    # (i: y = 1 after b and c)
    named = dict(a=(-1, 0, 0), b=(0, 0, 0), c=(7, 0, 0), d=(8, 0, 0), e=(-64, 0, 0),
                 f=(-65, 0, 0), g=(63, 0, 0), h=(64, 0, 0), i=(0, 1, 0), j=(0, 0, -1))
    want = "jfeabcidgh"
    keys = sorted(named)
    idx = np.array([named[k] for k in keys], np.int32)
    val = np.arange(1, len(keys) + 1, dtype=np.uint16)
    got, gval, bits = R.walk((idx, val))
    assert bits == 2   # -65 and 64 are outside the first 128^3 cube
    assert "".join(keys[v - 1] for v in gval) == want
    np.testing.assert_array_equal(got, [named[k] for k in want])


EDGES = (-65, -64, -9, -8, -1, 0, 7, 8, 63, 64)


def _blocked_key(idx):
    x, y, z = (idx[:, a].astype(np.int64) for a in range(3))
    return np.lexsort([x & 7, y & 7, z & 7, (x >> 3) & 7, (y >> 3) & 7, (z >> 3) & 7,
                       x >> 6, y >> 6, z >> 6])


@pytest.mark.parametrize("history", ["grow_once", "grow_many", "far_first"])
def test_walk_edges_on_both_signs(history):
    """Voxels straddling the 8- and 64-cell boundaries on both signs of every axis, written in
    an order that grows bits_ once or several times: the walk visits them in the blocked order
    (floor division for negatives) whatever the growth history."""
    g = np.array(np.meshgrid(EDGES, EDGES, EDGES, indexing="ij"), np.int32).reshape(3, -1).T
    rng = np.random.RandomState(5)
    g = g[rng.permutation(len(g))]
    val = rng.randint(1, 32768, len(g)).astype(np.uint16)
    far = np.array([[-8192, 8191, 3000], [8191, -8192, -8192]], np.int32)
    far_val = np.array([11, 12], np.uint16)
    writes = {"grow_once": [(g, val)],
              "grow_many": [(g, val), (far, far_val)],
              "far_first": [(far[:1], far_val[:1]), (g, val), (far[1:], far_val[1:])]}[history]
    idx, got, bits = R.walk(*writes)
    assert bits == (2 if history == "grow_once" else 8)
    all_idx = np.concatenate([w[0] for w in writes])
    all_val = np.concatenate([w[1] for w in writes])
    order = _blocked_key(all_idx)
    np.testing.assert_array_equal(idx, all_idx[order])
    np.testing.assert_array_equal(got, all_val[order])


def test_walk_skips_zero_values():
    idx = np.array([[0, 0, 0], [1, 0, 0], [200, 0, 0]], np.int32)
    got, val, _ = R.walk((idx, np.array([0, 5, 0], np.uint16)))
    np.testing.assert_array_equal(got, [[1, 0, 0]])
    np.testing.assert_array_equal(val, [5])


# ---- the reference encoders against hand-written bytes ----
def f32(v):
    return struct.pack("<f", v)


def f64(v):
    return struct.pack("<d", v)


def test_hybrid_grid_bytes():
    got = R.hybrid_grid_message(0.5, np.array([[-1, 0, 1], [64, -65, 2]]), np.array([3, 32767]))
    want = (b"\x0d" + f32(0.5) +
            b"\x1a\x03" + b"\x01" + b"\x80\x01" +        # zigzag(-1) = 1, zigzag(64) = 128
            b"\x22\x03" + b"\x00" + b"\x81\x01" +        # zigzag(0) = 0, zigzag(-65) = 129
            b"\x2a\x02" + b"\x02" + b"\x04" +
            b"\x32\x04" + b"\x03" + b"\xff\xff\x01")
    assert got == want


def test_empty_hybrid_grid_is_resolution_only():
    assert R.hybrid_grid_message(0.1, np.zeros((0, 3)), np.zeros(0)) == b"\x0d" + f32(0.1)


def test_probability_grid_bytes():
    """Zero scalars omitted (max.x = 0.0, box coordinates 0), -0.0 written (max.y), an empty
    probability_grid_2d present with length 0, the costs last."""
    cells = np.array([[0, 200]], np.uint16)
    got = R.grid2d_message(cells, 0.05, 0.0, -0.0, known_cells_box=(1, 0, 1, 0))
    limits = b"\x09" + f64(0.05) + b"\x12\x09" + b"\x11" + f64(-0.0) + b"\x1a\x04\x08\x02\x10\x01"
    want = (b"\x0a" + bytes([len(limits)]) + limits +
            b"\x12\x03\x00\xc8\x01" +
            b"\x1a\x04\x08\x01\x18\x01" +
            b"\x22\x00" +
            b"\x35" + f32(np.float32(R.K_MIN_CORRESPONDENCE_COST)) +
            b"\x3d" + f32(np.float32(R.K_MAX_CORRESPONDENCE_COST)))
    assert got == want


def test_fresh_grid_has_no_box_and_tsdf_layout():
    cells = np.zeros((1, 1), np.uint16)
    got = R.grid2d_message(cells, 0.05, 1.0, 2.0, weight_cells=np.array([[0]]),
                           truncation_distance=0.3, max_weight=10.0)
    limits = (b"\x09" + f64(0.05) + b"\x12\x12" + b"\x09" + f64(1.0) + b"\x11" + f64(2.0) +
              b"\x1a\x04\x08\x01\x10\x01")
    tsdf = b"\x0d" + f32(0.3) + b"\x15" + f32(10.0) + b"\x1a\x01\x00"
    want = (b"\x0a" + bytes([len(limits)]) + limits + b"\x12\x01\x00" +
            b"\x2a" + bytes([len(tsdf)]) + tsdf +
            b"\x35" + f32(-np.float32(0.3)) + b"\x3d" + f32(0.3))
    assert got == want


def test_packed_varints_match_protowire():
    v = np.concatenate([[0, 1, 127, 128, 16383, 16384, 32767, 32768 | 1000],
                        np.random.RandomState(0).randint(0, 1 << 16, 500)])
    assert R.packed_varints(v) == b"".join(pw.varint(int(x)) for x in v)


def test_hybrid_grid_message_matches_protowire():
    rng = np.random.RandomState(1)
    idx = rng.randint(-8192, 8192, (300, 3))
    val = rng.randint(1, 32768, 300)
    assert R.hybrid_grid_message(0.1, idx, val) == pw.hybrid_grid(0.1, idx, val)
