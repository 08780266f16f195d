"""The reference's OverlappingSubmapsTrimmer2D test cases (overlapping_submaps_trimmer_2d_test.cc)
as a fake pose graph, the duck-typed Trimmable that cartographer_b200.pose_graph's trimmer reads.
Each submap's grid is the serialised proto::Grid2D that the test's AddSquareSubmap writes
(num_cells x num_cells cells of value 1, resolution 1, max = the submap corner, the whole grid as
known-cells box, probability_grid_2d {}), decoded back as Grid2D(const proto::Grid2D&) reads it:
cells and limits by the library's host-only csm_grid2d_proto_decode, the known-cells box from the
message.  `make_grid(HostGrid)` turns the decoded grid into what the trimmer under test reads
(the host grid itself for the CPU restatement, a RealTimeGrid2D for the device)."""
import ctypes as C
import math
from dataclasses import dataclass, field

import numpy as np

from cartographer_b200 import pose_graph as P
from tests import protowire as pw
from tests import trimmer2d_oracle as O


@dataclass
class HostGrid:
    cells: np.ndarray               # [y, x], 0 = unknown
    known_box: tuple                # (min_x, min_y, max_x, max_y) or None
    limits: tuple                   # (max_x, max_y, resolution)


@dataclass
class Submap:
    grid: object
    local_pose: list
    insertion_finished: bool


@dataclass
class SubmapData:
    submap: Submap
    pose: list


@dataclass
class Node:
    time: int


@dataclass
class Constraint:
    submap_id: tuple
    node_id: tuple
    tag: str


@dataclass
class FakePoseGraph:
    submap_data: dict = field(default_factory=dict)
    nodes: dict = field(default_factory=dict)
    constraints: list = field(default_factory=list)
    trimmed: list = field(default_factory=list)

    def GetOptimizedSubmapData(self):
        return dict(self.submap_data)

    def GetTrajectoryNodes(self):
        return self.nodes

    def GetConstraints(self):
        return self.constraints

    def TrimSubmap(self, submap_id):
        self.trimmed.append(submap_id)


def embed3d(x, y, theta):
    """transform::Embed3D(Rigid2d({x, y}, theta)): (tx, ty, tz, qw, qx, qy, qz)."""
    return [x, y, 0.0, math.cos(theta / 2), 0.0, 0.0, math.sin(theta / 2)]


class OracleTrimmer(P.OverlappingSubmapsTrimmer2D):
    """The Python trimmer with the CPU restatement as its coverage pass over HostGrids."""

    def _limits(self, grid):
        return grid.limits

    def _coverage(self, records, first_limits, fresh, min_cells):
        subs = [(g.cells, g.known_box, g.limits, pose, t) for g, pose, t in records]
        return O.trim(subs, first_limits, fresh, min_cells)


def square_grid2d_message(num_cells, corner):
    """The proto::Grid2D of AddSquareSubmap (overlapping_submaps_trimmer_2d_test.cc:42-68): proto3
    omits the zero scalars (min_x, min_y, and max_x, max_y of a 1 x 1 box)."""
    def nonzero(field_number, v):
        return pw.f_varint(field_number, v) if v else b""
    limits = (pw.f_double(1, 1.0) +
              pw.f_bytes(2, pw.f_double(1, corner[0]) + pw.f_double(2, corner[1])) +
              pw.f_bytes(3, pw.f_varint(1, num_cells) + pw.f_varint(2, num_cells)))
    cells = pw.f_bytes(2, b"".join(pw.varint(1) for _ in range(num_cells * num_cells)))
    box = pw.f_bytes(3, nonzero(1, num_cells - 1) + nonzero(2, num_cells - 1))
    return pw.f_bytes(1, limits) + cells + box + pw.f_bytes(4, b"")


def _fields(msg):
    """(field number, value) of a message's fields: ints for varints, bytes otherwise."""
    i = 0
    while i < len(msg):
        key, i = _varint(msg, i)
        number, wire = key >> 3, key & 7
        if wire == 0:
            v, i = _varint(msg, i)
        elif wire == 1:
            v, i = msg[i:i + 8], i + 8
        elif wire == 5:
            v, i = msg[i:i + 4], i + 4
        else:
            n, i = _varint(msg, i)
            v, i = msg[i:i + n], i + n
        yield number, v


def _varint(msg, i):
    v = shift = 0
    while True:
        b = msg[i]
        i += 1
        v |= (b & 0x7F) << shift
        shift += 7
        if b < 0x80:
            return v, i


class _Info(C.Structure):
    _fields_ = [("num_x_cells", C.c_int32), ("num_y_cells", C.c_int32),
                ("resolution", C.c_double), ("max_x", C.c_double), ("max_y", C.c_double),
                ("min_correspondence_cost", C.c_float), ("max_correspondence_cost", C.c_float),
                ("is_tsdf", C.c_int32), ("reserved", C.c_int32)]


def decode_grid2d(msg):
    """A HostGrid from a serialised proto::Grid2D: cells and limits through the library's
    csm_grid2d_proto_decode, the known-cells box (grid_2d.cc:84-89: max_x, max_y, min_x, min_y;
    empty when the field is absent) from the message."""
    from cartographer_b200._lib import lib
    buf = (C.c_uint8 * len(msg)).from_buffer_copy(msg)
    info = _Info()
    assert lib().csm_grid2d_proto_decode(buf, C.c_int64(len(msg)), C.byref(info), None, 0) == 0
    cells = np.zeros((info.num_y_cells, info.num_x_cells), np.uint16)
    assert lib().csm_grid2d_proto_decode(buf, C.c_int64(len(msg)), C.byref(info),
                                         cells.ctypes.data_as(C.POINTER(C.c_uint16)),
                                         C.c_int64(cells.size)) == 0
    box = None
    for number, v in _fields(msg):
        if number == 3:
            b = dict(_fields(v))
            box = (b.get(3, 0), b.get(4, 0), b.get(1, 0), b.get(2, 0))
    return HostGrid(cells, box, (info.max_x, info.max_y, info.resolution))


class Builder:
    def __init__(self, make_grid):
        self.pg = FakePoseGraph()
        self.make_grid = make_grid

    def square(self, global_pose, local_pose, corner, index, num_cells, finished):
        grid = decode_grid2d(square_grid2d_message(num_cells, corner))
        self.pg.submap_data[(0, index)] = SubmapData(
            Submap(self.make_grid(grid), embed3d(*local_pose), finished), embed3d(*global_pose))

    def node(self, index, timestamp):
        self.pg.nodes[(0, index)] = Node(timestamp)

    def constraint(self, submap_index, node_index, intra):
        self.pg.constraints.append(Constraint((0, submap_index), (0, node_index),
                                              P.INTRA_SUBMAP if intra else P.INTER_SUBMAP))


IDENTITY = (0.0, 0.0, 0.0)


def _two_overlapping(b, finished0=True):
    b.square(IDENTITY, IDENTITY, (1.0, 1.0), 0, 1, finished0)
    b.square(IDENTITY, IDENTITY, (1.0, 1.0), 1, 1, True)
    b.node(0, 1000)
    b.node(1, 2000)
    b.constraint(0, 0, True)
    b.constraint(1, 1, True)


def empty_pose_graph(b, trimmer_cls):
    t = trimmer_cls(1, 0, 0)
    t.Trim(b.pg)
    assert b.pg.trimmed == []


def trim_one_of_two_overlapping_submaps(b, trimmer_cls):
    _two_overlapping(b)
    t = trimmer_cls(1, 0, 0)
    t.Trim(b.pg)
    assert b.pg.trimmed == [(0, 0)]


def min_added_submaps_count_param(b, trimmer_cls):
    _two_overlapping(b)
    t = trimmer_cls(1, 0, 2)
    t.Trim(b.pg)
    assert b.pg.trimmed == []
    b.square(IDENTITY, IDENTITY, (1.0, 1.0), 2, 1, True)
    b.node(2, 3000)
    b.constraint(2, 2, True)
    t.Trim(b.pg)
    assert b.pg.trimmed == [(0, 0), (0, 1)]


def do_not_trim_unfinished_submap(b, trimmer_cls):
    _two_overlapping(b, finished0=False)
    t = trimmer_cls(1, 0, 0)
    t.Trim(b.pg)
    assert b.pg.trimmed == []


def use_only_intra_submaps_to_compute_freshness(b, trimmer_cls):
    b.square(IDENTITY, IDENTITY, (1.0, 1.0), 0, 1, True)
    b.square(IDENTITY, IDENTITY, (1.0, 1.0), 1, 1, True)
    b.node(0, 1000)
    b.node(1, 2000)
    b.node(2, 3000)
    b.constraint(0, 0, False)
    b.constraint(0, 2, True)
    b.constraint(1, 1, True)
    t = trimmer_cls(1, 0, 0)
    t.Trim(b.pg)
    assert b.pg.trimmed == [(0, 1)]


def trim_submap_with_low_covered_cells_count(b, trimmer_cls):
    b.square(IDENTITY, IDENTITY, (1.0, 1.0), 0, 2, True)
    b.square((1.0, 1.0, 0.0), IDENTITY, (1.0, 1.0), 1, 2, True)
    b.node(0, 1000)
    b.node(1, 2000)
    b.constraint(0, 0, True)
    b.constraint(1, 1, True)
    t = trimmer_cls(1, 4, 0)
    t.Trim(b.pg)
    assert b.pg.trimmed == [(0, 0)]


def transformations(b, trimmer_cls):
    b.square(IDENTITY, IDENTITY, (1.0, 1.0), 0, 1, True)
    transform = (1.0, 1.0, math.pi / 2)
    b.square(transform, transform, (1.0, 1.0), 1, 1, True)
    b.node(0, 1000)
    b.node(1, 2000)
    b.constraint(0, 0, True)
    b.constraint(1, 1, True)
    t = trimmer_cls(1, 0, 0)
    t.Trim(b.pg)
    assert b.pg.trimmed == [(0, 0)]


REFERENCE_CASES = {
    "EmptyPoseGraph": empty_pose_graph,
    "TrimOneOfTwoOverlappingSubmaps": trim_one_of_two_overlapping_submaps,
    "TestMinAddedSubmapsCountParam": min_added_submaps_count_param,
    "DoNotTrimUnfinishedSubmap": do_not_trim_unfinished_submap,
    "UseOnlyIntraSubmapsToComputeFreshness": use_only_intra_submaps_to_compute_freshness,
    "TrimSubmapWithLowCoveredCellsCount": trim_submap_with_low_covered_cells_count,
    "TestTransformations": transformations,
}
