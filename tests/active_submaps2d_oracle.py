"""ActiveSubmaps2D (mapping/2d/submap_2d.cc:153-236) restated over the CPU ProbabilityGrid and
inserter of tests/insert2d_oracle.py: the parity reference of the device lifecycle.  Each
InsertRangeData returns what happened to the submaps, so that tests can check the schedule
without grids; `grids=False` runs the schedule alone."""
import numpy as np

from tests import insert2d_oracle as O

SUBPIXEL_SCALE = 1000


class Submap:
    def __init__(self, index, origin, resolution, grids):
        o = np.asarray(origin, np.float32).reshape(-1)
        self.index = index
        self.local_pose = (float(o[0]), float(o[1]), 0.0, 1.0, 0.0, 0.0, 0.0)
        self.grid = O.Grid.create_grid(o[:2], resolution) if grids else None
        self.num_range_data = 0
        self.insertion_finished = False

    def finish(self):
        """Submap2D::Finish: grid_ = grid_->ComputeCroppedGrid()."""
        if self.grid is not None:
            self.grid = self.grid.crop()
        self.insertion_finished = True


class ActiveSubmaps:
    def __init__(self, num_range_data, resolution=0.05, hit_probability=0.55,
                 miss_probability=0.49, insert_free_space=True, grids=True):
        assert num_range_data > 0
        self.num_range_data = num_range_data
        self.resolution = resolution
        self.inserter = (O.Inserter(hit_probability, miss_probability, insert_free_space)
                         if grids else None)
        self.submaps = []
        self._created = 0

    def insert_range_data(self, origin, returns=None, misses=None):
        """One scan; returns {"created": i or None, "evicted": i or None, "finished": i or None,
        "inserted": [i, ...]} with the submaps' creation indices."""
        event = {"created": None, "evicted": None, "finished": None, "inserted": []}
        o = np.asarray(origin, np.float32).reshape(-1)
        if not self.submaps or self.submaps[-1].num_range_data == self.num_range_data:
            if len(self.submaps) >= 2:
                assert self.submaps[0].insertion_finished
                event["evicted"] = self.submaps.pop(0).index
            self.submaps.append(Submap(self._created, o[:2], self.resolution,
                                       self.inserter is not None))
            event["created"] = self._created
            self._created += 1
        org = np.zeros(3, np.float32)
        org[:min(3, len(o))] = o[:3]
        ret = np.zeros((0, 3), np.float32) if returns is None else returns
        for s in self.submaps:
            assert not s.insertion_finished
            if self.inserter is not None:
                self.inserter.insert(org, ret, s.grid, misses)
            s.num_range_data += 1
            event["inserted"].append(s.index)
        if self.submaps[0].num_range_data == 2 * self.num_range_data:
            self.submaps[0].finish()
            event["finished"] = self.submaps[0].index
        return event


def superscaled_index(limits, px, py):
    """The superscaled cell (x, y) of a float point under MapLimits (resolution, max_x, max_y):
    GetCellIndex at resolution / kSubpixelScale, llround half away from zero."""
    res, max_x, max_y = limits[:3]
    s = res / SUBPIXEL_SCALE

    def llround(v):
        return int(np.floor(abs(v) + 0.5)) * (1 if v >= 0 else -1)

    return (llround((max_y - float(np.float32(py))) / s - 0.5),
            llround((max_x - float(np.float32(px))) / s - 0.5))


def slot_reservation(origin, points, resolution):
    """The slots csm_range_inserter2d_insert_submaps reserves for the rays from origin to
    `points` at `resolution` (insert2d.cu, SlotReservation)."""
    o = np.asarray(origin, np.float32).astype(np.float64)
    l1 = 0.0
    for p in np.asarray(points, np.float32).reshape(-1, 3).astype(np.float64):
        l1 += abs(p[0] - o[0]) + abs(p[1] - o[1])
    bound = l1 / resolution * (1.0 + 1e-9) + 3.0 * len(points) + 1.0
    return min(int(bound), 2 ** 31 - 1)
