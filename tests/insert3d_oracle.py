"""CPU restatement of RangeDataInserter3D — TEST INFRASTRUCTURE ONLY.

What is restated (the device inserter, csrc/insert3d.cu, is checked against this, never the
reverse):
  * ComputeLookupTableToApplyOdds (mapping/probability_values.cc:76-87) over
    kValueToProbability (:29-37), BoundedFloatToValue / Odds / ProbabilityFromOdds
    (probability_values.h:32-52), all in float32 as the reference evaluates them;
  * HybridGrid::ApplyLookupTable / FinishUpdate (mapping/3d/hybrid_grid.h:492-518): within one
    insert the first application to a cell sets kUpdateMarker and later ones are ignored; a
    value that already carries the marker is left alone;
  * RangeDataInserter3D::Insert (mapping/3d/range_data_inserter_3d.cc:27-68, 87-114): the hits
    in return order, then per return the last num_free_space_voxels samples
    origin_cell + delta * position / num_samples (C++ truncating division), then the
    intensities of returns not brighter than intensity_threshold;
  * IntensityHybridGrid::AddIntensity / GetIntensity (hybrid_grid.h:552-570): float32 sum in
    return order, int count, float32 mean.
The operation sequence of an insert is built in the reference's order and "first application
wins" is taken from it; the float32 sums are added one return at a time per voxel.
"""
import numpy as np

F = np.float32
K_UPDATE_MARKER = 1 << 15
K_MIN_PROBABILITY = F(0.1)
K_MAX_PROBABILITY = F(F(1) - K_MIN_PROBABILITY)
CUBE = 8192   # voxel indices lie in [-CUBE, CUBE) (hybrid_grid.h:387)


def lround(v):
    """std::lround (halves away from zero), elementwise."""
    v = np.asarray(v, np.float64)
    t = np.trunc(v)
    return (t + np.where(np.abs(v - t) >= 0.5, np.sign(v), 0.0)).astype(np.int64)


def odds(p):
    p = F(p) if np.ndim(p) == 0 else np.asarray(p, F)
    return p / (F(1) - p)


def probability_from_odds(o):
    return o / (o + F(1))


def probability_to_value(p):
    """BoundedFloatToValue(p, kMinProbability, kMaxProbability)."""
    c = np.clip(np.asarray(p, F), K_MIN_PROBABILITY, K_MAX_PROBABILITY).astype(F)
    scale = F(F(32766) / (K_MAX_PROBABILITY - K_MIN_PROBABILITY))
    return (lround((c - K_MIN_PROBABILITY) * scale) + 1).astype(np.int64)


def value_to_probability(v):
    """kValueToProbability (probability_values.cc:29-37), bit 15 masked."""
    v = np.asarray(v, np.int64) & 0x7fff
    scale = F((K_MAX_PROBABILITY - K_MIN_PROBABILITY) / F(32766))
    p = v.astype(F) * scale + F(K_MIN_PROBABILITY - scale)
    return np.where(v == 0, K_MIN_PROBABILITY, p).astype(F)


def lookup_table(o):
    """ComputeLookupTableToApplyOdds(odds): 32768 uint16 entries with the marker set."""
    o = F(o)
    cells = np.arange(32768)
    p = np.where(cells == 0, probability_from_odds(o),
                 probability_from_odds(o * odds(value_to_probability(cells))))
    return (probability_to_value(p) + K_UPDATE_MARKER).astype(np.uint16)


def cell_index(resolution, points):
    """HybridGridBase::GetCellIndex (hybrid_grid.h:428-433) of float32 points, n x 3."""
    return lround(np.asarray(points, F).reshape(-1, 3) / F(resolution))


def pack(cells):
    c = np.asarray(cells, np.int64).reshape(-1, 3) + CUBE
    return (c[:, 0] << 28) | (c[:, 1] << 14) | c[:, 2]


def unpack(keys):
    k = np.asarray(keys, np.int64)
    return np.stack([(k >> 28) & 0x3fff, (k >> 14) & 0x3fff, k & 0x3fff], 1) - CUBE


def _in_cube(cells):
    return bool(np.all((cells >= -CUBE) & (cells < CUBE)))


class _SparseGrid:
    """Voxels as sorted packed keys with per-voxel columns (0 for voxels never stored)."""

    def __init__(self, resolution, indices, columns):
        self.resolution = float(F(resolution))
        idx = np.asarray(indices, np.int64).reshape(-1, 3)
        keys = pack(idx)
        order = np.argsort(keys, kind="stable")
        self.keys = keys[order]
        self.cols = [np.asarray(c).reshape(-1)[order].copy() for c in columns]

    def _get(self, keys):
        pos = np.searchsorted(self.keys, keys)
        hit = pos < len(self.keys)
        hit[hit] = self.keys[pos[hit]] == keys[hit]
        return pos, hit

    def _put(self, keys, values):
        """keys unique; values one array per column."""
        pos, hit = self._get(keys)
        for c, v in zip(self.cols, values):
            c[pos[hit]] = v[hit]
        if (~hit).any():
            allk = np.concatenate([self.keys, keys[~hit]])
            order = np.argsort(allk, kind="stable")
            self.keys = allk[order]
            self.cols = [np.concatenate([c, v[~hit].astype(c.dtype)])[order]
                         for c, v in zip(self.cols, values)]

    def indices(self):
        return unpack(self.keys).astype(np.int32)

    def dense(self, lo, dims, col=0):
        """The column over box lo .. lo + dims, indexed [z, y, x]."""
        out = np.zeros(tuple(int(d) for d in dims[::-1]), self.cols[col].dtype)
        idx = unpack(self.keys) - np.asarray(lo, np.int64)
        inside = np.all((idx >= 0) & (idx < np.asarray(dims, np.int64)), 1)
        i = idx[inside]
        out[i[:, 2], i[:, 1], i[:, 0]] = self.cols[col][inside]
        return out


class HybridGrid(_SparseGrid):
    """HybridGrid of uint16 probability values, from the flat form (indices, values)."""

    def __init__(self, resolution, indices=(), values=()):
        super().__init__(resolution, indices, [np.asarray(values, np.uint16)])

    @property
    def values(self):
        return self.cols[0]

    def value(self, cells):
        keys = pack(cells)
        pos, hit = self._get(keys)
        out = np.zeros(len(keys), np.uint16)
        out[hit] = self.cols[0][pos[hit]]
        return out

    def get_probability(self, cells):
        return value_to_probability(self.value(cells))


class IntensityHybridGrid(_SparseGrid):
    """IntensityHybridGrid from the flat form (indices, sums, counts)."""

    def __init__(self, resolution, indices=(), sums=(), counts=()):
        super().__init__(resolution, indices,
                         [np.asarray(sums, F), np.asarray(counts, np.int32)])

    @property
    def sums(self):
        return self.cols[0]

    @property
    def counts(self):
        return self.cols[1]

    def means(self):
        c = self.cols[1]
        return np.where(c == 0, F(0), self.cols[0] / np.maximum(c, 1).astype(F)).astype(F)

    def get_intensity(self, cells):
        keys = pack(cells)
        pos, hit = self._get(keys)
        out = np.zeros(len(keys), F)
        out[hit] = self.means()[pos[hit]]
        return out

    def dense_mean(self, lo, dims):
        saved = self.cols
        self.cols = [self.means()]
        try:
            return self.dense(lo, dims)
        finally:
            self.cols = saved


class RangeDataInserter3D:
    def __init__(self, hit_probability, miss_probability, num_free_space_voxels,
                 intensity_threshold):
        if not hit_probability > 0.5 or not miss_probability < 0.5:
            raise ValueError("RangeDataInserter3D: CHECK_GT(hit, 0.5) / CHECK_LT(miss, 0.5)")
        self.num_free_space_voxels = int(num_free_space_voxels)
        self.intensity_threshold = F(intensity_threshold)
        self.hit_table = lookup_table(odds(F(hit_probability)))
        self.miss_table = lookup_table(odds(F(miss_probability)))

    def miss_cells(self, origin_cell, hit_cells):
        """InsertMissesIntoGrid's sample cells in the reference's order (return, position)."""
        delta = hit_cells - origin_cell
        ns = np.abs(delta).max(1) if len(delta) else np.zeros(0, np.int64)
        if (ns >= 1 << 15).any():
            raise ValueError("num_samples >= 1 << 15")
        per = min(self.num_free_space_voxels, int(ns.max()) if len(ns) else 0)
        if per == 0:
            return np.zeros((0, 3), np.int64)
        k = np.arange(per)
        pos = np.maximum(0, ns - self.num_free_space_voxels)[:, None] + k[None, :]
        valid = pos < ns[:, None]
        r = np.broadcast_to(np.arange(len(ns))[:, None], pos.shape)[valid]
        p = pos[valid][:, None]
        a = delta[r] * p
        q = np.sign(a) * (np.abs(a) // ns[r][:, None])   # truncating division
        return origin_cell + q

    def insert(self, origin, returns, intensities, grid, intensity_grid=None):
        returns = np.asarray(returns, F).reshape(-1, 3)
        origin_cell = cell_index(grid.resolution, origin)[0]
        hits = cell_index(grid.resolution, returns)
        if not _in_cube(origin_cell) or not _in_cube(hits):
            raise ValueError("cell outside the 2^14 cube")
        misses = self.miss_cells(origin_cell, hits)
        kept = None
        if intensity_grid is not None and intensities is not None:
            inten = np.asarray(intensities, F).reshape(-1)
            kept = ~(inten > self.intensity_threshold)
            icells = cell_index(intensity_grid.resolution, returns[kept])
            if not _in_cube(icells):
                raise ValueError("intensity cell outside the 2^14 cube")
        # ApplyLookupTable in the reference's order: the first application to a cell wins
        seq = np.concatenate([pack(hits), pack(misses)])
        keys, first = np.unique(seq, return_index=True)
        old = grid.value(unpack(keys))
        fresh = old < K_UPDATE_MARKER
        table = np.where(first < len(hits), 0, 1)
        new = np.where(table == 0, self.hit_table[old & 0x7fff], self.miss_table[old & 0x7fff])
        # FinishUpdate clears the markers it set
        new = np.where(fresh, new - K_UPDATE_MARKER, old).astype(np.uint16)
        grid._put(keys, [new])
        if kept is not None:
            self._add_intensities(intensity_grid, icells, inten[kept])

    @staticmethod
    def _add_intensities(ig, cells, values):
        """AddIntensity per return, in return order: the j-th return of each voxel is added in
        round j, so each voxel's float32 sum sees its returns one at a time, in order."""
        if len(values) == 0:
            return
        keys = pack(cells)
        order = np.argsort(keys, kind="stable")
        k, v = keys[order], values[order]
        uk, start, cnt = np.unique(k, return_index=True, return_counts=True)
        pos, hit = ig._get(uk)
        s = np.zeros(len(uk), F)
        c = np.zeros(len(uk), np.int32)
        s[hit] = ig.cols[0][pos[hit]]
        c[hit] = ig.cols[1][pos[hit]]
        for j in range(int(cnt.max())):
            live = cnt > j
            s[live] = s[live] + v[start[live] + j]
            c[live] += 1
        ig._put(uk, [s, c])
