"""Test-side references for the point-batch edge tests — TEST INFRASTRUCTURE ONLY.

Written in exact integer, Fraction or float32-scalar arithmetic from the reference's definitions
(sensor/internal/voxel_filter.cc, io/outlier_removing_points_processor.cc,
io/xray_points_processor.cc), sharing no code with tests/voxel_filter_oracle.{cc,py},
tests/outlier_removal_oracle.{cc,py} or tests/xray_oracle.{cc,py}:

* cell_index() / cell_indices(): common::RoundToInt(p / r) narrowed to int, from the exact
  quotient of the two float32 values, with a flag that says whether the float32 division can only
  round to that index; voxel_filter_key(), pack() and column_key() build the keys on top.
* voxel_filter(): VoxelFilter's reservoir sampling over a key sequence, with minstd_rand0 as
  16807^j mod (2^31 - 1) in Python ints and libstdc++'s scaling draw with its rejection; it
  returns the kept indices and the rejection trace.
* adaptive_search(): AdaptivelyVoxelFiltered's loop in float32 scalars over a set of wrapped
  64-bit keys: the final length, the trials and each trial's distinct count.
* outlier_removal(): the three phases of OutlierRemovingPointsProcessor over a dict of
  {hits, rays}, the sample points one float32 operation at a time, the keep test in Fraction.
* xray(): the voxel set, the column sums as sequential float32 additions, the per-pixel voxel
  counts and IntoImage's float and double steps.
* mix() (point_batch.cuh's Mix) and keys_at_slot(), which finds packed keys whose home slot is
  a chosen slot (the last, for chains that wrap) of a 2^k-slot table.
Checked against brute force and the restatements in tests/test_point_batch_refs_cpu.py.
"""
import math
from fractions import Fraction

import numpy as np

F = np.float32
D = np.float64
M64 = (1 << 64) - 1
MODULUS = (1 << 31) - 1          # minstd_rand0: x_{j+1} = 16807 x_j mod (2^31 - 1), x_0 = 1
URNG_RANGE = (1 << 31) - 3       # max() - min() = (2^31 - 2) - 1
CUBE_HALF = 8192
EMPTY_KEY = M64
FLT_MIN = float(np.finfo(np.float32).tiny)
LONG_LIMIT = 1 << 63


# ---------------------------------------------------------------------------------------------
# Cell indices
# ---------------------------------------------------------------------------------------------
def _narrow(v):
    """A 64-bit lround result narrowed to int (two's complement, low 32 bits)."""
    return ((v + (1 << 31)) & 0xffffffff) - (1 << 31)


def _ulp32(a):
    """The float32 ulp at the non-negative Fraction a."""
    if a < Fraction(1, 1 << 126):
        return Fraction(1, 1 << 149)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    return Fraction(2) ** (e - 23)


def cell_index(p, r):
    """(index, decided): RoundToInt(p / r) for float32 p and r, narrowed to int.  lround of a
    value at or beyond 2^63 in magnitude (an overflowed quotient included) is LONG_MIN, whose
    low 32 bits are 0.  decided: the exact quotient is more than one float32 ulp away from every
    half-integer and from 2^63, so the rounded quotient lands on the same index."""
    q = Fraction(float(F(p))) / Fraction(float(F(r)))
    a = abs(q)
    ulp = _ulp32(a)
    dist = abs(a - math.floor(a) - Fraction(1, 2))
    decided = dist > ulp and abs(a - LONG_LIMIT) > ulp
    if a >= LONG_LIMIT:
        return 0, decided
    n = math.floor(a + Fraction(1, 2))
    return _narrow(n if q >= 0 else -n), decided


def cell_indices(p, r):
    """cell_index of every element of the float32 array p (any shape) at float32 r, from the
    float64 quotient, whose error (2^-53 relative) the margins absorb: (int64 indices, decided).
    Only for |p / r| < 2^62; test_point_batch_refs_cpu checks it against cell_index."""
    q = np.asarray(p, F).astype(D) / D(F(r))
    a = np.abs(q)
    assert np.all(a < 2.0 ** 62)
    _, e = np.frexp(np.maximum(a, FLT_MIN))
    ulp = np.ldexp(1.0, e - 24)                            # a in [2^(e-1), 2^e)
    dist = np.abs(a - np.floor(a) - 0.5)
    decided = dist > ulp + 4.0 * a * 2.0 ** -53
    n = np.floor(a + 0.5).astype(np.int64)
    v = np.where(q >= 0, n, -n)
    return ((v + (1 << 31)) & 0xffffffff) - (1 << 31), decided


def voxel_filter_key(ix, iy, iz):
    """GetVoxelCellIndex's key: (x << 42) + (y << 21) + z of the sign-extended 64-bit indices,
    wrapping."""
    return (((ix & M64) << 42) + ((iy & M64) << 21) + (iz & M64)) & M64


def pack(ix, iy, iz):
    """The 42-bit voxel key of point_batch.cuh: 14 bits each of z, y, x offset by 8192."""
    return ((iz + CUBE_HALF) << 28) | ((iy + CUBE_HALF) << 14) | (ix + CUBE_HALF)


def column_key(iy, iz):
    return ((iz + CUBE_HALF) << 14) | (iy + CUBE_HALF)


def in_cube(*v):
    return all(-CUBE_HALF <= a < CUBE_HALF for a in v)


def cloud_keys(points, r):
    """(voxel-filter keys, decided) of a float32 (n, 3) cloud at resolution r."""
    idx, ok = cell_indices(np.asarray(points, F).reshape(-1, 3), r)
    keys = [voxel_filter_key(int(x), int(y), int(z)) for x, y, z in idx]
    return keys, bool(ok.all())


# ---------------------------------------------------------------------------------------------
# VoxelFilter and the adaptive search
# ---------------------------------------------------------------------------------------------
def generator(count):
    """The first `count` outputs of a default-seeded minstd_rand0."""
    out, x = [], 1
    for _ in range(count):
        x = x * 16807 % MODULUS
        out.append(x)
    return out


def uniform_draw(k, raw):
    """uniform_int_distribution<int>(1, k) on the raw outputs `raw` by libstdc++'s scaling:
    (result, outputs used)."""
    scaling = URNG_RANGE // k
    past = k * scaling
    for used, x in enumerate(raw, 1):
        ret = x - 1
        if ret < past:
            return ret // scaling + 1, used
    raise ValueError("every output was rejected")


def voxel_filter(keys):
    """VoxelFilter over the voxel keys of a cloud, in input order: (kept indices, trace), trace
    the (call, rejected draws) of every distribution call that rejected, calls counted from 0."""
    x = 1
    voxels = {}
    trace = []
    call = 0
    for i, key in enumerate(keys):
        v = voxels.get(key)
        if v is None:
            voxels[key] = [1, i]
            continue
        v[0] += 1
        k = v[0]
        scaling = URNG_RANGE // k
        past = k * scaling
        rejected = 0
        while True:
            x = x * 16807 % MODULUS
            if x - 1 < past:
                break
            rejected += 1
        if (x - 1) // scaling + 1 == k:
            v[1] = i
        if rejected:
            trace.append((call, rejected))
        call += 1
    return sorted(v[1] for v in voxels.values()), trace


def single_voxel_rejections(num_calls):
    """The rejection trace of `num_calls` calls in one voxel (call m draws with k = m + 2)."""
    x = 1
    trace = []
    for m in range(num_calls):
        k = m + 2
        past = k * (URNG_RANGE // k)
        rejected = 0
        while True:
            x = x * 16807 % MODULUS
            if x - 1 < past:
                break
            rejected += 1
        if rejected:
            trace.append((m, rejected))
    return trace


def range_filter(points, max_range):
    """FilterByMaxRange's mask: float32 ((x*x + y*y) + z*z) then sqrt, <= max_range."""
    p = np.asarray(points, F).reshape(-1, 3)
    n = np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2])
    return n <= F(max_range)


def adaptive_search(points, max_length, min_num_points, max_range):
    """AdaptivelyVoxelFiltered (voxel_filter.cc:38-75) on the range-filtered cloud, counting
    distinct keys only: {"length" (None: the range-filtered cloud is returned), "trials",
    "halvings" (trials at L / 2^h), "counts" [(length, distinct)], "decided"}."""
    pts = np.asarray(points, F).reshape(-1, 3)[range_filter(points, max_range)]
    L, m = F(max_length), F(min_num_points)
    counts = []
    decided = [True]

    def distinct(length):
        keys, ok = cloud_keys(pts, length)
        decided[0] &= ok
        c = len(set(keys))
        counts.append((length, c))
        return F(c)

    def done(length):
        halvings = sum(1 for length, _ in counts if length < L and (L / length).is_integer())
        return {"length": length, "trials": len(counts), "halvings": halvings,
                "counts": counts, "decided": decided[0]}

    if F(len(pts)) <= m:
        return done(None)
    if distinct(L) >= m:
        return done(L)
    high = L
    low = F(0)
    while high > F(1e-2) * L:
        low = high / F(2)
        if distinct(low) >= m:
            while (high - low) / low > F(1e-1):
                mid = (low + high) / F(2)
                if distinct(mid) >= m:
                    low = mid
                else:
                    high = mid
            return done(low)
        high = high / F(2)
    return done(low)


def adaptive_voxel_filter(points, max_length, min_num_points, max_range):
    """(kept indices into the unfiltered cloud, adaptive_search's result)."""
    s = adaptive_search(points, max_length, min_num_points, max_range)
    index = np.flatnonzero(range_filter(points, max_range))
    if s["length"] is None:
        return index, s
    keys, ok = cloud_keys(np.asarray(points, F).reshape(-1, 3)[index], s["length"])
    s["decided"] &= ok
    kept, _ = voxel_filter(keys)
    return index[kept], s


# ---------------------------------------------------------------------------------------------
# OutlierRemovingPointsProcessor
# ---------------------------------------------------------------------------------------------
def ray_samples(voxel_size, length):
    """The x of `for (float x = 0; x < length; x += voxel_size)`, voxel_size a double:
    x_{k+1} = float32(float64(x_k) + voxel_size)."""
    xs = [F(0)]
    while xs[-1] < F(length):
        nxt = F(D(xs[-1]) + voxel_size)
        if nxt == xs[-1]:
            raise ValueError("x stops growing below the length")
        xs.append(nxt)
    return np.array([x for x in xs if x < F(length)], F)


def ray_lengths(origin, points):
    """Each ray's float32 length sqrt((dx*dx + dy*dy) + dz*dz)."""
    d = np.asarray(points, F).reshape(-1, 3) - np.asarray(origin, F).reshape(1, 3)
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def _voxels_of(points, resolution):
    idx, ok = cell_indices(points, resolution)
    return [tuple(int(v) for v in row) for row in idx], ok


def outlier_removal(batches, voxel_size, miss_per_hit_limit):
    """The three phases over (origin, points) batches: {"hits": {voxel: hits} after phase 1,
    "rays": {voxel: (hits, rays)} after phase 2, "kept": [indices per batch], "decided"}.  Every
    hit must lie in the cube."""
    res = F(voxel_size)
    decided = True
    hits = {}
    for _, pts in batches:
        cells, ok = _voxels_of(np.asarray(pts, F).reshape(-1, 3), res)
        decided &= bool(ok.all())
        for c in cells:
            assert in_cube(*c)
            hits[c] = hits.get(c, 0) + 1
    rays = dict.fromkeys(hits, 0)
    table = ray_samples(voxel_size, max([F(0)] + [ray_lengths(o, p).max()
                                                  for o, p in batches if len(p)]))
    for o, pts in batches:
        o = np.asarray(o, F).reshape(3)
        for p, length in zip(np.asarray(pts, F).reshape(-1, 3), ray_lengths(o, pts)):
            d = p - o
            xs = table[table < length]
            if not len(xs):
                continue
            s = xs / length
            q = o[None, :] + s[:, None] * d[None, :]          # one float32 operation at a time
            cells, ok = _voxels_of(q, res)
            decided &= bool(ok.all())
            for c in cells:
                if hits.get(c, 0) > 0:
                    rays[c] += 1
    limit = Fraction(miss_per_hit_limit)
    kept = []
    for _, pts in batches:
        cells, ok = _voxels_of(np.asarray(pts, F).reshape(-1, 3), res)
        decided &= bool(ok.all())
        kept.append(np.array([i for i, c in enumerate(cells)
                              if rays.get(c, 0) < limit * hits.get(c, 0)], np.int32))
    return {"hits": hits, "rays": {c: (hits[c], rays[c]) for c in hits}, "kept": kept,
            "decided": decided}


def voxel_arrays(table):
    """A {voxel: value} dict as the device's read-back: (indices (n, 3), values...) in
    ascending (z, y, x)."""
    keys = sorted(table, key=lambda c: (c[2], c[1], c[0]))
    idx = np.array(keys, np.int32).reshape(-1, 3)
    vals = [table[c] for c in keys]
    if vals and isinstance(vals[0], tuple):
        return (idx,) + tuple(np.array(v, np.int32) for v in zip(*vals))
    return idx, np.array(vals, np.int32)


# ---------------------------------------------------------------------------------------------
# XRayPointsProcessor (identity transform)
# ---------------------------------------------------------------------------------------------
def to_uint8(c):
    """FloatComponentToUint8: RoundToInt(Clamp(c, 0, 1) * 255) as a byte.  A NaN passes the
    clamp, and lround(NaN) is LONG_MIN, whose low byte is 0."""
    c = F(1) if c > F(1) else (F(0) if c < F(0) else F(c))
    v = float(c * F(255))
    if not abs(v) < 2.0 ** 63:
        return 0
    return int(math.floor(abs(v) + 0.5)) & 0xff


def mix_from_white(b, t):
    """Mix(1.f, b, t) = 1.f * (1. - t) + t * b: a double, a float product, a double sum, a
    float."""
    with np.errstate(invalid="ignore"):
        return F(1.0 * (1.0 - float(t)) + float(F(t) * F(b)))


def xray(batches, voxel_size, saturation_factor=1.0):
    """One aggregation of XRayPointsProcessor under the identity transform over (points,
    colours or None) batches in stream order: {"voxels" set, "columns" {(y, z): [r, g, b, n]},
    "box" (lo, hi), "counts" (h, w) per-pixel voxel counts, "pixels" (h, w) cairo words,
    "decided"}."""
    res = F(voxel_size)
    voxels, columns = set(), {}
    lo = hi = None
    decided = True
    for pts, rgb in batches:
        pts = np.asarray(pts, F).reshape(-1, 3)
        idx, ok = cell_indices(pts, res)
        decided &= bool(ok.all())
        rgb = np.zeros_like(pts) if rgb is None else np.asarray(rgb, F).reshape(-1, 3)
        for (x, y, z), c in zip(idx.tolist(), rgb):
            assert in_cube(x, y, z)
            voxels.add((x, y, z))
            lo = (x, y, z) if lo is None else tuple(min(a, b) for a, b in zip(lo, (x, y, z)))
            hi = (x, y, z) if hi is None else tuple(max(a, b) for a, b in zip(hi, (x, y, z)))
            col = columns.setdefault((y, z), [F(0), F(0), F(0), 0])
            col[0] = F(col[0] + c[0])
            col[1] = F(col[1] + c[1])
            col[2] = F(col[2] + c[2])
            col[3] += 1
    out = {"voxels": voxels, "columns": columns, "box": (lo, hi), "decided": decided}
    if lo is None:
        return out
    w, h = hi[1] - lo[1] + 1, hi[2] - lo[2] + 1
    counts = np.zeros((h, w), np.int64)
    for _, y, z in voxels:
        counts[hi[2] - z, hi[1] - y] += 1
    top = F(FLT_MIN)
    for n in np.unique(counts[counts > 0]):
        top = max(top, F(math.log(int(n))))
    pixels = np.full((h, w), 0xffffffff, np.uint32)
    for r, c in zip(*np.nonzero(counts)):
        n = int(counts[r, c])
        with np.errstate(over="ignore"):
            s = F(min(F(1.0), F(math.log(n) / float(top) * saturation_factor)))
        col = columns[(hi[1] - c, hi[2] - r)]
        cnt = F(col[3])
        rgb = [to_uint8(mix_from_white(F(col[a] / cnt), s)) for a in range(3)]
        pixels[r, c] = 0xff000000 | rgb[0] << 16 | rgb[1] << 8 | rgb[2]
    out.update(counts=counts, pixels=pixels)
    return out


# ---------------------------------------------------------------------------------------------
# Hash helpers
# ---------------------------------------------------------------------------------------------
def mix(k):
    """point_batch.cuh's Mix, the fmix64 finaliser, in Python ints."""
    k &= M64
    k ^= k >> 33
    k = (k * 0xff51afd7ed558ccd) & M64
    k ^= k >> 33
    k = (k * 0xc4ceb9fe1a85ec53) & M64
    return k ^ (k >> 33)


def mix_array(keys):
    """mix over a uint64 array (numpy's uint64 products wrap mod 2^64)."""
    k = np.asarray(keys, np.uint64).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xff51afd7ed558ccd)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xc4ceb9fe1a85ec53)
        k ^= k >> np.uint64(33)
    return k


def keys_at_slot(candidates, slots, slot=None, count=1):
    """The first `count` of the candidate keys (in order) whose home slot Mix(key) & (slots - 1)
    is `slot` (default: the last slot)."""
    assert slots & (slots - 1) == 0
    slot = slots - 1 if slot is None else slot
    cand = np.asarray(candidates, np.uint64)
    hit = cand[(mix_array(cand) & np.uint64(slots - 1)) == np.uint64(slot)]
    assert len(hit) >= count, "too few candidates"
    return [int(k) for k in hit[:count]]


def table_slots(current, entries, initial=1 << 12):
    """The slot count a table grows to so that `entries` keep it at most half full."""
    slots = max(current, initial)
    while 2 * entries > slots:
        slots *= 2
    return slots


def probe_chain(keys, slots):
    """The slots that inserting `keys` in order into an empty linear-probing table takes."""
    table = {}
    out = []
    for k in keys:
        h = mix(k) & (slots - 1)
        while h in table and table[h] != k:
            h = (h + 1) & (slots - 1)
        table[h] = k
        out.append(h)
    return out
