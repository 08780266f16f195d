"""The point-batch references (tests/point_batch_refs.py) checked without a GPU: against brute
force, against the CPU restatements of the three processors, and, for the hash and the rounding,
against point_batch.cuh itself compiled for the host."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import outlier_removal_oracle as ORO
from tests import point_batch_refs as R
from tests import voxel_filter_oracle as VFO
from tests import xray_oracle as XO

F = np.float32
HEADER_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                          "cartographer_b200", "csrc")

# point_batch.cuh on the host: the CUDA qualifiers defined away, atomicCAS a plain
# compare-and-swap (one thread), the launch built-ins stubbed for k_rehash's template.
HOST_SRC = r"""
#include <cmath>
#include <cstdint>
#define __host__
#define __device__
#define __global__
struct Dim3Stub { unsigned x, y, z; };
static Dim3Stub blockIdx, blockDim, threadIdx;
static unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp,
                                    unsigned long long v) {
  const unsigned long long old = *p;
  if (old == cmp) *p = v;
  return old;
}
#include "point_batch.cuh"
extern "C" {
uint64_t pb_mix(uint64_t k) { return csm::Mix(k); }
int pb_round_to_int(float p, float r) { return csm::RoundToInt(p / r); }
long long pb_insert(unsigned long long* keys, unsigned long long mask, unsigned long long key,
                    int* inserted) {
  bool ins;
  const unsigned long long h = csm::Insert(keys, mask, key, &ins);
  *inserted = ins;
  return static_cast<long long>(h);
}
long long pb_find(const unsigned long long* keys, unsigned long long mask,
                  unsigned long long key) {
  return csm::Find(keys, mask, key);
}
unsigned long long pb_pack(int x, int y, int z) { return csm::Pack(x, y, z); }
}
"""


@pytest.fixture(scope="module")
def H():
    d = tempfile.mkdtemp(prefix="point_batch_host_")
    try:
        src = os.path.join(d, "point_batch_host.cc")
        with open(src, "w") as f:
            f.write(HOST_SRC)
        so = os.path.join(d, "libpoint_batch_host.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC",
                               "-shared", "-I", HEADER_DIR, src, "-o", so])
        L = C.CDLL(so)
    finally:
        shutil.rmtree(d, True)
    L.pb_mix.restype = C.c_uint64
    L.pb_mix.argtypes = [C.c_uint64]
    L.pb_round_to_int.argtypes = [C.c_float, C.c_float]
    L.pb_insert.restype = C.c_longlong
    L.pb_insert.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
    L.pb_find.restype = C.c_longlong
    L.pb_find.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    L.pb_pack.restype = C.c_uint64
    L.pb_pack.argtypes = [C.c_int] * 3
    return L


def _brute_round(p, r):
    """RoundToInt(float32(p / r)) from numpy's float32 division."""
    q = F(p) / F(r)
    a = np.floor(np.float64(abs(q)) + 0.5)
    if not a < 2.0 ** 63:
        return 0
    v = int(a) if q >= 0 else -int(a)
    return ((v + (1 << 31)) & 0xffffffff) - (1 << 31)


def _cell_cases():
    rng = np.random.RandomState(3)
    p = (rng.uniform(-1, 1, 3000) * 10.0 ** rng.uniform(-3, 5, 3000)).astype(F)
    r = (10.0 ** rng.uniform(-3, 1, 3000)).astype(F)
    hand = [(0.5, 1.0), (-0.5, 1.0), (1.5, 1.0), (-2.5, 1.0), (np.nextafter(F(0.5), F(0)), 1.0),
            (np.nextafter(F(0.5), F(1)), 1.0), (0.15, 0.1), (-0.15, 0.1), (0.3, 0.1),
            (2.0 ** 31, 1.0), (-(2.0 ** 31) - 256, 1.0), (2.0 ** 34 + 2048, 0.25), (1e30, 0.01),
            (-3e9, 1.0), (1e19, 1.0), (0.0, 0.3), (-0.0, 0.3), (3.0, 1e-3), (-1.0, 1.0)]
    return list(zip(p, r)) + [(F(a), F(b)) for a, b in hand]


def test_cell_index_against_float32_division_and_the_header(H):
    undecided = 0
    for p, r in _cell_cases():
        v, ok = R.cell_index(p, r)
        if ok:
            assert v == _brute_round(p, r), (p, r)
            assert v == H.pb_round_to_int(p, r), (p, r)
        else:
            undecided += 1
    assert undecided < len(_cell_cases()) // 10
    # exact half-integers and huge quotients are never decided; one ulp off a half is decided
    assert not R.cell_index(0.5, 1.0)[1] and not R.cell_index(1e30, 0.01)[1]
    assert R.cell_index(np.nextafter(F(0.5), F(0)), 1.0) == (0, False)
    assert R.cell_index(0.25, 1.0) == (0, True) and R.cell_index(-0.75, 1.0) == (-1, True)
    assert R.cell_index(2.0 ** 31, 1.0) == (-(2 ** 31), False)     # 2^31 narrows to INT_MIN


def test_vectorised_cell_indices_agree_with_the_exact_ones():
    cases = [(p, r) for p, r in _cell_cases() if abs(float(p) / float(r)) < 2.0 ** 62]
    for p, r in cases:
        (v,), (ok,) = R.cell_indices(np.array([p], F), r)
        e, eok = R.cell_index(p, r)
        assert not ok or eok, (p, r)               # the float64 margin only gives up more
        if ok:
            assert v == e


def test_keys_against_the_restatements():
    rng = np.random.RandomState(5)
    pts = (rng.uniform(-1, 1, (400, 3)) * 10.0 ** rng.uniform(-2, 8, (400, 1))).astype(F)
    pts = np.vstack([pts, F([[0, 0, -1], [0, 0, -0.8], [3, -1, 2.0 ** 21], [0, -1, 2.0 ** 21 - 1]])])
    for r in (F(1.0), F(0.1), F(0.37)):
        keys, _ = R.cloud_keys(pts, r)
        idx, ok = R.cell_indices(pts, r)
        for p, k, d in zip(pts, keys, ok.all(1)):
            if d:
                assert k == VFO.key(*[float(v) for v in p], float(r))
        for p, i, d in zip(pts, idx, ok.all(1)):
            if d:
                assert tuple(i) == ORO.cell_index(p, float(r))
    # (0, 0, -L) and (0, -1, 2^21 - 1) both wrap to the empty-slot key
    assert R.voxel_filter_key(0, 0, -1) == R.EMPTY_KEY
    assert R.voxel_filter_key(0, -1, (1 << 21) - 1) == R.EMPTY_KEY
    assert VFO.key(0.0, 0.0, -1.0, 1.0) == R.EMPTY_KEY


def test_generator_and_uniform_draw():
    np.testing.assert_array_equal(np.array(R.generator(5000), np.uint32), VFO.generator(5000))
    rng = np.random.RandomState(2)
    for k in [2, 3, 7, 1000, 65537, 2 ** 20 + 3, 2 ** 30 + 1, 2 ** 31 - 3]:
        past = k * (R.URNG_RANGE // k)
        for raw in ([past + 1, past, 5], [past, 1], [2 ** 31 - 2] * 2 + [past],
                    list(rng.randint(1, 2 ** 31 - 1, 3))):
            raw = [min(int(v), 2 ** 31 - 2) for v in raw]
            if all(v - 1 >= past for v in raw):
                continue
            assert R.uniform_draw(k, raw) == VFO.uniform(k, np.array(raw, np.uint32)), (k, raw)


def test_voxel_filter_against_the_restatement():
    rng = np.random.RandomState(4)
    for seed in range(12):
        n = int(rng.randint(1, 3000))
        pts = rng.uniform(-2, 2, (n, 3)).astype(F)
        res = float(F(10 ** rng.uniform(-1.5, 0.5)))
        keys, ok = R.cloud_keys(pts, res)
        assert ok
        kept, trace = R.voxel_filter(keys)
        want, st = VFO.voxel_filter(pts, res)
        np.testing.assert_array_equal(kept, want)
        assert sum(r for _, r in trace) == st["rejections"]
    assert R.voxel_filter([]) == ([], [])


def test_rejection_trace_prefixes_of_one_voxel():
    trace = R.single_voxel_rejections(750883)
    cum = np.cumsum([r for _, r in trace])
    calls = [m for m, _ in trace]
    # the 1st, 2nd, 63rd, 64th and 65th extra draws and where they fall
    at = {j: calls[int(np.searchsorted(cum, j))] for j in (1, 2, 63, 64, 65)}
    assert at == {1: 1310, 2: 122566, 63: 746093, 64: 747943, 65: 750882}
    # a cloud of n points in one voxel makes n - 1 calls
    for n in (1311, 1312, 122567, 122568, 747944, 747945, 747946, 750883, 750884):
        pts = np.full((n, 3), 0.25, F)
        want = VFO.voxel_filter(pts, 2.0)[1]["rejections"]
        assert sum(r for m, r in trace if m < n - 1) == want, n
    kept, t = R.voxel_filter([7] * 122568)
    assert t == [(1310, 1), (122566, 1)]
    np.testing.assert_array_equal(kept, VFO.voxel_filter(np.zeros((122568, 3), F), 1.0)[0])


def _adaptive_clouds():
    rng = np.random.RandomState(9)
    out = [rng.uniform(-3, 3, (300, 3)).astype(F), rng.normal(0, 2, (800, 3)).astype(F),
           np.vstack([np.zeros((5, 3)), [[0, 0, -1], [0, 0, -1.1], [0, 0, -0.6]]]).astype(F)]
    out.append(np.vstack([out[0], out[0][:50]]))
    return out


@pytest.mark.parametrize("opts", [(2.0, 20.0, 1e9), (0.5, 250.0, 4.0), (8.0, 100.0, 1e9),
                                  (1.0, 3.0, 1.0), (1.0, 600.0, 1e9), (1.0, 0.0, 1e9),
                                  (1.0, -2.0, 1e9), (1.0, 10.0, float("inf")),
                                  (1.0, 10.0, -1.0), (4.0, 7.0, 1e9)])
def test_adaptive_search_against_the_restatement(opts):
    decided = 0
    for pts in _adaptive_clouds():
        kept, s = R.adaptive_voxel_filter(pts, *opts)
        want, st = VFO.adaptive_voxel_filter(pts, *opts)
        if not s["decided"]:
            continue
        decided += 1
        np.testing.assert_array_equal(kept, want)
        assert s["trials"] == st["trials"]
        assert (s["length"] or 0.0) == st["length"]
    assert decided >= 3


def _outlier_batches(seed, nb=4, n=300):
    rng = np.random.RandomState(seed)
    out = []
    for b in range(nb):
        o = rng.uniform(-1, 1, 3).astype(F)
        d = rng.normal(0, 1, (n, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        p = (o + d * rng.uniform(0.5, 4.0, (n, 1))).astype(F)
        p[::37] = o                                   # zero-length rays
        out.append((o, p))
    return out


@pytest.mark.parametrize("voxel_size,limit", [(0.25, 3.0), (0.1, 0.5), (0.3, 0.0), (0.2, -1.0)])
def test_outlier_removal_against_the_restatement(voxel_size, limit):
    for seed in range(10):                # a seed whose every cell is decided
        batches = _outlier_batches(seed)
        got = R.outlier_removal(batches, voxel_size, limit)
        if got["decided"]:
            break
    assert got["decided"]
    hits, rays, kept = ORO.run(batches, voxel_size, limit)
    idx, h = R.voxel_arrays(got["hits"])
    np.testing.assert_array_equal(idx, hits[0])
    np.testing.assert_array_equal(h, hits[1])
    idx, h2, r2 = R.voxel_arrays(got["rays"])
    np.testing.assert_array_equal(idx, rays[0])
    np.testing.assert_array_equal(h2, rays[1])
    np.testing.assert_array_equal(r2, rays[2])
    for a, b in zip(got["kept"], kept):
        np.testing.assert_array_equal(a, b)


def test_ray_samples_and_exact_ties():
    for vs, length in ((0.1, 3.0), (0.25, 1.0), (0.25, 1.0000001), (0.05, 0.0), (1e-3, 7.5)):
        np.testing.assert_array_equal(R.ray_samples(vs, F(length)), ORO.ray_samples(vs, F(length)))
    # x_4 = 1.0 exactly at voxel_size 0.25: a ray of length 1 takes 4 samples, not 5
    assert len(R.ray_samples(0.25, F(1.0))) == 4
    # rays == limit * hits exactly drops the point; a voxel with no hits drops it too
    b = [(F([0, 0, 0]), F([[1.0, 0, 0], [0.5, 0, 0], [0.5, 0, 0]]))]
    got = R.outlier_removal(b, 0.25, 0.5)
    assert got["decided"] and got["rays"][(2, 0, 0)] == (2, 1) and list(got["kept"][0]) == [0]
    assert list(R.outlier_removal(b, 0.25, 0.5 + 2.0 ** -40)["kept"][0]) == [0, 1, 2]


def test_xray_against_the_restatement():
    rng = np.random.RandomState(6)
    for vs, factor in ((0.1, 1.0), (0.05, 0.0), (0.2, -1.5), (0.1, 1e30), (0.07, 2.0)):
        batches = []
        for b in range(3):
            n = int(rng.randint(1, 500))
            p = rng.uniform(-1, 1, (n, 3)).astype(F)
            c = None if b == 1 else rng.uniform(0, 1, (n, 3)).astype(F)
            batches.append((p, c))
        got = R.xray(batches, vs, factor)
        o = XO.Processor(vs, factor)
        for p, c in batches:
            assert o.insert(p, c)
        assert got["decided"]
        lo, hi, empty = o.bounding_box()
        assert not empty and got["box"] == (tuple(lo), tuple(hi))
        np.testing.assert_array_equal(np.array(sorted(got["voxels"], key=lambda v: v[::-1])),
                                      o.voxels())
        yz, sums, counts = o.columns()
        cols = sorted(got["columns"])
        np.testing.assert_array_equal(np.array(cols), yz)
        np.testing.assert_array_equal(
            np.array([got["columns"][k][:3] for k in cols], F).view(np.uint32), sums.view(np.uint32))
        np.testing.assert_array_equal([got["columns"][k][3] for k in cols], counts)
        np.testing.assert_array_equal(got["pixels"], o.draw())
    for mean in (0.0, 0.3, 1.0, 1.7, -0.2):
        for t in (0.0, 0.25, 1.0, -3.0, 0.999):
            assert R.to_uint8(R.mix_from_white(F(mean), F(t))) == XO.channel(mean, t)


def test_mix_and_slots_against_the_header(H):
    rng = np.random.RandomState(8)
    keys = [0, 1, R.EMPTY_KEY, R.pack(-8192, -8192, -8192), R.pack(8191, 8191, 8191)] + \
        [int(v) for v in rng.randint(0, 2 ** 63, 500, dtype=np.int64)]
    for k in keys:
        assert R.mix(k) == H.pb_mix(k)
    np.testing.assert_array_equal(R.mix_array(np.array(keys, np.uint64)),
                                  np.array([R.mix(k) for k in keys], np.uint64))
    for x, y, z in ((0, 0, 0), (-8192, 5, 8191), (17, -3, -8000)):
        assert R.pack(x, y, z) == H.pb_pack(x, y, z)
    assert R.table_slots(0, 0) == 4096 and R.table_slots(4096, 2048) == 4096
    assert R.table_slots(4096, 2049) == 8192


@pytest.mark.parametrize("slots", [16, 4096, 8192])
def test_probe_chains_that_wrap(H, slots):
    """Keys whose home is the last slot take it, then slots 0, 1, ...: in the header's Insert
    and Find, before and after moving every key into a table twice the size."""
    cand = [R.pack(x, y, 3) for x in range(-200, 200) for y in range(-100, 100)]
    last = R.keys_at_slot(cand, slots, count=3)
    first = R.keys_at_slot(cand, slots, slot=0, count=2)
    for k in last:
        assert H.pb_mix(k) & (slots - 1) == slots - 1
    for k in first:
        assert H.pb_mix(k) & (slots - 1) == 0
    order = [last[0], first[0], last[1], last[2], first[1]]
    want = R.probe_chain(order, slots)
    assert want == [slots - 1, 0, 1, 2, 3]
    table = np.full(slots, R.EMPTY_KEY, np.uint64)
    tp = table.ctypes.data_as(C.c_void_p)
    ins = C.c_int()
    got = [H.pb_insert(tp, slots - 1, k, C.byref(ins)) for k in order]
    assert got == want
    assert H.pb_insert(tp, slots - 1, last[2], C.byref(ins)) == 2 and ins.value == 0
    for k, h in zip(order, want):
        assert H.pb_find(tp, slots - 1, k) == h
    absent = R.keys_at_slot(cand[::-1], slots, count=1)[0]
    assert absent not in order and H.pb_find(tp, slots - 1, absent) == -1
    # k_rehash's order: slot by slot into a table of twice the size
    big = np.full(2 * slots, R.EMPTY_KEY, np.uint64)
    bp = big.ctypes.data_as(C.c_void_p)
    moved = [int(k) for k in table if int(k) != R.EMPTY_KEY]
    for k in moved:
        H.pb_insert(bp, 2 * slots - 1, k, C.byref(ins))
    for k, h in zip(moved, R.probe_chain(moved, 2 * slots)):
        assert H.pb_find(bp, 2 * slots - 1, k) == h
