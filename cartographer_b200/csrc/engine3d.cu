// FastCorrelativeScanMatcher3D on H100.  Reference: cartographer/mapping/internal/3d/
// scan_matching/{fast_correlative_scan_matcher_3d,precomputation_grid_3d,
// rotational_scan_matcher,low_resolution_matcher}.cc and mapping/3d/hybrid_grid.h.
//
// The reference's HybridGrid is a 3-level pointer tree; on the device every
// precomputation depth is a DENSE uint8 box over the bounding box of its non-zero
// voxels (value() of an unallocated or out-of-range cell is 0 in the reference,
// hybrid_grid.h:267-275, which is exactly "outside the box reads 0").  Pose
// algebra (a few quaternion products per rotated scan) and all transcendentals run
// on the host, as in the 2D path; every float expression that reaches an output
// uses round-to-nearest intrinsics in the reference's operation order.
#include <algorithm>
#include <climits>
#include <cmath>
#include <functional>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "grid3d.cuh"
#include "proto_write.h"
#include "rigid3f.h"
#include "value_conversion.h"

#include <atomic>
#include <mutex>
#include <string>
#include <thread>

namespace csm {

constexpr int kMaxDepth3 = 12;

struct Vol8 {
  const uint8_t* p;
  int lo[3];
  int n[3];
};
struct Stack3Dev {
  Vol8 level[kMaxDepth3];
  int depth, frd;
  float resolution;
};
struct Low3Dev {
  const uint16_t* p;
  int lo[3];
  int n[3];
  float resolution, k_scale, bias, min_probability;
};
struct Scan3 {
  float tx, ty, tz, qw, qx, qy, qz;  // DiscreteScan3D::pose
  float nw, nx, ny, nz;              // rotation of GetPoseFromCandidate (normalised)
  float rot_score;
};
struct Job3 {
  const Stack3Dev* stack;
  const Low3Dev* low;
  const float* hi_xyz;
  const float* lo_xyz;
  const Scan3* scans;  // the scans that passed the rotational filter (written on the device)
  const int* ctl;      // control block (kC3*): [kC3Scans] = number of such scans
  short4* cells;       // [scan][point]
  int n_hi, n_lo, max_scans;   // max_scans = number of angles (upper bound of the scan count)
  int wxy, wz;         // linear window sizes in voxels
  int nxc, nzc;        // lowest-resolution candidates per axis (x == y)
  float min_score;
  float min_low;       // min_low_resolution_score as float? compared in double below
  double min_low_d;
};
struct Node3 { int scan, ox, oy, oz; float score; };
struct Leaf3 { int scan, ox, oy, oz; float score, low; };

// HybridGridBase::GetCellIndex (hybrid_grid.h:428-433): lround(p / resolution) in float.
__device__ __forceinline__ int CellOf(float p, float resolution) {
  return static_cast<int>(lroundf(__fdiv_rn(p, resolution)));
}
// PrecomputationGrid3D::ToProbability(sum / float(N))  (precomputation_grid_3d.h:32-35)
__device__ __forceinline__ float ToScore3(int sum, int n) {
  const float kMin = kMinProbability;
  const float kMax = __fsub_rn(1.f, kMin);
  const float k = __fdiv_rn(__fsub_rn(kMax, kMin), 255.f);
  return __fadd_rn(kMin, __fmul_rn(__fdiv_rn(__int2float_rn(sum), __int2float_rn(n)), k));
}
__device__ __forceinline__ int Val8(const Vol8& v, int x, int y, int z) {
  const int lx = x - v.lo[0], ly = y - v.lo[1], lz = z - v.lo[2];
  if (static_cast<unsigned>(lx) >= static_cast<unsigned>(v.n[0]) ||
      static_cast<unsigned>(ly) >= static_cast<unsigned>(v.n[1]) ||
      static_cast<unsigned>(lz) >= static_cast<unsigned>(v.n[2]))
    return 0;
  return __ldg(v.p + (static_cast<size_t>(lz) * v.n[1] + ly) * v.n[0] + lx);
}

// ---------------------------------------------------------------------------
// K5: precomputation stack
// ---------------------------------------------------------------------------
__global__ void k3_scatter_u8(const int* __restrict__ idx, const uint16_t* __restrict__ values,
                              long long n, const uint8_t* __restrict__ lut, Vol8 v,
                              uint8_t* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int x = idx[3 * i] - v.lo[0], y = idx[3 * i + 1] - v.lo[1], z = idx[3 * i + 2] - v.lo[2];
  out[(static_cast<size_t>(z) * v.n[1] + y) * v.n[0] + x] = lut[values[i]];
}
__global__ void k3_scatter_u16(const int* __restrict__ idx, const uint16_t* __restrict__ values,
                               long long n, Low3Dev v, uint16_t* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int x = idx[3 * i] - v.lo[0], y = idx[3 * i + 1] - v.lo[1], z = idx[3 * i + 2] - v.lo[2];
  out[(static_cast<size_t>(z) * v.n[1] + y) * v.n[0] + x] = values[i];
}

// ---- the same from a csm_grid3d's dense box (csm_matcher3d_create_from_grid3d) ----
// Launch shape of the three kernels below: x along a row of the box they walk (coalesced),
// blockIdx.y strides over the rows (y + n1 * z).
struct Box16 {
  const uint16_t* p;
  int lo[3];
  int n[3];
};

// The bounding box of the non-zero cells of `b`, as offsets from b.lo: mn[0..2] receives the
// min (atomicMin; the caller sets them to 0xffffffff), mx[0..2] the max + 1 (atomicMax; the
// caller zeroes them), so mx[0] != 0 is the "any non-zero cell" flag.  Per thread, then per
// block (warp reductions + shared memory), then six atomics per block that saw a cell.
__global__ void __launch_bounds__(256)
k3_nonzero_box(Box16 b, unsigned* __restrict__ mn_out, unsigned* __restrict__ mx_out) {
  __shared__ unsigned s[6][8];
  unsigned mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u};
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const long long rows = static_cast<long long>(b.n[1]) * b.n[2];
  if (x < b.n[0]) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
      if (__ldg(b.p + r * b.n[0] + x) == 0) continue;
      const unsigned y = static_cast<unsigned>(r % b.n[1]), z = static_cast<unsigned>(r / b.n[1]);
      const unsigned c[3] = {static_cast<unsigned>(x), y, z};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        mn[a] = min(mn[a], c[a]);
        mx[a] = max(mx[a], c[a] + 1u);
      }
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
    if (lane == 0) {
      s[a][warp] = mn[a];
      s[3 + a][warp] = mx[a];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned v[6];
    for (int a = 0; a < 6; ++a) {
      v[a] = s[a][0];
      for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w)
        v[a] = a < 3 ? min(v[a], s[a][w]) : max(v[a], s[a][w]);
    }
    if (v[3] != 0u)
      for (int a = 0; a < 3; ++a) {
        atomicMin(&mn_out[a], v[a]);
        atomicMax(&mx_out[a], v[3 + a]);
      }
  }
}

// The value of cell (x, y, z) of the source box, 0 outside it.
__device__ __forceinline__ uint16_t Val16(const Box16& b, int x, int y, int z) {
  const int lx = x - b.lo[0], ly = y - b.lo[1], lz = z - b.lo[2];
  if (static_cast<unsigned>(lx) >= static_cast<unsigned>(b.n[0]) ||
      static_cast<unsigned>(ly) >= static_cast<unsigned>(b.n[1]) ||
      static_cast<unsigned>(lz) >= static_cast<unsigned>(b.n[2]))
    return 0;
  return __ldg(b.p + (static_cast<size_t>(lz) * b.n[1] + ly) * b.n[0] + lx);
}

// Depth 0 (ConvertToPrecomputationGrid) in gather form: one thread per level-0 cell.  A cell
// outside the source box reads 0, which the LUT maps to 0 as the scatter form's memset leaves it.
__global__ void __launch_bounds__(256)
k3_gather_u8(Box16 src, const uint8_t* __restrict__ lut, Vol8 v, uint8_t* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= v.n[0]) return;
  const long long rows = static_cast<long long>(v.n[1]) * v.n[2];
  for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
    const int y = static_cast<int>(r % v.n[1]), z = static_cast<int>(r / v.n[1]);
    out[r * v.n[0] + x] = __ldg(lut + Val16(src, x + v.lo[0], y + v.lo[1], z + v.lo[2]));
  }
}

// The low-resolution volume: the cells of the source box inside `v`, copied as they are.
__global__ void __launch_bounds__(256)
k3_gather_u16(Box16 src, Low3Dev v, uint16_t* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= v.n[0]) return;
  const long long rows = static_cast<long long>(v.n[1]) * v.n[2];
  for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
    const int y = static_cast<int>(r % v.n[1]), z = static_cast<int>(r / v.n[1]);
    out[r * v.n[0] + x] = Val16(src, x + v.lo[0], y + v.lo[1], z + v.lo[2]);
  }
}

// ---- the non-zero voxels of a csm_grid3d in HybridGrid's iteration order (csm_grid3d_voxels) ----
// HybridGrid is DynamicGrid<NestedGrid<FlatGrid<uint16, 3>, 3>> (hybrid_grid.h), and each level
// walks its cells in ToFlatIndex order, z outermost (:40-43), skipping null meta cells and value 0
// (:57, :106-115).  The DynamicGrid shifts an index by grid_size() / 2 = 2^(bits - 1) * 64, a
// multiple of 64 (:263-264), so its meta cells are the 64^3 blocks floor(index / 64) in z, y, x
// order, whatever bits_ is and however the grid grew; inside them come the NestedGrid's 8^3 blocks
// and inside those the cells, both in z, y, x order.  The kernels below enumerate the 64-aligned
// cover of the non-zero box in that blocked order and compact the non-zero cells stably: tile t is
// kVoxTile consecutive cells of the enumeration (4 of the 8^3 blocks, 128 tiles per 64^3 block),
// and thread k of a tile holds the x-row (z & 7, y & 7) = ((k & 63) >> 3, k & 7) of its block
// k >> 6.  No sort is needed.
constexpr int kVoxThreads = 256;
constexpr int kVoxTile = 8 * kVoxThreads;

struct VoxCover {
  Box16 src;
  int lo[3];   // multiples of 64
  int nb[3];   // 64^3 blocks per axis
};

// The 8 cells x .. x + 7 of this thread's row in tile t, and their values in v.
__device__ __forceinline__ void VoxRow(const VoxCover& c, long long t, int* x, int* y, int* z,
                                       uint16_t v[8]) {
  const long long m = t >> 7;                                          // the 64^3 block
  const int f = static_cast<int>(t & 127) * 4 + (threadIdx.x >> 6);    // the 8^3 block in it
  const int r = threadIdx.x & 63;
  const long long bxy = static_cast<long long>(c.nb[0]) * c.nb[1];
  const int bz = static_cast<int>(m / bxy);
  const int by = static_cast<int>((m % bxy) / c.nb[0]);
  const int bx = static_cast<int>(m % c.nb[0]);
  *x = c.lo[0] + 64 * bx + 8 * (f & 7);
  *y = c.lo[1] + 64 * by + 8 * ((f >> 3) & 7) + (r & 7);
  *z = c.lo[2] + 64 * bz + 8 * (f >> 6) + (r >> 3);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = Val16(c.src, *x + i, *y, *z);
}

// Pass 1: counts[t] = the non-zero cells of tile t.
__global__ void __launch_bounds__(kVoxThreads)
k3_voxel_count(VoxCover c, long long* __restrict__ counts) {
  __shared__ int s[kVoxThreads / 32];
  int x, y, z;
  uint16_t v[8];
  VoxRow(c, blockIdx.x, &x, &y, &z, v);
  int n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) n += v[i] != 0;
  n = __reduce_add_sync(0xffffffffu, n);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < kVoxThreads / 32; ++w) total += s[w];
    counts[blockIdx.x] = total;
  }
}

// Pass 2: the non-zero cells of tile t written from offsets[t] on, in enumeration order:
// idx as {x, y, z}, val as held.
__global__ void __launch_bounds__(kVoxThreads)
k3_voxel_write(VoxCover c, const long long* __restrict__ counts,
               const long long* __restrict__ offsets, int* __restrict__ idx,
               uint16_t* __restrict__ val) {
  typedef cub::BlockScan<int, kVoxThreads> Scan;
  __shared__ typename Scan::TempStorage scan;
  if (counts[blockIdx.x] == 0) return;   // uniform over the block
  int x, y, z;
  uint16_t v[8];
  VoxRow(c, blockIdx.x, &x, &y, &z, v);
  int n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) n += v[i] != 0;
  int before;
  Scan(scan).ExclusiveSum(n, before);
  long long o = offsets[blockIdx.x] + before;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (v[i] == 0) continue;
    idx[3 * o] = x + i;
    idx[3 * o + 1] = y;
    idx[3 * o + 2] = z;
    val[o] = v[i];
    ++o;
  }
}

// PrecomputeGrid (precomputation_grid_3d.cc:63-81) in gather form: the reference
// scatters every source voxel to the 8 cells idx - shift*octant (then floor-halves
// the index if half_resolution); the cell c therefore receives the max over
//   full resolution : prev[c + shift*o],                o in {0,1}^3
//   half resolution : prev[2c + {0,1} + shift*o] per axis.
__global__ void k3_precompute(Vol8 prev, Vol8 out, uint8_t* __restrict__ dst, int shift,
                              int half) {
  const long long total = static_cast<long long>(out.n[0]) * out.n[1] * out.n[2];
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(t % out.n[0]) + out.lo[0];
    const int y = static_cast<int>((t / out.n[0]) % out.n[1]) + out.lo[1];
    const int z = static_cast<int>(t / (static_cast<long long>(out.n[0]) * out.n[1])) + out.lo[2];
    int m = 0;
    if (!half) {
      for (int o = 0; o < 8; ++o)
        m = max(m, Val8(prev, x + shift * (o & 1), y + shift * ((o >> 1) & 1),
                        z + shift * ((o >> 2) & 1)));
    } else {
      const int xs[4] = {2 * x, 2 * x + 1, 2 * x + shift, 2 * x + 1 + shift};
      const int ys[4] = {2 * y, 2 * y + 1, 2 * y + shift, 2 * y + 1 + shift};
      const int zs[4] = {2 * z, 2 * z + 1, 2 * z + shift, 2 * z + 1 + shift};
      for (int a = 0; a < 4; ++a)
        for (int b = 0; b < 4; ++b)
          for (int c = 0; c < 4; ++c) m = max(m, Val8(prev, xs[c], ys[b], zs[a]));
    }
    dst[t] = static_cast<uint8_t>(m);
  }
}

// ---------------------------------------------------------------------------
// K7: RotationalScanMatcher::Match — one thread per angle, sequential float ops
// ---------------------------------------------------------------------------
__global__ void k3_rotational(const float* __restrict__ submap_hist,
                              const float* __restrict__ hist, int size, float initial_angle,
                              const float* __restrict__ angles, int num_angles,
                              float* __restrict__ scores) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= num_angles) return;
  const float angle = __fadd_rn(initial_angle, angles[a]);
  // RotateHistogram (rotational_scan_matcher.cc:141-162)
  const float rotate_by_buckets = __double2float_rn(
      __ddiv_rn(static_cast<double>(__fmul_rn(-angle, __int2float_rn(size))), M_PI));
  int full_buckets = static_cast<int>(lroundf(__fsub_rn(rotate_by_buckets, 0.5f)));
  const float fraction = __fsub_rn(rotate_by_buckets, __int2float_rn(full_buckets));
  while (full_buckets < 0) full_buckets += size;
  const float one_minus = __fsub_rn(1.f, fraction);
  // MatchHistograms (:121-132)
  float scan_sq = 0.f, submap_sq = 0.f, dot = 0.f;
  for (int i = 0; i < size; ++i) {
    const float r0 = hist[(i + full_buckets) % size];
    const float r1 = hist[(i + 1 + full_buckets) % size];
    const float s = __fadd_rn(__fmul_rn(fraction, r1), __fmul_rn(one_minus, r0));
    const float m = submap_hist[i];
    scan_sq = __fadd_rn(scan_sq, __fmul_rn(s, s));
    submap_sq = __fadd_rn(submap_sq, __fmul_rn(m, m));
    dot = __fadd_rn(dot, __fmul_rn(m, s));
  }
  const float normalization = __fmul_rn(__fsqrt_rn(scan_sq), __fsqrt_rn(submap_sq));
  scores[a] = normalization < 1e-3f ? 1.f : __fdiv_rn(dot, normalization);
}

__global__ void k3_fill(float* __restrict__ p, int n, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ---- device-resident control of a match ---------------------------------------------
// Frontier sizes, the scan count after the rotational filter and the bound never visit the
// host between kernels: a match is one stream of launches and one synchronisation.
enum : int {
  kC3Leaf = 16,      // leaves recorded
  kC3Best = 17,      // optimal leaves after compaction
  kC3Scans = 18,     // scans that passed the rotational filter
  kC3TopBest = 19,   // largest lowest-resolution sum of the match (dive selection)
  kC3Overflow = 20,
  kC3Start = 25,     // chunk of the current level: first node / count
  kC3Count = 26,
  kC3Bound = 28,     // the bound (order-preserving uint)
  kC3Ints = 32
};

// GenerateDiscreteScans' filter (:273-281): keeps the angles whose rotational score is not
// below min_rotational_score (float < double), in angle order.  One CTA, ordered compaction.
__global__ void __launch_bounds__(1024)
k3_select_scans(const Scan3* __restrict__ all, const float* __restrict__ rot_scores,
                int num_angles, double min_rotational_score, Scan3* __restrict__ out,
                int* __restrict__ sel, int* __restrict__ ctl, unsigned lb0) {
  __shared__ int s_warp[32];
  __shared__ int s_base;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int a0 = 0; a0 < num_angles; a0 += 1024) {
    const int a = a0 + threadIdx.x;
    const float rs = a < num_angles ? rot_scores[a] : 0.f;
    const bool keep = a < num_angles && !(static_cast<double>(rs) < min_rotational_score);
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < 32; ++w) {
      const int c = s_warp[w];
      if (w < warp) before += c;
      total += c;
    }
    if (keep) {
      const int k = s_base + before + __popc(m & ((1u << lane) - 1));
      Scan3 sc = all[a];
      sc.rot_score = rs;
      out[k] = sc;
      sel[k] = a;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    ctl[kC3Scans] = s_base;
    reinterpret_cast<unsigned*>(ctl)[kC3Bound] = lb0;
  }
}

__global__ void k3_level_begin(int* __restrict__ ctl, int h, int chunk_cap) {
  if (threadIdx.x != 0) return;
  const int have = ctl[h];
  const int n = min(have, chunk_cap);
  ctl[h] = have - n;          // the chunk is taken from the END of the queue
  ctl[kC3Start] = have - n;
  ctl[kC3Count] = n;
}

// ---------------------------------------------------------------------------
// K2-3D: DiscretizeScan (full-resolution cell indices; :200-218)
// ---------------------------------------------------------------------------
__global__ void k3_discretize(Job3 jb) {
  const int s = blockIdx.y;
  if (s >= jb.ctl[kC3Scans]) return;
  const Scan3 sc = jb.scans[s];
  const Rigid3f pose{Vec3f{sc.tx, sc.ty, sc.tz}, Quatf{sc.qw, sc.qx, sc.qy, sc.qz}};
  const float res = jb.stack->resolution;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < jb.n_hi; p += gridDim.x * blockDim.x) {
    const Vec3f v{jb.hi_xyz[3 * p], jb.hi_xyz[3 * p + 1], jb.hi_xyz[3 * p + 2]};
    const Vec3f w = Rigid3Apply(pose, v);
    const int cx = max(-30000, min(30000, CellOf(w.x, res)));
    const int cy = max(-30000, min(30000, CellOf(w.y, res)));
    const int cz = max(-30000, min(30000, CellOf(w.z, res)));
    jb.cells[static_cast<size_t>(s) * jb.n_hi + p] =
        make_short4(static_cast<short>(cx), static_cast<short>(cy), static_cast<short>(cz), 0);
  }
}

// ---------------------------------------------------------------------------
// K6: ScoreCandidates (:332-355)
// ---------------------------------------------------------------------------
// Scores up to 8 candidates of one scan that share the point loads: offsets
// base + half * {ix, iy, iz}, slot t = 4*iz + 2*iy + ix (the reference's child
// generation order: z outer, y, x inner, :412-430).  `mask` selects the slots.
// All threads of the CTA take part; sums[] is valid in thread 0 only.
#ifndef CSM_T3
#define CSM_T3 512   // 256: 0.57 ms dive, 512: 0.33 ms, 1024: 0.24 ms but one CTA per SM
#endif
constexpr int kT3 = CSM_T3;   // threads per CTA of the 3D scoring kernels
__device__ __forceinline__ void ScoreOct(const Job3& jb, int scan, int depth, int bx, int by,
                                         int bz, int half, unsigned mask, int sums[8],
                                         int* s_red) {
  const Stack3Dev& st = *jb.stack;
  const Vol8 v = st.level[depth];
  const int e = max(0, depth - st.frd + 1);             // reduction_exponent (:335-336)
  const int sx = -jb.wxy, sz = -jb.wz;                   // search_window_start (:223-226)
  int ox[2], oy[2], oz[2];
  ox[0] = bx >> e; ox[1] = (bx + half) >> e;             // candidate.offset >> e (:340-342)
  oy[0] = by >> e; oy[1] = (by + half) >> e;
  oz[0] = bz >> e; oz[1] = (bz + half) >> e;
  int acc[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) acc[t] = 0;
  const short4* __restrict__ cells = jb.cells + static_cast<size_t>(scan) * jb.n_hi;
  for (int p = threadIdx.x; p < jb.n_hi; p += kT3) {
    const short4 c = cells[p];
    int cx = c.x, cy = c.y, cz = c.z;
    if (e > 0) {  // low-resolution indices (:226-242)
      cx = ((cx + sx) >> e) - (sx >> e);
      cy = ((cy + sx) >> e) - (sx >> e);
      cz = ((cz + sz) >> e) - (sz >> e);
    }
#pragma unroll
    for (int t = 0; t < 8; ++t)
      if ((mask >> t) & 1u)
        acc[t] += Val8(v, cx + ox[t & 1], cy + oy[(t >> 1) & 1], cz + oz[(t >> 2) & 1]);
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    int a = acc[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if ((threadIdx.x & 31) == 0) s_red[(threadIdx.x >> 5) * 8 + t] = a;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      int a = 0;
      for (int w = 0; w < kT3 / 32; ++w) a += s_red[w * 8 + t];
      sums[t] = a;
    }
  }
  __syncthreads();
}

// child validity mask of a node at level h (children at h-1), clipped by the window
__device__ __forceinline__ unsigned ChildMask3(const Job3& jb, int ox, int oy, int oz, int half) {
  const bool x2 = !(ox + half > jb.wxy), y2 = !(oy + half > jb.wxy), z2 = !(oz + half > jb.wz);
  unsigned m = 0;
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const bool ok = ((t & 1) ? x2 : true) && ((t & 2) ? y2 : true) && ((t & 4) ? z2 : true);
    if (ok) m |= 1u << t;
  }
  return m;
}

// low-resolution matcher (low_resolution_matcher.cc:23-35) for the pose of a leaf
// candidate: ordered float sum over the low-resolution cloud.  CTA-cooperative:
// probabilities are computed in parallel, thread 0 adds them in point order.
__device__ float LowResScore(const Job3& jb, int scan, int ox, int oy, int oz, float* s_buf) {
  const Scan3 sc = jb.scans[scan];
  const float res = jb.stack->resolution;
  // GetPoseFromCandidate (:369-375): Translation(res * offset) * scan.pose
  const Rigid3f pose{Vec3f{__fadd_rn(sc.tx, __fmul_rn(res, __int2float_rn(ox))),
                           __fadd_rn(sc.ty, __fmul_rn(res, __int2float_rn(oy))),
                           __fadd_rn(sc.tz, __fmul_rn(res, __int2float_rn(oz)))},
                     Quatf{sc.nw, sc.nx, sc.ny, sc.nz}};
  const Low3Dev& lg = *jb.low;
  __shared__ float s_sum;
  __syncthreads();  // a previous call's readers of s_sum are done
  if (threadIdx.x == 0) s_sum = 0.f;
  for (int p0 = 0; p0 < jb.n_lo; p0 += kT3) {
    const int p = p0 + threadIdx.x;
    if (p < jb.n_lo) {
      const Vec3f v{jb.lo_xyz[3 * p], jb.lo_xyz[3 * p + 1], jb.lo_xyz[3 * p + 2]};
      const Vec3f w = Rigid3Apply(pose, v);
      const int x = CellOf(w.x, lg.resolution) - lg.lo[0];
      const int y = CellOf(w.y, lg.resolution) - lg.lo[1];
      const int z = CellOf(w.z, lg.resolution) - lg.lo[2];
      int value = 0;
      if (static_cast<unsigned>(x) < static_cast<unsigned>(lg.n[0]) &&
          static_cast<unsigned>(y) < static_cast<unsigned>(lg.n[1]) &&
          static_cast<unsigned>(z) < static_cast<unsigned>(lg.n[2]))
        value = __ldg(lg.p + (static_cast<size_t>(z) * lg.n[1] + y) * lg.n[0] + x) & 0x7fff;
      // ValueToProbability (probability_values.cc:29-37,56-60)
      s_buf[threadIdx.x] = value == 0 ? lg.min_probability
                                      : __fadd_rn(__fmul_rn(__int2float_rn(value), lg.k_scale),
                                                  lg.bias);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = s_sum;
      const int cnt = min(kT3, jb.n_lo - p0);
      for (int i = 0; i < cnt; ++i) s = __fadd_rn(s, s_buf[i]);
      s_sum = s;
    }
    __syncthreads();
  }
  return __fdiv_rn(s_sum, __int2float_rn(jb.n_lo));  // every thread reads the same value
}

// Lowest-resolution pass: one CTA per candidate, generation order
// scan-major, z outer, y, x inner (:315-327).
__global__ void __launch_bounds__(kT3)
k3_score_top(Job3 jb, int* __restrict__ top_sum, int* __restrict__ ctl) {
  __shared__ int s_red[kT3 / 32 * 8];
  const int per_scan = jb.nxc * jb.nxc * jb.nzc;
  const int c = blockIdx.x;
  const int scan = c / per_scan;
  if (scan >= jb.ctl[kC3Scans]) return;
  int r = c - scan * per_scan;
  const int kz = r / (jb.nxc * jb.nxc);
  r -= kz * jb.nxc * jb.nxc;
  const int ky = r / jb.nxc, kx = r - ky * jb.nxc;
  const int hmax = jb.stack->depth - 1;
  int sums[8];
  ScoreOct(jb, scan, hmax, -jb.wxy + (kx << hmax), -jb.wxy + (ky << hmax), -jb.wz + (kz << hmax),
           0, 1u, sums, s_red);
  if (threadIdx.x == 0) {
    top_sum[c] = sums[0];
    atomicMax(&ctl[kC3TopBest], sums[0]);
  }
}

// Greedy dive of one scan's best lowest-resolution candidate; a leaf only raises
// the bound if it passes the low-resolution gate (:389-397).
__global__ void __launch_bounds__(kT3)
k3_dive(Job3 jb, const int* __restrict__ top_sum, float dive_ratio, unsigned* __restrict__ lb,
        unsigned long long* __restrict__ counters) {
  __shared__ int s_red[kT3 / 32 * 8];
  __shared__ float s_buf[kT3];
  __shared__ int s_pick[4];
  const int scan = blockIdx.x;
  if (scan >= jb.ctl[kC3Scans]) return;
  const int per_scan = jb.nxc * jb.nxc * jb.nzc;
  if (threadIdx.x == 0) {
    int best = -1, bi = 0;
    for (int i = 0; i < per_scan; ++i) {
      const int v = top_sum[scan * per_scan + i];
      if (v > best) { best = v; bi = i; }
    }
    s_pick[0] = best;
    s_pick[1] = bi;
  }
  __syncthreads();
  const int best = s_pick[0];
  int r = s_pick[1];
  if (!(ToScore3(best, jb.n_hi) > jb.min_score)) return;
  // only scans whose best bound is close to the match's best are worth a dive (any subset
  // keeps the bound valid; as in the 2D engine this keeps it tight at a fraction of the cost)
  if (static_cast<float>(best) < dive_ratio * static_cast<float>(jb.ctl[kC3TopBest])) return;
  int h = jb.stack->depth - 1;
  const int kz = r / (jb.nxc * jb.nxc);
  r -= kz * jb.nxc * jb.nxc;
  const int ky = r / jb.nxc, kx = r - ky * jb.nxc;
  int ox = -jb.wxy + (kx << h), oy = -jb.wxy + (ky << h), oz = -jb.wz + (kz << h);
  int leaf_sum = best;
  unsigned long long scored = 0;
  while (h > 0) {
    const int half = 1 << (h - 1);
    const unsigned mask = ChildMask3(jb, ox, oy, oz, half);
    int sums[8];
    ScoreOct(jb, scan, h - 1, ox, oy, oz, half, mask, sums, s_red);
    if (threadIdx.x == 0) {
      int b = 0, bs = sums[0];
      for (int t = 1; t < 8; ++t)
        if (((mask >> t) & 1u) && sums[t] > bs) { b = t; bs = sums[t]; }
      s_pick[0] = b;
      s_pick[1] = bs;
    }
    __syncthreads();
    const int b = s_pick[0];
    leaf_sum = s_pick[1];
    __syncthreads();
    scored += __popc(mask);
    ox += (b & 1) * half;
    oy += ((b >> 1) & 1) * half;
    oz += ((b >> 2) & 1) * half;
    --h;
  }
  const float score = ToScore3(leaf_sum, jb.n_hi);
  if (score > jb.min_score) {
    const float low = LowResScore(jb, scan, ox, oy, oz, s_buf);
    if (threadIdx.x == 0) {
      atomicAdd(&counters[2], 1ull);
      if (static_cast<double>(low) >= jb.min_low_d) atomicMax(lb, FloatToOrdered(score));
    }
  }
  if (threadIdx.x == 0) atomicAdd(&counters[0], scored);
}

__global__ void k3_filter_top(Job3 jb, const int* __restrict__ top_sum,
                              const unsigned* __restrict__ lb, Node3* __restrict__ queue,
                              int* __restrict__ qcount) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int per_scan = jb.nxc * jb.nxc * jb.nzc;
  if (c >= jb.ctl[kC3Scans] * per_scan) return;
  const float score = ToScore3(top_sum[c], jb.n_hi);
  if (!(score > jb.min_score && score >= OrderedToFloat(*lb))) return;
  const int scan = c / per_scan;
  int r = c - scan * per_scan;
  const int kz = r / (jb.nxc * jb.nxc);
  r -= kz * jb.nxc * jb.nxc;
  const int ky = r / jb.nxc, kx = r - ky * jb.nxc;
  const int hmax = jb.stack->depth - 1;
  const int idx = atomicAdd(qcount, 1);
  queue[idx] = Node3{scan, -jb.wxy + (kx << hmax), -jb.wxy + (ky << hmax),
                     -jb.wz + (kz << hmax), score};
}

// Branch step (:403-437): CTAs walk the parents of the current chunk (device-side start /
// count, grid-stride), one parent at a time.
__global__ void __launch_bounds__(kT3)
k3_expand(Job3 jb, const Node3* __restrict__ queue, int* __restrict__ ctl, int h,
          Node3* __restrict__ next, int* __restrict__ next_count,
          int next_cap, Leaf3* __restrict__ leaves, int leaf_cap,
          unsigned long long* __restrict__ counters) {
  __shared__ int s_red[kT3 / 32 * 8];
  __shared__ float s_buf[kT3];
  __shared__ int s_sums[8];
  __shared__ float s_bound;
  __shared__ int s_go;
  unsigned* lb = reinterpret_cast<unsigned*>(ctl) + kC3Bound;
  int* leaf_count = ctl + kC3Leaf;
  int* overflow = ctl + kC3Overflow;
  const int count = ctl[kC3Count];
  const Node3* __restrict__ parents = queue + ctl[kC3Start];
  for (int pi = blockIdx.x; pi < count; pi += gridDim.x) {
    const Node3 nd = parents[pi];
    // the bound moves while the kernel runs: one thread samples it, all threads agree
    __syncthreads();
    if (threadIdx.x == 0) s_bound = OrderedToFloat(*lb);
    __syncthreads();
    if (!(nd.score >= s_bound)) continue;
    const int half = 1 << (h - 1);
    const unsigned mask = ChildMask3(jb, nd.ox, nd.oy, nd.oz, half);
    int sums[8];
    ScoreOct(jb, nd.scan, h - 1, nd.ox, nd.oy, nd.oz, half, mask, sums, s_red);
    if (threadIdx.x == 0) {
      for (int t = 0; t < 8; ++t) s_sums[t] = sums[t];
      atomicAdd(&counters[0], (unsigned long long)__popc(mask));
      atomicAdd(&counters[1], 1ull);
    }
    __syncthreads();
    if (h - 1 == 0) {
      for (int t = 0; t < 8; ++t) {
        if (!((mask >> t) & 1u)) continue;
        const float sc = ToScore3(s_sums[t], jb.n_hi);
        // leaf candidates that cannot beat (or tie) the bound need no gate evaluation
        __syncthreads();
        if (threadIdx.x == 0) s_go = (sc > jb.min_score && sc >= OrderedToFloat(*lb)) ? 1 : 0;
        __syncthreads();
        if (!s_go) continue;
        const int ox = nd.ox + (t & 1) * half, oy = nd.oy + ((t >> 1) & 1) * half,
                  oz = nd.oz + ((t >> 2) & 1) * half;
        const float low = LowResScore(jb, nd.scan, ox, oy, oz, s_buf);
        if (threadIdx.x == 0) {
          atomicAdd(&counters[2], 1ull);
          if (static_cast<double>(low) >= jb.min_low_d) {
            const unsigned o = FloatToOrdered(sc);
            const unsigned old = atomicMax(lb, o);
            if (o >= old) {
              const int idx = atomicAdd(leaf_count, 1);
              if (idx < leaf_cap) leaves[idx] = Leaf3{nd.scan, ox, oy, oz, sc, low};
              else *overflow = 1;
            }
          }
        }
        __syncthreads();
      }
    } else if (threadIdx.x == 0) {
      const float bound = OrderedToFloat(*lb);
      for (int t = 0; t < 8; ++t) {
        if (!((mask >> t) & 1u)) continue;
        const float sc = ToScore3(s_sums[t], jb.n_hi);
        if (sc > jb.min_score && sc >= bound) {
          const int idx = atomicAdd(next_count, 1);
          if (idx < next_cap)
            next[idx] = Node3{nd.scan, nd.ox + (t & 1) * half, nd.oy + ((t >> 1) & 1) * half,
                              nd.oz + ((t >> 2) & 1) * half, sc};
          else
            *overflow = 1;
        }
      }
    }
  }
}

// Leaves whose score equals the final bound, with the angle index and rotational score of
// their scan (what the host needs to assemble the Result).
struct BestLeaf3 { int scan, angle, ox, oy, oz; float score, low, rot; };
__global__ void __launch_bounds__(256)
k3_collect(const Leaf3* __restrict__ leaves, const Scan3* __restrict__ scans,
           const int* __restrict__ sel, int* __restrict__ ctl, int leaf_cap,
           BestLeaf3* __restrict__ out, int out_cap) {
  const unsigned bound = reinterpret_cast<const unsigned*>(ctl)[kC3Bound];
  const int count = min(ctl[kC3Leaf], leaf_cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const Leaf3 l = leaves[i];
    if (FloatToOrdered(l.score) != bound) continue;
    const int idx = atomicAdd(&ctl[kC3Best], 1);
    if (idx < out_cap)
      out[idx] = BestLeaf3{l.scan, sel[l.scan], l.ox, l.oy, l.oz, l.score, l.low,
                           scans[l.scan].rot_score};
    else
      ctl[kC3Overflow] = 1;
  }
}

// scores an explicit candidate list (tie resolution): one CTA per candidate; `sums` (may be
// null) also receives the integer sums (test hook csm_score_candidates3d)
struct List3 { int scan, ox, oy, oz, depth; };
__global__ void __launch_bounds__(kT3)
k3_score_list(Job3 jb, const List3* __restrict__ cands, float* __restrict__ scores,
              int* __restrict__ sums_out) {
  __shared__ int s_red[kT3 / 32 * 8];
  const List3 c = cands[blockIdx.x];
  int sums[8];
  ScoreOct(jb, c.scan, c.depth, c.ox, c.oy, c.oz, 0, 1u, sums, s_red);
  if (threadIdx.x == 0) {
    scores[blockIdx.x] = ToScore3(sums[0], jb.n_hi);
    if (sums_out) sums_out[blockIdx.x] = sums[0];
  }
}

}  // namespace csm

// ===========================================================================
// Host side
// ===========================================================================
using namespace csm;

struct csm_matcher3d {
  Ctx* ctx = nullptr;
  Stack3Dev hs;            // host copy (device pointers inside)
  Stack3Dev* d_stack = nullptr;
  Low3Dev hl;
  Low3Dev* d_low = nullptr;
  uint8_t* d_levels = nullptr;
  uint16_t* d_lowvol = nullptr;
  float* d_hist = nullptr;
  std::vector<float> hist;
  csm_options3d opt;
  int grid_size = 0;
  // also runs when csm_matcher3d_create fails half-way (cudaFree(nullptr) is a no-op)
  ~csm_matcher3d() {
    cudaFree(d_levels);
    cudaFree(d_lowvol);
    cudaFree(d_stack);
    cudaFree(d_low);
    cudaFree(d_hist);
  }
};

namespace {

struct HostSearch3 {
  int wxy, wz;
  double angular;
  Rigid3f node, submap;
};

struct ScanPlan {
  std::vector<Scan3> scans;
  std::vector<float> angles;
  std::vector<float> all_scores;
  int num_angles = 0;
};

// The level loop (see engine2d.cu): chunks of the queues, their capacity, the leaf lists and
// the optimal leaves read back with the first (usually only) synchronise.
constexpr int kChunk = 1 << 16;
constexpr int kQueueCap = 8 * kChunk;
constexpr int kLeafCap = 1 << 20;
constexpr int kInlineBest = 256;
// read-back area (pinned): control block | counters | first optimal leaves
constexpr size_t kRbCtr = 4 * kC3Ints;
constexpr size_t kRbBest = kRbCtr + 8 * 8;
// Dives start only from scans whose best lowest-resolution sum is within 3 % of the best.
constexpr float kDiveRatio = 0.97f;

// The options csm_matcher3d_create accepts (fast_correlative_scan_matcher_3d.cc:60-61).
csm_status CheckOptions3D(const csm_options3d* options) {
  CSM_REQUIRE(options->branch_and_bound_depth >= 1 &&
              options->branch_and_bound_depth <= kMaxDepth3, "branch_and_bound_depth");  // :60
  CSM_REQUIRE(options->full_resolution_depth >= 1, "full_resolution_depth");            // :61
  return CSM_OK;
}

// The inclusive bounding box of a set of voxels; {0, 0, 0} for an empty set.
struct VoxelBox3 {
  int lo[3] = {0, 0, 0};
  int hi[3] = {0, 0, 0};
};

// What the two ways to build a csm_matcher3d differ in: how depth 0 and the low-resolution
// volume are filled, on the context's stream, into volumes already zeroed.  Each gets the
// box it fills and its destination; FillDepth0 also gets the device LUT of
// ConvertToPrecomputationGrid (precomputation_grid_3d.cc:49-61).
using FillDepth0 = std::function<csm_status(const Vol8& level0, uint8_t* dst, const uint8_t* lut)>;
using FillLow = std::function<csm_status(const Low3Dev& low, uint16_t* dst)>;

// FastCorrelativeScanMatcher3D's ctor over voxel boxes that are already known: level
// geometry, the 24 GB guard, the allocations, the precomputation chain, the low-resolution
// volume and the upload of the records and histogram; one stream synchronisation at the end.
// The caller holds ctx->mu, has made the context's device current and checked `options`.
csm_status BuildMatcher3D(Ctx* ctx, const VoxelBox3& hi_box, float hi_res, int32_t hi_grid_size,
                          const VoxelBox3& lo_box, float lo_res, const float* submap_hist,
                          int32_t hist_n, const csm_options3d* options,
                          const FillDepth0& fill_depth0, const FillLow& fill_low,
                          csm_matcher3d** out) {
  const int* lo0 = hi_box.lo;
  const int* hi0 = hi_box.hi;
  for (int a = 0; a < 3; ++a)
    CSM_REQUIRE(lo0[a] >= -8192 && hi0[a] < 8192, "voxel index outside the 2^14 cube");  // :387
  cudaStream_t s = ctx->stream;
  std::unique_ptr<csm_matcher3d> m(new csm_matcher3d);
  m->ctx = ctx;
  m->opt = *options;
  m->hist.assign(submap_hist, submap_hist + hist_n);
  // HybridGrid::grid_size(): 64 << bits, bits >= 1, grown until every index fits
  int gs = 128;
  for (int a = 0; a < 3; ++a)
    while (lo0[a] < -(gs >> 1) || hi0[a] >= (gs >> 1)) gs <<= 1;
  m->grid_size = hi_grid_size > 0 ? hi_grid_size : gs;

  // ---- level geometry ----
  Stack3Dev& hs = m->hs;
  std::memset(&hs, 0, sizeof(hs));
  hs.depth = options->branch_and_bound_depth;
  hs.frd = options->full_resolution_depth;
  hs.resolution = hi_res;
  int lo[3] = {lo0[0], lo0[1], lo0[2]}, hi[3] = {hi0[0], hi0[1], hi0[2]};
  std::vector<int> shifts(hs.depth, 0), halfs(hs.depth, 0);
  size_t total = 0;
  std::vector<size_t> off(hs.depth);
  int last_width = 1;
  for (int d = 0; d < hs.depth; ++d) {
    if (d > 0) {
      const bool half = d >= hs.frd;
      const int next_width = 1 << d;
      const int f = 1 << std::max(0, d - hs.frd);
      const int shift = (next_width - last_width + (f - 1)) / f;  // :66-72
      shifts[d] = shift;
      halfs[d] = half ? 1 : 0;
      for (int a = 0; a < 3; ++a) {
        lo[a] -= shift;
        if (half) { lo[a] >>= 1; hi[a] >>= 1; }
      }
      last_width = next_width;
    }
    for (int a = 0; a < 3; ++a) {
      hs.level[d].lo[a] = lo[a];
      hs.level[d].n[a] = hi[a] - lo[a] + 1;
    }
    off[d] = total;
    total += (static_cast<size_t>(hs.level[d].n[0]) * hs.level[d].n[1] * hs.level[d].n[2] + 255) /
             256 * 256;
  }
  CSM_REQUIRE(total < (size_t(24) << 30), "dense precomputation volume exceeds 24 GB");
  CSM_CUDA(cudaMalloc(&m->d_levels, std::max<size_t>(total, 256)));
  CSM_CUDA(cudaMemsetAsync(m->d_levels, 0, std::max<size_t>(total, 256), s));
  for (int d = 0; d < hs.depth; ++d) hs.level[d].p = m->d_levels + off[d];

  // ---- depth 0: ConvertToPrecomputationGrid (precomputation_grid_3d.cc:49-61) ----
  std::vector<uint8_t> lut(65536);
  {
    const ValueConversion probability = MakeValueConversion(kMinProbability, kMaxProbability);
    for (int v = 0; v < 65536; ++v) {
      const uint16_t value = static_cast<uint16_t>(v) & 0x7fff;
      const float p = value == 0 ? kMinProbability : probability(value);
      const long q =
          std::lround((p - kMinProbability) * (255.f / (kMaxProbability - kMinProbability)));
      lut[v] = static_cast<uint8_t>(q < 0 ? 0 : (q > 255 ? 255 : q));
    }
  }
  DevBuf& d_lut = ctx->D("m3_lut");
  CSM_TRY(d_lut.Reserve(65536));
  CSM_CUDA(cudaMemcpyAsync(d_lut.p, lut.data(), 65536, cudaMemcpyHostToDevice, s));
  CSM_TRY(fill_depth0(hs.level[0], m->d_levels + off[0], d_lut.as<uint8_t>()));
  for (int d = 1; d < hs.depth; ++d) {
    k3_precompute<<<ctx->sm_count * 16, 256, 0, s>>>(hs.level[d - 1], hs.level[d],
                                                     m->d_levels + off[d], shifts[d], halfs[d]);
    CSM_LAUNCH_CHECK();
  }

  // ---- low-resolution grid ----
  Low3Dev& hl = m->hl;
  std::memset(&hl, 0, sizeof(hl));
  for (int a = 0; a < 3; ++a) {
    hl.lo[a] = lo_box.lo[a];
    hl.n[a] = lo_box.hi[a] - lo_box.lo[a] + 1;
  }
  const size_t lvox = static_cast<size_t>(hl.n[0]) * hl.n[1] * hl.n[2];
  CSM_REQUIRE(lvox < (size_t(4) << 30), "dense low-resolution volume too large");
  CSM_CUDA(cudaMalloc(&m->d_lowvol, std::max<size_t>(lvox * 2, 256)));
  CSM_CUDA(cudaMemsetAsync(m->d_lowvol, 0, std::max<size_t>(lvox * 2, 256), s));
  hl.p = m->d_lowvol;
  hl.resolution = lo_res;
  {
    const ValueConversion probability = MakeValueConversion(kMinProbability, kMaxProbability);
    hl.k_scale = probability.scale;
    hl.bias = probability.bias;
    hl.min_probability = kMinProbability;
  }
  CSM_TRY(fill_low(hl, m->d_lowvol));
  CSM_CUDA(cudaMalloc(&m->d_stack, sizeof(Stack3Dev)));
  CSM_CUDA(cudaMalloc(&m->d_low, sizeof(Low3Dev)));
  CSM_CUDA(cudaMalloc(&m->d_hist, sizeof(float) * std::max(1, hist_n)));
  CSM_CUDA(cudaMemcpyAsync(m->d_stack, &hs, sizeof(hs), cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(m->d_low, &hl, sizeof(hl), cudaMemcpyHostToDevice, s));
  if (hist_n)
    CSM_CUDA(cudaMemcpyAsync(m->d_hist, m->hist.data(), sizeof(float) * hist_n,
                             cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  *out = m.release();
  return CSM_OK;
}

VoxelBox3 ListBox3(const int32_t* idx, int64_t n) {
  VoxelBox3 b;
  if (n == 0) return b;
  for (int a = 0; a < 3; ++a) { b.lo[a] = INT_MAX; b.hi[a] = INT_MIN; }
  for (int64_t i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) {
      b.lo[a] = std::min(b.lo[a], idx[3 * i + a]);
      b.hi[a] = std::max(b.hi[a], idx[3 * i + a]);
    }
  return b;
}

Box16 HandleBox(const csm_grid3d* g) {
  Box16 b;
  b.p = g->g.p;
  for (int a = 0; a < 3; ++a) {
    b.lo[a] = g->g.lo[a];
    b.n[a] = g->g.n[a];
  }
  return b;
}

// Launch shape of k3_nonzero_box / k3_gather_*: x along the rows of a box of n[0] x rows
// cells, blockIdx.y over the rows, at most `max_blocks` blocks in all.
dim3 RowGrid(int nx, long long rows, int max_blocks) {
  const int bx = DivUp(nx, 256);
  const long long by = std::max<long long>(1, std::min<long long>(rows, max_blocks / bx));
  return dim3(bx, static_cast<unsigned>(std::min<long long>(by, 65535)));
}

// The number *n of non-zero voxels of `g` and, when it is at most list_capacity, the voxels in
// HybridGrid's iteration order (k3_voxel_*) in the device workspaces "g3v_idx" ({x, y, z} each)
// and "g3v_val" (*d_idx, *d_val), ready on the stream.  Caller holds ctx->mu.  One stream synchronisation for
// the non-zero box and, if the grid has a non-zero voxel, one for the count.
csm_status DeviceVoxels3D(const csm_grid3d* g, long long list_capacity, long long* n,
                          const int** d_idx, const uint16_t** d_val) {
  Ctx* ctx = g->ctx;
  cudaStream_t s = ctx->stream;
  VoxCover c;
  c.src = HandleBox(g);
  DevBuf* d_box;
  CSM_TRY(ctx->Reserve("g3v_box", 6 * sizeof(unsigned), &d_box));
  unsigned* box = d_box->as<unsigned>();
  CSM_CUDA(cudaMemsetAsync(box, 0xff, 3 * sizeof(unsigned), s));
  CSM_CUDA(cudaMemsetAsync(box + 3, 0, 3 * sizeof(unsigned), s));
  const long long rows = static_cast<long long>(c.src.n[1]) * c.src.n[2];
  k3_nonzero_box<<<RowGrid(c.src.n[0], rows, ctx->sm_count * 8), 256, 0, s>>>(c.src, box, box + 3);
  CSM_LAUNCH_CHECK();
  PinnedBuf& pin = ctx->P("g3v_box");
  CSM_TRY(pin.Reserve(6 * sizeof(unsigned) + sizeof(long long)));
  unsigned* h = pin.as<unsigned>();
  CSM_CUDA(cudaMemcpyAsync(h, box, 6 * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  *n = 0;
  if (h[3] == 0u) return CSM_OK;   // no non-zero cell
  // the 64-aligned cover of the non-zero box (floor division: indices may be negative)
  long long tiles = static_cast<long long>(262144 / kVoxTile);
  for (int a = 0; a < 3; ++a) {
    const int b0 = (c.src.lo[a] + static_cast<int>(h[a]) + 8192) / 64 - 128;
    const int b1 = (c.src.lo[a] + static_cast<int>(h[3 + a]) - 1 + 8192) / 64 - 128;
    c.lo[a] = 64 * b0;
    c.nb[a] = b1 - b0 + 1;
    tiles *= c.nb[a];
  }
  if (tiles >= INT_MAX) {   // one block per tile
    SetError("the non-zero box of the grid is too large to enumerate");
    return CSM_E_CAPACITY;
  }
  // counts[tiles] stays 0, so that the exclusive scan's last entry is the total
  size_t scan_bytes = 0;
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<long long*>(nullptr),
                                         static_cast<long long*>(nullptr), tiles + 1, s));
  const size_t o_off = (sizeof(long long) * (tiles + 1) + 255) / 256 * 256;
  const size_t o_temp = 2 * o_off;
  DevBuf* d_work;
  CSM_TRY(ctx->Reserve("g3v_scan", o_temp + scan_bytes, &d_work));
  long long* counts = d_work->as<long long>();
  long long* offsets = reinterpret_cast<long long*>(d_work->as<char>() + o_off);
  CSM_CUDA(cudaMemsetAsync(counts + tiles, 0, sizeof(long long), s));
  k3_voxel_count<<<static_cast<unsigned>(tiles), kVoxThreads, 0, s>>>(c, counts);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(d_work->as<char>() + o_temp, scan_bytes, counts, offsets,
                                         tiles + 1, s));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  long long* h_n = reinterpret_cast<long long*>(h + 6);
  CSM_CUDA(cudaMemcpyAsync(h_n, offsets + tiles, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  *n = *h_n;
  if (*n > list_capacity) return CSM_OK;
  DevBuf* out_idx;
  DevBuf* out_val;
  CSM_TRY(ctx->Reserve("g3v_idx", sizeof(int) * 3 * *n, &out_idx));
  CSM_TRY(ctx->Reserve("g3v_val", sizeof(uint16_t) * *n, &out_val));
  k3_voxel_write<<<static_cast<unsigned>(tiles), kVoxThreads, 0, s>>>(
      c, counts, offsets, out_idx->as<int>(), out_val->as<uint16_t>());
  CSM_LAUNCH_CHECK();
  *d_idx = out_idx->as<int>();
  *d_val = out_val->as<uint16_t>();
  return CSM_OK;
}

}  // namespace

namespace csm {

csm_status NonZeroVoxels3D(const csm_grid3d* g, long long list_capacity, long long* n,
                           const int** d_idx, const uint16_t** d_val) {
  return DeviceVoxels3D(g, list_capacity, n, d_idx, d_val);
}

}  // namespace csm

extern "C" {

csm_status csm_matcher3d_create(const int32_t* hi_idx, const uint16_t* hi_val, int64_t hi_n,
                                float hi_res, int32_t hi_grid_size, const int32_t* lo_idx,
                                const uint16_t* lo_val, int64_t lo_n, float lo_res,
                                const float* submap_hist, int32_t hist_n,
                                const csm_options3d* options, int32_t device,
                                csm_matcher3d** out) {
  CSM_REQUIRE(out && options, "null pointer");
  CSM_REQUIRE(hi_n >= 0 && lo_n >= 0 && (hi_n == 0 || (hi_idx && hi_val)) &&
              (lo_n == 0 || (lo_idx && lo_val)), "voxel lists");
  CSM_REQUIRE(hi_res > 0.f && lo_res > 0.f, "resolution");
  CSM_TRY(CheckOptions3D(options));
  CSM_REQUIRE(hist_n >= 0 && (hist_n == 0 || submap_hist), "histogram");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  cudaStream_t s = ctx->stream;
  DevBuf& d_idx = ctx->D("m3_idx");
  DevBuf& d_val = ctx->D("m3_val");
  // depth 0 and the low-resolution volume scattered from the lists; both lists go through
  // the same staging, so the second waits until the first has been read
  auto fill_depth0 = [&](const Vol8& level0, uint8_t* dst, const uint8_t* lut) -> csm_status {
    if (hi_n == 0) return CSM_OK;
    CSM_TRY(d_idx.Reserve(sizeof(int) * 3 * hi_n));
    CSM_TRY(d_val.Reserve(sizeof(uint16_t) * hi_n));
    CSM_CUDA(cudaMemcpyAsync(d_idx.p, hi_idx, sizeof(int) * 3 * hi_n, cudaMemcpyHostToDevice, s));
    CSM_CUDA(cudaMemcpyAsync(d_val.p, hi_val, sizeof(uint16_t) * hi_n, cudaMemcpyHostToDevice, s));
    k3_scatter_u8<<<DivUp(hi_n, 256), 256, 0, s>>>(d_idx.as<int>(), d_val.as<uint16_t>(), hi_n,
                                                    lut, level0, dst);
    CSM_LAUNCH_CHECK();
    return CSM_OK;
  };
  auto fill_low = [&](const Low3Dev& low, uint16_t* dst) -> csm_status {
    CSM_CUDA(cudaStreamSynchronize(s));
    if (lo_n == 0) return CSM_OK;
    CSM_TRY(d_idx.Reserve(sizeof(int) * 3 * lo_n));
    CSM_TRY(d_val.Reserve(sizeof(uint16_t) * lo_n));
    CSM_CUDA(cudaMemcpyAsync(d_idx.p, lo_idx, sizeof(int) * 3 * lo_n, cudaMemcpyHostToDevice, s));
    CSM_CUDA(cudaMemcpyAsync(d_val.p, lo_val, sizeof(uint16_t) * lo_n, cudaMemcpyHostToDevice, s));
    k3_scatter_u16<<<DivUp(lo_n, 256), 256, 0, s>>>(d_idx.as<int>(), d_val.as<uint16_t>(), lo_n,
                                                     low, dst);
    CSM_LAUNCH_CHECK();
    return CSM_OK;
  };
  return BuildMatcher3D(ctx, ListBox3(hi_idx, hi_n), hi_res, hi_grid_size, ListBox3(lo_idx, lo_n),
                        lo_res, submap_hist, hist_n, options, fill_depth0, fill_low, out);
}

csm_status csm_matcher3d_create_from_grid3d(const csm_grid3d* hybrid_grid,
                                            int32_t grid_size_in_voxels,
                                            const csm_grid3d* low_resolution_hybrid_grid,
                                            const float* submap_hist, int32_t hist_n,
                                            const csm_options3d* options, csm_matcher3d** out) {
  CSM_REQUIRE(hybrid_grid && low_resolution_hybrid_grid && options && out, "null pointer");
  CSM_REQUIRE(hybrid_grid->ctx == low_resolution_hybrid_grid->ctx,
              "the two grids are on different devices");
  CSM_TRY(CheckOptions3D(options));
  CSM_REQUIRE(hist_n >= 0 && (hist_n == 0 || submap_hist), "histogram");
  Ctx* ctx = hybrid_grid->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const Box16 src[2] = {HandleBox(hybrid_grid), HandleBox(low_resolution_hybrid_grid)};
  // ---- the non-zero boxes: [min x y z of both handles | max + 1 of both handles] ----
  DevBuf* d_box;
  CSM_TRY(ctx->Reserve("m3g_box", 12 * sizeof(unsigned), &d_box));
  unsigned* box = d_box->as<unsigned>();
  // with csm_profile_enable, the device spans of this call are recorded as "m3g_nonzero_box"
  // (the two passes) and "m3g_build" (everything after the read-back)
  ProfBegin(ctx);
  CSM_CUDA(cudaMemsetAsync(box, 0xff, 6 * sizeof(unsigned), s));
  CSM_CUDA(cudaMemsetAsync(box + 6, 0, 6 * sizeof(unsigned), s));
  double cells = 0.;
  for (int k = 0; k < 2; ++k) {
    const long long rows = static_cast<long long>(src[k].n[1]) * src[k].n[2];
    k3_nonzero_box<<<RowGrid(src[k].n[0], rows, ctx->sm_count * 8), 256, 0, s>>>(
        src[k], box + 3 * k, box + 6 + 3 * k);
    CSM_LAUNCH_CHECK();
    cells += static_cast<double>(rows) * src[k].n[0];
  }
  ProfEnd(ctx, "m3g_nonzero_box", cells);
  PinnedBuf& pin = ctx->P("m3g_box");
  CSM_TRY(pin.Reserve(12 * sizeof(unsigned)));
  unsigned* h = pin.as<unsigned>();
  CSM_CUDA(cudaMemcpyAsync(h, box, 12 * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  VoxelBox3 vb[2];
  for (int k = 0; k < 2; ++k) {
    if (h[6 + 3 * k] == 0u) continue;   // no non-zero cell: the empty list's box
    for (int a = 0; a < 3; ++a) {
      vb[k].lo[a] = src[k].lo[a] + static_cast<int>(h[3 * k + a]);
      vb[k].hi[a] = src[k].lo[a] + static_cast<int>(h[6 + 3 * k + a]) - 1;
    }
  }
  // ---- depth 0 and the low-resolution volume gathered from the handles ----
  auto fill_depth0 = [&](const Vol8& level0, uint8_t* dst, const uint8_t* lut) -> csm_status {
    const long long rows = static_cast<long long>(level0.n[1]) * level0.n[2];
    k3_gather_u8<<<RowGrid(level0.n[0], rows, 1 << 16), 256, 0, s>>>(src[0], lut, level0, dst);
    CSM_LAUNCH_CHECK();
    return CSM_OK;
  };
  auto fill_low = [&](const Low3Dev& low, uint16_t* dst) -> csm_status {
    const long long rows = static_cast<long long>(low.n[1]) * low.n[2];
    k3_gather_u16<<<RowGrid(low.n[0], rows, 1 << 16), 256, 0, s>>>(src[1], low, dst);
    CSM_LAUNCH_CHECK();
    return CSM_OK;
  };
  ProfBegin(ctx);
  CSM_TRY(BuildMatcher3D(ctx, vb[0], hybrid_grid->g.resolution, grid_size_in_voxels, vb[1],
                         low_resolution_hybrid_grid->g.resolution, submap_hist, hist_n, options,
                         fill_depth0, fill_low, out));
  ProfEnd(ctx, "m3g_build", 0.);
  return CSM_OK;
}

csm_status csm_grid3d_voxels(const csm_grid3d* grid, int32_t* indices, uint16_t* values,
                             int64_t capacity, int64_t* num_voxels) {
  CSM_REQUIRE(grid && num_voxels, "null pointer");
  CSM_REQUIRE((indices == nullptr) == (values == nullptr), "indices and values go together");
  Ctx* ctx = grid->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  long long n = 0;
  const int* d_idx = nullptr;
  const uint16_t* d_val = nullptr;
  CSM_TRY(DeviceVoxels3D(grid, indices ? capacity : -1, &n, &d_idx, &d_val));
  *num_voxels = n;
  if (!indices || n == 0) return CSM_OK;
  if (capacity < n) {
    SetError("capacity %lld is below the %lld non-zero voxels", static_cast<long long>(capacity), n);
    return CSM_E_CAPACITY;
  }
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaMemcpyAsync(indices, d_idx, sizeof(int) * 3 * n, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(values, d_val, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

csm_status csm_grid3d_to_proto(const csm_grid3d* grid, uint8_t* buf, int64_t capacity,
                               int64_t* size) {
  using namespace wire;
  CSM_REQUIRE(grid && size, "null pointer");
  Ctx* ctx = grid->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  long long n = 0;
  const int* d_idx = nullptr;
  const uint16_t* d_val = nullptr;
  CSM_TRY(DeviceVoxels3D(grid, LLONG_MAX, &n, &d_idx, &d_val));
  PinnedBuf& h_idx = ctx->P("g3v_idx");
  PinnedBuf& h_val = ctx->P("g3v_val");
  if (n > 0) {
    CSM_TRY(h_idx.Reserve(sizeof(int) * 3 * n));
    CSM_TRY(h_val.Reserve(sizeof(uint16_t) * n));
    cudaStream_t s = ctx->stream;
    CSM_CUDA(cudaMemcpyAsync(h_idx.p, d_idx, sizeof(int) * 3 * n, cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaMemcpyAsync(h_val.p, d_val, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaStreamSynchronize(s));
  }
  const int* idx = h_idx.as<int>();
  const uint16_t* val = h_val.as<uint16_t>();
  // proto::HybridGrid (hybrid_grid.proto): resolution = 1, packed sint32 x / y / z_indices =
  // 3 / 4 / 5, packed int32 values = 6; HybridGrid::ToProto adds the voxels in iteration order
  int64_t len[4] = {0, 0, 0, 0};
  for (long long i = 0; i < n; ++i) {
    for (int a = 0; a < 3; ++a) len[a] += VarintSize(ZigZag32(idx[3 * i + a]));
    len[3] += VarintSize(val[i]);
  }
  const float resolution = grid->g.resolution;
  int64_t total = FloatFieldSize(resolution);
  if (n > 0)
    for (int f = 0; f < 4; ++f) total += DelimitedSize(len[f]);
  *size = total;
  if (total >= (int64_t(1) << 31)) {
    SetError("a serialized HybridGrid of %lld bytes exceeds protobuf's 2 GiB limit",
             static_cast<long long>(total));
    return CSM_E_CAPACITY;
  }
  if (!buf) return CSM_OK;
  if (capacity < total) {
    SetError("capacity %lld is below the %lld bytes of the message",
             static_cast<long long>(capacity), static_cast<long long>(total));
    return CSM_E_CAPACITY;
  }
  uint8_t* p = PutFloatField(buf, 1, resolution);
  if (n > 0) {
    for (int a = 0; a < 3; ++a) {
      p = PutDelimitedHeader(p, 3 + a, len[a]);
      for (long long i = 0; i < n; ++i) p = PutVarint(p, ZigZag32(idx[3 * i + a]));
    }
    p = PutDelimitedHeader(p, 6, len[3]);
    for (long long i = 0; i < n; ++i) p = PutVarint(p, val[i]);
  }
  return CSM_OK;
}

csm_status csm_matcher3d_destroy(csm_matcher3d* m) {
  if (!m) return CSM_OK;
  std::lock_guard<std::mutex> lock(m->ctx->mu);
  cudaSetDevice(m->ctx->device);
  cudaStreamSynchronize(m->ctx->stream);
  delete m;  // the destructor frees the device buffers
  return CSM_OK;
}

csm_status csm_matcher3d_read_level(const csm_matcher3d* m, int32_t depth, int32_t lo[3],
                                    int32_t dims[3], uint8_t* out) {
  CSM_REQUIRE(m && lo && dims, "null pointer");
  CSM_REQUIRE(depth >= 0 && depth < m->hs.depth, "depth out of range");
  const Vol8& v = m->hs.level[depth];
  if (!out) {
    for (int a = 0; a < 3; ++a) { lo[a] = v.lo[a]; dims[a] = v.n[a]; }
    return CSM_OK;
  }
  std::lock_guard<std::mutex> lock(m->ctx->mu);
  CSM_CUDA(cudaSetDevice(m->ctx->device));
  std::vector<uint8_t> h(static_cast<size_t>(v.n[0]) * v.n[1] * v.n[2]);
  CSM_CUDA(cudaMemcpy(h.data(), v.p, h.size(), cudaMemcpyDeviceToHost));
  const long long nx = dims[0], ny = dims[1], nz = dims[2];
  std::memset(out, 0, static_cast<size_t>(nx * ny * nz));
  for (int z = 0; z < v.n[2]; ++z)
    for (int y = 0; y < v.n[1]; ++y)
      for (int x = 0; x < v.n[0]; ++x) {
        const long long X = x + v.lo[0] - lo[0], Y = y + v.lo[1] - lo[1], Z = z + v.lo[2] - lo[2];
        if (X >= 0 && Y >= 0 && Z >= 0 && X < nx && Y < ny && Z < nz)
          out[(Z * ny + Y) * nx + X] = h[(static_cast<size_t>(z) * v.n[1] + y) * v.n[0] + x];
      }
  return CSM_OK;
}

csm_status csm_rotational_match3d(const float* submap_hist, const float* hist, int32_t n,
                                  float initial_angle, const float* angles, int32_t num_angles,
                                  int32_t device, float* scores) {
  CSM_REQUIRE(submap_hist && hist && angles && scores && n >= 1 && num_angles >= 1, "arguments");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  cudaStream_t s = ctx->stream;
  DevBuf *a, *b, *c, *d;
  CSM_TRY(ctx->Reserve("rot_a", 4 * n, &a));
  CSM_TRY(ctx->Reserve("rot_b", 4 * n, &b));
  CSM_TRY(ctx->Reserve("rot_c", 4 * num_angles, &c));
  CSM_TRY(ctx->Reserve("rot_d", 4 * num_angles, &d));
  CSM_CUDA(cudaMemcpyAsync(a->p, submap_hist, 4 * n, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(b->p, hist, 4 * n, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(c->p, angles, 4 * num_angles, cudaMemcpyHostToDevice, s));
  k3_rotational<<<DivUp(num_angles, 128), 128, 0, s>>>(a->as<float>(), b->as<float>(), n,
                                                        initial_angle, c->as<float>(), num_angles,
                                                        d->as<float>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(scores, d->p, 4 * num_angles, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

}  // extern "C"

// A node's clouds and histogram on the device (a queue matches one node against many
// submaps: uploaded once per csm_match3d_batch call), plus the max point range both
// SearchParameters need (:151-158, :255-260).
struct NodeDev3 {
  const float* hi = nullptr;
  const float* lo = nullptr;
  const float* hist = nullptr;
  float max_range = 0.f;   // max_i |p_i| over the high-resolution cloud (0 if it is empty)
};

static float MaxRange3(const csm_node3d* node) {
  float m = 0.f;
  for (int i = 0; i < node->num_high; ++i) {
    const float* p = node->high_resolution_point_cloud + 3 * i;
    m = std::max(m, std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
  }
  return m;
}

// GenerateDiscreteScans up to (not including) DiscretizeScan (:246-295), host part: the
// angles and the scan pose of EVERY angle.  The rotational scores and the filter (:273-281)
// run on the device (k3_rotational, k3_select_scans), so nothing is read back here.
static csm_status PlanScans(const csm_matcher3d* m, const csm_node3d* node, float max_range,
                            const HostSearch3& sp, ScanPlan* plan, float* initial_angle) {
  const float resolution = m->hs.resolution;
  const float max_scan_range = std::max(max_range, 3.f * resolution);
  const float kSafetyMargin = 1.f - 1e-2f;
  const float angular_step_size =
      kSafetyMargin * std::acos(1.f - (resolution * resolution) /
                                          (2.f * (max_scan_range * max_scan_range)));
  const int angular_window_size =
      static_cast<int>(std::lround(sp.angular / angular_step_size));
  CSM_REQUIRE(angular_window_size >= 0 && angular_window_size < (1 << 20), "angular window");
  plan->angles.clear();
  for (int rz = -angular_window_size; rz <= angular_window_size; ++rz)
    plan->angles.push_back(rz * angular_step_size);
  plan->num_angles = static_cast<int>(plan->angles.size());
  const Rigid3f node_to_submap = Rigid3Mul(Rigid3Inverse(sp.submap), sp.node);
  // gravity_alignment.inverse().cast<float>()
  const double* g = node->gravity_alignment;
  const Quatf ginv = QuatCastInverseD(Quatd{g[0], g[1], g[2], g[3]});
  *initial_angle = GetYaw(QuatMul(node_to_submap.q, ginv));
  CSM_REQUIRE(node->histogram_size == static_cast<int>(m->hist.size()), "histogram sizes differ");
  plan->scans.clear();
  plan->scans.reserve(plan->num_angles);
  const Quatf sub_inv = QuatInverse(sp.submap.q);
  for (int i = 0; i < plan->num_angles; ++i) {
    const Quatf q = QuatMul(
        QuatMul(sub_inv, AngleAxisVectorToRotationQuaternion(Vec3f{0.f, 0.f, plan->angles[i]})),
        sp.node.q);
    // GetPoseFromCandidate's rotation: (identity * q).normalized()
    const Quatf nq = QuatNormalized(QuatMul(Quatf{1.f, 0.f, 0.f, 0.f}, q));
    Scan3 sc;
    sc.tx = node_to_submap.t.x; sc.ty = node_to_submap.t.y; sc.tz = node_to_submap.t.z;
    sc.qw = q.w; sc.qx = q.x; sc.qy = q.y; sc.qz = q.z;
    sc.nw = nq.w; sc.nx = nq.x; sc.ny = nq.y; sc.nz = nq.z;
    sc.rot_score = 1.f;   // overwritten on the device for the scans that are kept
    plan->scans.push_back(sc);
  }
  return CSM_OK;
}

static csm_status MakeSearch3(const csm_matcher3d* m, float max_range, const double node_pose[7],
                              const double submap_pose[7], int full, HostSearch3* sp) {
  auto cast = [](const double p[7], bool rotation_only) {
    Rigid3f r;
    r.t = rotation_only ? Vec3f{0.f, 0.f, 0.f}
                        : Vec3f{static_cast<float>(p[0]), static_cast<float>(p[1]),
                                static_cast<float>(p[2])};
    r.q = Quatf{static_cast<float>(p[3]), static_cast<float>(p[4]), static_cast<float>(p[5]),
                static_cast<float>(p[6])};
    return r;
  };
  const float resolution = m->hs.resolution;
  if (full) {  // :146-170
    const float max_point_distance = max_range;
    const int w = (m->grid_size + 1) / 2 +
                  static_cast<int>(std::lround(max_point_distance / resolution + 0.5f));
    sp->wxy = w;
    sp->wz = w;
    sp->angular = M_PI;
  } else {     // :127-144
    sp->wxy = static_cast<int>(std::lround(m->opt.linear_xy_search_window / resolution));
    sp->wz = static_cast<int>(std::lround(m->opt.linear_z_search_window / resolution));
    sp->angular = m->opt.angular_search_window;
  }
  sp->node = cast(node_pose, full != 0);
  sp->submap = cast(submap_pose, full != 0);
  CSM_REQUIRE(sp->wxy >= 0 && sp->wz >= 0 && sp->wxy < 20000 && sp->wz < 20000, "linear window");
  return CSM_OK;
}

namespace {

// One 3D match: its search, scan plan, job record, staging layout, control block and
// read-back area.  Match3D runs the phases below over it in order; the test hooks run the
// ones they need.
struct Match3 {
  Ctx* ctx = nullptr;
  cudaStream_t s = nullptr;
  const csm_matcher3d* m = nullptr;
  const csm_node3d* node = nullptr;
  const NodeDev3* dev = nullptr;  // the node's clouds already on the device (optional)
  float min_score = 0.f;
  HostSearch3 sp;
  ScanPlan plan;
  float initial_angle = 0.f;
  int hmax = 0;
  Job3 jb;
  long long per_scan = 0, max_top = 0;
  // uploads through pinned staging: scans | angles | ones | histogram | clouds
  size_t o_ang = 0, o_hist = 0;
  const char* dup = nullptr;
  DevBuf *d_scans = nullptr, *d_sel = nullptr, *d_rot = nullptr, *d_cells = nullptr,
         *d_top = nullptr, *d_ctr = nullptr;
  DevBuf *d_qtop = nullptr, *d_q = nullptr, *d_leaves = nullptr, *d_best = nullptr;
  unsigned long long* ctr = nullptr;
  int* ictr = nullptr;    // the control block (kC3*)
  unsigned* lb = nullptr;
  // read-back area (pinned): control block | counters | first optimal leaves
  PinnedBuf* pin = nullptr;
  int* hp = nullptr;
  const unsigned long long* hctr = nullptr;
  const BestLeaf3* best_inline = nullptr;
  int host_syncs = 0;
  // Sweep limits (csm_sweep_limits3d).  A limit below its constant changes only the control
  // flow: every buffer is still reserved at the constant's size.
  int chunk = kChunk;              // nodes per level chunk (k3_level_begin)
  int leaf_cap = kLeafCap;         // leaves recorded before the capacity error
  int inline_best = kInlineBest;   // optimal leaves read back with each collect
  float dive_ratio = kDiveRatio;   // k3_dive's gate; > 1 runs no dive
  // sweep trace: collects (1 + continuation sweeps), most leaves recorded at a collect
  int collects = 0, max_leaves = 0;

  Node3* Queue(int h) const {
    return h == hmax ? d_qtop->as<Node3>() : d_q->as<Node3>() + static_cast<size_t>(kQueueCap) * h;
  }
};

// Host plan: the search, the scan poses of every angle and the lowest-resolution lattice.
csm_status Plan3D(Match3& x, Ctx* ctx, const csm_matcher3d* m, const csm_node3d* node,
                  const NodeDev3* dev, const double node_pose[7], const double submap_pose[7],
                  int full, float min_score) {
  x.ctx = ctx;
  x.s = ctx->stream;
  x.m = m;
  x.node = node;
  x.dev = dev;
  x.min_score = min_score;
  CSM_CUDA(cudaSetDevice(ctx->device));
  const float max_range = dev ? dev->max_range : MaxRange3(node);
  CSM_TRY(MakeSearch3(m, max_range, node_pose, submap_pose, full, &x.sp));
  CSM_TRY(PlanScans(m, node, max_range, x.sp, &x.plan, &x.initial_angle));
  x.hmax = m->hs.depth - 1;
  return CSM_OK;
}

// A match needs a low-resolution cloud and two levels; discretisation alone does not.
csm_status RequireMatchable3D(const Match3& x) {
  CSM_REQUIRE(x.node->num_low >= 1, "empty low-resolution point cloud");
  if (x.hmax == 0) {
    SetError("branch_and_bound_depth == 1 is not supported by the 3D engine");
    return CSM_E_INVALID;
  }
  return CSM_OK;
}

// Workspaces, the job record and the upload of scans, angles, histogram and clouds.
csm_status Upload3D(Match3& x) {
  Ctx* ctx = x.ctx;
  const csm_matcher3d* m = x.m;
  const int A = x.plan.num_angles, n_hi = x.node->num_high, n_lo = x.node->num_low;
  const int hn = x.node->histogram_size;
  x.o_ang = (sizeof(Scan3) * A + 255) / 256 * 256;
  x.o_hist = (x.o_ang + 4 * static_cast<size_t>(A) + 255) / 256 * 256;
  const size_t o_hi = (x.o_hist + 4 * static_cast<size_t>(std::max(1, hn)) + 255) / 256 * 256;
  const size_t o_lo = x.dev ? o_hi : (o_hi + 12 * static_cast<size_t>(n_hi) + 255) / 256 * 256;
  const size_t up_bytes = x.dev ? o_hi : o_lo + 12 * static_cast<size_t>(std::max(1, n_lo));
  PinnedBuf& up = ctx->P("m3_upload");
  DevBuf* d_up;
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(ctx->Reserve("m3_upload", up_bytes, &d_up));
  char* hup = up.as<char>();
  std::memcpy(hup, x.plan.scans.data(), sizeof(Scan3) * A);
  std::memcpy(hup + x.o_ang, x.plan.angles.data(), 4 * static_cast<size_t>(A));
  if (hn) std::memcpy(hup + x.o_hist, x.node->rotational_scan_matcher_histogram, 4 * static_cast<size_t>(hn));
  if (!x.dev) {
    std::memcpy(hup + o_hi, x.node->high_resolution_point_cloud, 12 * static_cast<size_t>(n_hi));
    if (n_lo) std::memcpy(hup + o_lo, x.node->low_resolution_point_cloud, 12 * static_cast<size_t>(n_lo));
  }
  CSM_TRY(ctx->Reserve("m3_scans", sizeof(Scan3) * A, &x.d_scans));
  CSM_TRY(ctx->Reserve("m3_sel", 4 * static_cast<size_t>(A), &x.d_sel));
  CSM_TRY(ctx->Reserve("m3_rot", 4 * static_cast<size_t>(A), &x.d_rot));
  CSM_TRY(ctx->Reserve("m3_cells", sizeof(short4) * static_cast<size_t>(A) * n_hi, &x.d_cells));
  CSM_TRY(ctx->Reserve("m3_ctr", 8 * 8 + 4 * kC3Ints, &x.d_ctr));
  x.dup = d_up->as<char>();
  x.ctr = x.d_ctr->as<unsigned long long>();
  x.ictr = reinterpret_cast<int*>(x.ctr + 8);
  x.lb = reinterpret_cast<unsigned*>(x.ictr) + kC3Bound;

  Job3& jb = x.jb;
  std::memset(&jb, 0, sizeof(jb));
  jb.stack = m->d_stack;
  jb.low = m->d_low;
  jb.hi_xyz = x.dev ? x.dev->hi : reinterpret_cast<const float*>(x.dup + o_hi);
  jb.lo_xyz = x.dev ? x.dev->lo : reinterpret_cast<const float*>(x.dup + o_lo);
  jb.scans = x.d_scans->as<Scan3>();
  jb.ctl = x.ictr;
  jb.cells = x.d_cells->as<short4>();
  jb.n_hi = n_hi;
  jb.n_lo = n_lo;
  jb.max_scans = A;
  jb.wxy = x.sp.wxy;
  jb.wz = x.sp.wz;
  const int step = 1 << x.hmax;
  jb.nxc = (2 * x.sp.wxy + step) / step;   // :301-306
  jb.nzc = (2 * x.sp.wz + step) / step;
  jb.min_score = x.min_score;
  jb.min_low_d = m->opt.min_low_resolution_score;
  x.per_scan = static_cast<long long>(jb.nxc) * jb.nxc * jb.nzc;
  x.max_top = x.per_scan * A;
  CSM_REQUIRE(x.max_top < (1LL << 30), "too many lowest-resolution candidates");

  CSM_CUDA(cudaEventRecord(ctx->ev0, x.s));
  CSM_CUDA(cudaMemcpyAsync(d_up->p, hup, up_bytes, cudaMemcpyHostToDevice, x.s));
  CSM_CUDA(cudaMemsetAsync(x.d_ctr->p, 0, 8 * 8 + 4 * kC3Ints, x.s));
  return CSM_OK;
}

// Rotational scores (K7), the filter and the discretisation of the kept scans, on the device.
csm_status Discretize3D(Match3& x) {
  Ctx* ctx = x.ctx;
  cudaStream_t s = x.s;
  const int A = x.plan.num_angles, hn = x.node->histogram_size;
  const float* d_node_hist = x.dev && x.dev->hist ? x.dev->hist
                                                  : reinterpret_cast<const float*>(x.dup + x.o_hist);
  if (hn > 0) {
    ProfBegin(ctx);
    k3_rotational<<<DivUp(A, 128), 128, 0, s>>>(x.m->d_hist, d_node_hist, hn, x.initial_angle,
                                                reinterpret_cast<const float*>(x.dup + x.o_ang), A,
                                                x.d_rot->as<float>());
    CSM_LAUNCH_CHECK();
    ProfEnd(ctx, "k3_rotational", A);
  } else {
    k3_fill<<<DivUp(A, 256), 256, 0, s>>>(x.d_rot->as<float>(), A, 1.f);
    CSM_LAUNCH_CHECK();
  }
  k3_select_scans<<<1, 1024, 0, s>>>(reinterpret_cast<const Scan3*>(x.dup), x.d_rot->as<float>(),
                                     A, x.m->opt.min_rotational_score, x.d_scans->as<Scan3>(),
                                     x.d_sel->as<int>(), x.ictr, FloatToOrdered(x.min_score));
  CSM_LAUNCH_CHECK();
  ProfBegin(ctx);
  k3_discretize<<<dim3(std::min(DivUp(x.jb.n_hi, 256), 64), A), 256, 0, s>>>(x.jb);
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, "k3_discretize", static_cast<double>(A) * x.jb.n_hi);

  x.pin = &ctx->P("m3_readback");
  CSM_TRY(x.pin->Reserve(kRbBest + sizeof(BestLeaf3) * kInlineBest));
  x.hp = x.pin->as<int>();
  x.hctr = reinterpret_cast<const unsigned long long*>(x.pin->as<char>() + kRbCtr);
  x.best_inline = reinterpret_cast<const BestLeaf3*>(x.pin->as<char>() + kRbBest);
  return CSM_OK;
}

// Reads the control block back into x.hp after the work queued so far (one synchronise).
csm_status ReadCtl3D(Match3& x) {
  CSM_CUDA(cudaMemcpyAsync(x.hp, x.ictr, kRbCtr, cudaMemcpyDeviceToHost, x.s));
  CSM_CUDA(cudaStreamSynchronize(x.s));
  return CSM_OK;
}

// Lowest-resolution pass and dives (grids sized for all angles; filtered-out scans exit).
csm_status TopDive3D(Match3& x) {
  Ctx* ctx = x.ctx;
  CSM_TRY(ctx->Reserve("m3_top", sizeof(int) * x.max_top, &x.d_top));
  ProfBegin(ctx);
  k3_score_top<<<static_cast<int>(x.max_top), kT3, 0, x.s>>>(x.jb, x.d_top->as<int>(), x.ictr);
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, "k3_score_top", static_cast<double>(x.max_top));
  ProfBegin(ctx);
  k3_dive<<<x.plan.num_angles, kT3, 0, x.s>>>(x.jb, x.d_top->as<int>(), x.dive_ratio, x.lb,
                                               x.ctr);
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, "k3_dive", static_cast<double>(x.plan.num_angles) * 8 * x.hmax);
  return CSM_OK;
}

// Queues of the level loop (the top one holds at least `top_queue` nodes) and the
// lowest-resolution candidates above the bound as its top queue.
csm_status FilterTop3D(Match3& x, long long top_queue) {
  Ctx* ctx = x.ctx;
  CSM_TRY(ctx->Reserve("m3_qtop", sizeof(Node3) * top_queue, &x.d_qtop));
  CSM_TRY(ctx->Reserve("m3_queues", sizeof(Node3) * kQueueCap * std::max(1, x.hmax), &x.d_q));
  CSM_TRY(ctx->Reserve("m3_leaves", sizeof(Leaf3) * kLeafCap, &x.d_leaves));
  CSM_TRY(ctx->Reserve("m3_best", sizeof(BestLeaf3) * kLeafCap, &x.d_best));
  k3_filter_top<<<DivUp(x.max_top, 256), 256, 0, x.s>>>(x.jb, x.d_top->as<int>(), x.lb,
                                                        x.Queue(x.hmax), x.ictr + x.hmax);
  CSM_LAUNCH_CHECK();
  return CSM_OK;
}

// One level step of the device-driven level loop (see engine2d.cu).
csm_status LevelStep3D(Match3& x, int h) {
  k3_level_begin<<<1, 32, 0, x.s>>>(x.ictr, h, x.chunk);
  CSM_LAUNCH_CHECK();
  ProfBegin(x.ctx);
  k3_expand<<<x.ctx->sm_count * 4, kT3, 0, x.s>>>(x.jb, x.Queue(h), x.ictr, h,
                                                   h - 1 >= 1 ? x.Queue(h - 1) : nullptr,
                                                   x.ictr + (h - 1 >= 1 ? h - 1 : 23), kQueueCap,
                                                   x.d_leaves->as<Leaf3>(), x.leaf_cap, x.ctr);
  CSM_LAUNCH_CHECK();
  ProfEnd(x.ctx, "k3_expand", 0.);
  return CSM_OK;
}

// Compaction of the gate-passing optimal leaves + read-back of everything the host needs.
csm_status Collect3D(Match3& x) {
  cudaStream_t s = x.s;
  char* pin = x.pin->as<char>();
  CSM_CUDA(cudaMemsetAsync(x.ictr + kC3Best, 0, 4, s));
  k3_collect<<<x.ctx->sm_count, 256, 0, s>>>(x.d_leaves->as<Leaf3>(), x.d_scans->as<Scan3>(),
                                             x.d_sel->as<int>(), x.ictr, x.leaf_cap,
                                             x.d_best->as<BestLeaf3>(), x.leaf_cap);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaEventRecord(x.ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(pin, x.ictr, kRbCtr, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(pin + kRbCtr, x.ctr, 8 * 8, cudaMemcpyDeviceToHost, s));
  if (x.inline_best > 0)
    CSM_CUDA(cudaMemcpyAsync(pin + kRbBest, x.d_best->p, sizeof(BestLeaf3) * x.inline_best,
                             cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  ++x.host_syncs;
  ++x.collects;
  x.max_leaves = std::max(x.max_leaves, x.hp[kC3Leaf]);
  return CSM_OK;
}

// The sweep hmax -> 1, then continuation sweeps for frontiers larger than one chunk,
// deepest non-empty level first.
csm_status Sweep3D(Match3& x) {
  for (int h = x.hmax; h >= 1; --h) CSM_TRY(LevelStep3D(x, h));
  CSM_TRY(Collect3D(x));
  for (;;) {
    if (x.hp[kC3Overflow]) { SetError("3D branch-and-bound capacity exceeded"); return CSM_E_CAPACITY; }
    int h = -1;
    for (int l = 1; l <= x.hmax; ++l)
      if (x.hp[l] > 0) { h = l; break; }
    if (h < 0) break;
    for (int l = h; l >= 1; --l) CSM_TRY(LevelStep3D(x, l));
    CSM_TRY(Collect3D(x));
  }
  return CSM_OK;
}

// Tie resolution: the first optimal, gate-passing leaf in the reference's DFS order is moved
// to ties[0].
csm_status ResolveTies3D(Match3& x, std::vector<BestLeaf3>& ties, int* host_resolves) {
  cudaStream_t s = x.s;
  const int hmax = x.hmax;
  const HostSearch3& sp = x.sp;
  const Job3& jb = x.jb;
  const int T = static_cast<int>(ties.size());
  std::vector<List3> lc;
  for (const BestLeaf3& t : ties)
    for (int l = 1; l <= hmax; ++l)
      lc.push_back(List3{t.scan, -sp.wxy + (((t.ox + sp.wxy) >> l) << l),
                         -sp.wxy + (((t.oy + sp.wxy) >> l) << l),
                         -sp.wz + (((t.oz + sp.wz) >> l) << l), l});
  std::vector<float> anc(lc.size());
  DevBuf *d_lc, *d_ls;
  CSM_TRY(x.ctx->Reserve("m3_tie_c", sizeof(List3) * lc.size(), &d_lc));
  CSM_TRY(x.ctx->Reserve("m3_tie_s", sizeof(float) * lc.size(), &d_ls));
  CSM_CUDA(cudaMemcpyAsync(d_lc->p, lc.data(), sizeof(List3) * lc.size(),
                           cudaMemcpyHostToDevice, s));
  k3_score_list<<<static_cast<int>(lc.size()), kT3, 0, s>>>(jb, d_lc->as<List3>(),
                                                             d_ls->as<float>(), nullptr);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(anc.data(), d_ls->p, sizeof(float) * lc.size(),
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  ++x.host_syncs;
  const long long total_top = x.per_scan * x.hp[kC3Scans];
  std::vector<int> top_rank;
  auto ensure_top_rank = [&]() -> csm_status {
    if (!top_rank.empty()) return CSM_OK;
    ++*host_resolves;
    std::vector<int> sums(total_top);
    CSM_CUDA(cudaMemcpy(sums.data(), x.d_top->p, sizeof(int) * total_top, cudaMemcpyDeviceToHost));
    struct Item { float score; int gen; };
    std::vector<Item> items(total_top);
    for (long long i = 0; i < total_top; ++i)
      items[i] = Item{kMinProbability +
                          (static_cast<float>(sums[i]) / static_cast<float>(x.jb.n_hi)) *
                              ((kMaxProbability - kMinProbability) / 255.f),
                      static_cast<int>(i)};
    std::sort(items.begin(), items.end(),
              [](const Item& a, const Item& b) { return a.score > b.score; });
    top_rank.resize(total_top);
    for (long long r = 0; r < total_top; ++r) top_rank[items[r].gen] = static_cast<int>(r);
    return CSM_OK;
  };
  csm_status err = CSM_OK;
  auto before = [&](int a, int b) -> bool {
    const BestLeaf3& A_ = ties[a];
    const BestLeaf3& B_ = ties[b];
    for (int l = hmax; l >= 0; --l) {
      const int ax = (A_.ox + sp.wxy) >> l, ay = (A_.oy + sp.wxy) >> l, az = (A_.oz + sp.wz) >> l;
      const int bx = (B_.ox + sp.wxy) >> l, by = (B_.oy + sp.wxy) >> l, bz = (B_.oz + sp.wz) >> l;
      if (A_.scan == B_.scan && ax == bx && ay == by && az == bz) continue;
      const float fa = l == 0 ? 0.f : anc[static_cast<size_t>(a) * hmax + (l - 1)];
      const float fb = l == 0 ? 0.f : anc[static_cast<size_t>(b) * hmax + (l - 1)];
      if (l > 0 && fa != fb) return fa > fb;
      if (l == hmax) {
        if (ensure_top_rank() != CSM_OK) { err = CSM_E_CUDA; return false; }
        const long long ga = ((static_cast<long long>(A_.scan) * jb.nzc + az) * jb.nxc + ay) * jb.nxc + ax;
        const long long gb = ((static_cast<long long>(B_.scan) * jb.nzc + bz) * jb.nxc + by) * jb.nxc + bx;
        return top_rank[ga] < top_rank[gb];
      }
      // siblings: generation order z outer, y, x inner
      if ((az & 1) != (bz & 1)) return (az & 1) < (bz & 1);
      if ((ay & 1) != (by & 1)) return (ay & 1) < (by & 1);
      return (ax & 1) < (bx & 1);
    }
    return false;
  };
  int w = 0;
  for (int t = 1; t < T; ++t)
    if (before(t, w)) w = t;
  if (err != CSM_OK) return err;
  std::swap(ties[0], ties[w]);
  return CSM_OK;
}

// The result from the first optimal leaf, and the match's statistics.
void Result3D(const Match3& x, const std::vector<BestLeaf3>& ties, int host_resolves,
              csm_result3d* result, csm_stats* stats) {
  const int S = x.hp[kC3Scans];
  const long long total_top = x.per_scan * S;
  const float best_score = OrderedToFloat(static_cast<unsigned>(x.hp[kC3Bound]));
  result->leaves_tied = static_cast<int32_t>(ties.size());
  if (!ties.empty() && best_score > x.min_score) {
    const BestLeaf3& t = ties[0];
    const Scan3& sc = x.plan.scans[t.angle];
    const float res = x.m->hs.resolution;
    result->found = 1;
    result->score = best_score;
    // GetPoseFromCandidate(...).cast<double>() (:369-375)
    result->pose_estimate[0] = sc.tx + res * static_cast<float>(t.ox);
    result->pose_estimate[1] = sc.ty + res * static_cast<float>(t.oy);
    result->pose_estimate[2] = sc.tz + res * static_cast<float>(t.oz);
    result->pose_estimate[3] = sc.nw;
    result->pose_estimate[4] = sc.nx;
    result->pose_estimate[5] = sc.ny;
    result->pose_estimate[6] = sc.nz;
    result->rotational_score = t.rot;
    result->low_resolution_score = t.low;
    result->best_scan_index = t.scan;
    result->best_offset[0] = t.ox;
    result->best_offset[1] = t.oy;
    result->best_offset[2] = t.oz;
  }
  if (stats) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, x.ctx->ev0, x.ctx->ev1);
    stats->candidates_scored = static_cast<int64_t>(total_top + x.hctr[0]);
    stats->lowest_resolution_candidates = total_top;
    stats->nodes_expanded = static_cast<int64_t>(x.hctr[1]);
    stats->leaves_tied = static_cast<int64_t>(ties.size());
    stats->num_scans = S;
    stats->host_tie_resolves = host_resolves;
    stats->host_syncs = x.host_syncs;
    stats->device_ms = ms;
    if (result->found) {
      stats->best_scan_index = result->best_scan_index;
      stats->best_x_offset = result->best_offset[0];
      stats->best_y_offset = result->best_offset[1];
    }
  }
}

// One match = one stream of launches + one synchronisation.  `dev` (optional) carries the
// node's clouds already on the device; `lim` (NULL: the defaults) the sweep limits, already
// validated.  trace (may be NULL) receives {collects, most leaves recorded at a collect,
// optimal leaves}.
csm_status Match3D(Ctx* ctx, const csm_matcher3d* m, const csm_node3d* node,
                   const NodeDev3* dev, const double node_pose[7], const double submap_pose[7],
                   int full, float min_score, csm_result3d* result, csm_stats* stats,
                   const csm_sweep_limits3d* lim = nullptr, int32_t trace[3] = nullptr) {
  Match3 x;
  if (lim) {
    x.chunk = lim->chunk;
    x.leaf_cap = lim->leaf_cap;
    x.inline_best = lim->inline_best;
    x.dive_ratio = lim->dive_ratio;
  }
  CSM_TRY(Plan3D(x, ctx, m, node, dev, node_pose, submap_pose, full, min_score));
  std::memset(result, 0, sizeof(*result));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  CSM_TRY(RequireMatchable3D(x));
  CSM_TRY(Upload3D(x));
  CSM_TRY(Discretize3D(x));
  CSM_TRY(TopDive3D(x));
  CSM_TRY(FilterTop3D(x, x.max_top));
  CSM_TRY(Sweep3D(x));
  const int n_best = x.hp[kC3Best];
  if (trace) {
    trace[0] = x.collects;
    trace[1] = x.max_leaves;
    trace[2] = n_best;
  }
  std::vector<BestLeaf3> ties(x.best_inline, x.best_inline + std::min(n_best, x.inline_best));
  if (n_best > x.inline_best) {
    ties.resize(n_best);
    CSM_CUDA(cudaMemcpy(ties.data(), x.d_best->p, sizeof(BestLeaf3) * n_best, cudaMemcpyDeviceToHost));
    ++x.host_syncs;
  }
  int host_resolves = 0;
  if (ties.size() > 1) CSM_TRY(ResolveTies3D(x, ties, &host_resolves));
  Result3D(x, ties, host_resolves, result, stats);
  return CSM_OK;
}

// A test-hook call on a lane.  One that fails after a launch waits for it before the lane
// goes back, as every call that succeeds does.
struct Hook3D {
  LaneGuard guard;
  Match3 x;
  ~Hook3D() { if (guard.lane) cudaStreamSynchronize(guard.lane->stream); }
};

// The start of a test-hook call: the match csm_match3d would run with the same arguments,
// planned, uploaded and discretised on a lane.
csm_status StartHook3D(Hook3D& hk, const csm_matcher3d* m,
                       const csm_node3d* node, const double node_pose[7],
                       const double submap_pose[7], int32_t full, float min_score) {
  CSM_REQUIRE(m && node && node_pose && submap_pose, "null pointer");
  CSM_REQUIRE(node->num_high >= 1 && node->high_resolution_point_cloud, "high-resolution cloud");
  CSM_REQUIRE(node->num_low >= 0 && (node->num_low == 0 || node->low_resolution_point_cloud),
              "low-resolution cloud");
  CSM_TRY(AcquireLane(m->ctx->device, &hk.guard));
  Match3& x = hk.x;
  CSM_TRY(Plan3D(x, hk.guard.lane, m, node, nullptr, node_pose, submap_pose, full, min_score));
  CSM_TRY(RequireMatchable3D(x));
  CSM_TRY(Upload3D(x));
  return Discretize3D(x);
}

}  // namespace

extern "C" {

csm_status csm_match3d(const csm_matcher3d* m, const csm_node3d* node, const double node_pose[7],
                       const double submap_pose[7], int32_t full, float min_score,
                       csm_result3d* result, csm_stats* stats) {
  CSM_REQUIRE(m && node && node_pose && submap_pose && result, "null pointer");
  CSM_REQUIRE(node->num_high >= 1 && node->high_resolution_point_cloud, "high-resolution cloud");
  CSM_REQUIRE(node->num_low >= 0 && (node->num_low == 0 || node->low_resolution_point_cloud),
              "low-resolution cloud");
  LaneGuard guard;
  CSM_TRY(AcquireLane(m->ctx->device, &guard));
  return Match3D(guard.lane, m, node, nullptr, node_pose, submap_pose, full, min_score, result,
                 stats);
}
void csm_sweep_limits3d_default(csm_sweep_limits3d* out) {
  if (!out) return;
  out->chunk = kChunk;
  out->leaf_cap = kLeafCap;
  out->inline_best = kInlineBest;
  out->dive_ratio = kDiveRatio;
}

csm_status csm_match3d_batch(const csm_matcher3d* const* matchers, int32_t num_matchers,
                             const csm_node3d* nodes, int32_t num_nodes, const csm_job3d* jobs,
                             int32_t num_jobs, int32_t max_concurrency, csm_result3d* results,
                             csm_stats* stats) {
  return csm_match3d_batch_limits(matchers, num_matchers, nodes, num_nodes, jobs, num_jobs,
                                  max_concurrency, nullptr, results, stats, nullptr);
}

csm_status csm_match3d_batch_limits(const csm_matcher3d* const* matchers, int32_t num_matchers,
                                    const csm_node3d* nodes, int32_t num_nodes,
                                    const csm_job3d* jobs, int32_t num_jobs,
                                    int32_t max_concurrency, const csm_sweep_limits3d* limits,
                                    csm_result3d* results, csm_stats* stats, int32_t trace[3]) {
  csm_sweep_limits3d lim;
  csm_sweep_limits3d_default(&lim);
  if (limits) {
    lim = *limits;
    CSM_REQUIRE(lim.chunk >= 1 && lim.chunk <= kChunk, "limits: chunk");
    CSM_REQUIRE(lim.leaf_cap >= 1 && lim.leaf_cap <= kLeafCap, "limits: leaf_cap");
    CSM_REQUIRE(lim.inline_best >= 0 && lim.inline_best <= kInlineBest, "limits: inline_best");
    CSM_REQUIRE(std::isfinite(lim.dive_ratio) && lim.dive_ratio >= 0.f, "limits: dive_ratio");
  }
  CSM_REQUIRE(num_jobs >= 0 && num_matchers >= 0 && num_nodes >= 0, "negative count");
  if (stats) std::memset(stats, 0, sizeof(*stats));
  if (trace) std::memset(trace, 0, sizeof(int32_t) * 3);
  if (num_jobs == 0) return CSM_OK;
  CSM_REQUIRE(matchers && nodes && jobs && results, "null pointer");
  int device = -1;
  std::vector<char> used(num_nodes, 0);
  for (int j = 0; j < num_jobs; ++j) {
    CSM_REQUIRE(jobs[j].matcher_index >= 0 && jobs[j].matcher_index < num_matchers &&
                    matchers[jobs[j].matcher_index] != nullptr,
                "matcher_index out of range");
    CSM_REQUIRE(jobs[j].node_index >= 0 && jobs[j].node_index < num_nodes,
                "node_index out of range");
    const csm_node3d& nd = nodes[jobs[j].node_index];
    CSM_REQUIRE(nd.num_high >= 1 && nd.high_resolution_point_cloud, "high-resolution cloud");
    CSM_REQUIRE(nd.num_low >= 0 && (nd.num_low == 0 || nd.low_resolution_point_cloud),
                "low-resolution cloud");
    used[jobs[j].node_index] = 1;
    const int dv = matchers[jobs[j].matcher_index]->ctx->device;
    CSM_REQUIRE(device < 0 || device == dv, "all matchers of a batch must share one device");
    device = dv;
  }
  // The queue matches every node against many submaps: its clouds and histogram go to the
  // device ONCE per call (one allocation, one staged copy), not once per job.
  CSM_CUDA(cudaSetDevice(device));
  std::vector<NodeDev3> ndev(num_nodes);
  std::vector<size_t> off_hi(num_nodes, 0), off_lo(num_nodes, 0), off_h(num_nodes, 0);
  size_t bytes = 0;
  for (int i = 0; i < num_nodes; ++i) {
    if (!used[i]) continue;
    off_hi[i] = bytes; bytes += (12 * static_cast<size_t>(nodes[i].num_high) + 255) / 256 * 256;
    off_lo[i] = bytes; bytes += (12 * static_cast<size_t>(std::max(1, nodes[i].num_low)) + 255) / 256 * 256;
    off_h[i] = bytes; bytes += (4 * static_cast<size_t>(std::max(1, nodes[i].histogram_size)) + 255) / 256 * 256;
  }
  char* d_nodes = nullptr;
  char* h_nodes = nullptr;
  CSM_CUDA(cudaMalloc(&d_nodes, std::max<size_t>(bytes, 256)));
  struct Free {
    char* d; char* h;
    ~Free() { cudaFree(d); cudaFreeHost(h); }
  } guard_free{d_nodes, nullptr};
  CSM_CUDA(cudaMallocHost(&h_nodes, std::max<size_t>(bytes, 256)));
  guard_free.h = h_nodes;
  for (int i = 0; i < num_nodes; ++i) {
    if (!used[i]) continue;
    std::memcpy(h_nodes + off_hi[i], nodes[i].high_resolution_point_cloud, 12 * static_cast<size_t>(nodes[i].num_high));
    if (nodes[i].num_low)
      std::memcpy(h_nodes + off_lo[i], nodes[i].low_resolution_point_cloud, 12 * static_cast<size_t>(nodes[i].num_low));
    if (nodes[i].histogram_size)
      std::memcpy(h_nodes + off_h[i], nodes[i].rotational_scan_matcher_histogram, 4 * static_cast<size_t>(nodes[i].histogram_size));
    ndev[i].hi = reinterpret_cast<const float*>(d_nodes + off_hi[i]);
    ndev[i].lo = reinterpret_cast<const float*>(d_nodes + off_lo[i]);
    ndev[i].hist = reinterpret_cast<const float*>(d_nodes + off_h[i]);
    ndev[i].max_range = MaxRange3(&nodes[i]);
  }
  CSM_CUDA(cudaMemcpy(d_nodes, h_nodes, std::max<size_t>(bytes, 256), cudaMemcpyHostToDevice));
  // Worker threads stand in for the reference's pool threads: every match borrows its own
  // lane (stream + workspace), so the matches overlap on the device.
  const int workers = std::max(1, std::min(num_jobs, max_concurrency > 0 ? max_concurrency : 8));
  std::atomic<int> next{0};
  std::atomic<int> failed{0};
  std::mutex mu;
  std::string first_error;
  csm_status first_status = CSM_OK;
  csm_stats total;
  std::memset(&total, 0, sizeof(total));
  auto work = [&]() {
    for (;;) {
      const int j = next.fetch_add(1);
      if (j >= num_jobs || failed.load()) return;
      const csm_job3d& jb = jobs[j];
      csm_stats st;
      std::memset(&st, 0, sizeof(st));
      int32_t tr[3] = {0, 0, 0};
      csm_status rc;
      {
        LaneGuard guard;
        rc = AcquireLane(device, &guard);
        if (rc == CSM_OK)
          rc = Match3D(guard.lane, matchers[jb.matcher_index], &nodes[jb.node_index],
                       &ndev[jb.node_index], jb.global_node_pose, jb.global_submap_pose,
                       jb.full_submap, jb.min_score, &results[j], &st, &lim, tr);
      }
      std::lock_guard<std::mutex> lock(mu);
      if (rc != CSM_OK) {
        if (!failed.exchange(1)) {
          first_status = rc;
          first_error = csm_last_error_string();  // this worker's thread-local message
        }
        return;
      }
      total.candidates_scored += st.candidates_scored;
      total.lowest_resolution_candidates += st.lowest_resolution_candidates;
      total.nodes_expanded += st.nodes_expanded;
      total.num_scans += st.num_scans;
      total.host_tie_resolves += st.host_tie_resolves;
      total.host_syncs += st.host_syncs;
      total.device_ms += st.device_ms;
      if (trace) {
        trace[0] += tr[0];
        trace[1] = std::max(trace[1], tr[1]);
        trace[2] += tr[2];
      }
    }
  };
  std::vector<std::thread> pool;
  for (int w = 1; w < workers; ++w) pool.emplace_back(work);
  work();
  for (std::thread& t : pool) t.join();
  if (failed.load()) {
    SetError("%s", first_error.c_str());
    return first_status;
  }
  if (stats) *stats = total;
  return CSM_OK;
}

csm_status csm_discretize3d(const csm_matcher3d* m, const csm_node3d* node,
                            const double node_pose[7], const double submap_pose[7], int32_t full,
                            int32_t* num_scans, int32_t* cells, float* poses, float* rot) {
  CSM_REQUIRE(m && node && node_pose && submap_pose && num_scans, "null pointer");
  CSM_REQUIRE(node->num_high >= 1 && node->high_resolution_point_cloud, "high-resolution cloud");
  Hook3D hk;
  CSM_TRY(AcquireLane(m->ctx->device, &hk.guard));
  Match3& x = hk.x;
  CSM_TRY(Plan3D(x, hk.guard.lane, m, node, nullptr, node_pose, submap_pose, full, 0.f));
  CSM_TRY(Upload3D(x));
  CSM_TRY(Discretize3D(x));
  CSM_TRY(ReadCtl3D(x));
  const int S = x.hp[kC3Scans];
  *num_scans = S;
  if (S == 0 || !cells) return CSM_OK;
  std::vector<short4> h(static_cast<size_t>(S) * x.jb.n_hi);
  std::vector<Scan3> hs(S);
  CSM_CUDA(cudaMemcpy(h.data(), x.d_cells->p, sizeof(short4) * h.size(), cudaMemcpyDeviceToHost));
  CSM_CUDA(cudaMemcpy(hs.data(), x.d_scans->p, sizeof(Scan3) * S, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < h.size(); ++i) {
    cells[3 * i] = h[i].x;
    cells[3 * i + 1] = h[i].y;
    cells[3 * i + 2] = h[i].z;
  }
  for (int k = 0; k < S; ++k) {
    const Scan3& sc = hs[k];
    const float v[7] = {sc.tx, sc.ty, sc.tz, sc.qw, sc.qx, sc.qy, sc.qz};
    if (poses) std::memcpy(poses + 7 * k, v, sizeof(v));
    if (rot) rot[k] = sc.rot_score;
  }
  return CSM_OK;
}

csm_status csm_score_candidates3d(const csm_matcher3d* m, const csm_node3d* node,
                                  const double node_pose[7], const double submap_pose[7],
                                  int32_t full_submap, const csm_candidate3d* candidates,
                                  int32_t num_candidates, int32_t* sums, float* scores) {
  static_assert(sizeof(csm_candidate3d) == sizeof(List3), "csm_candidate3d is List3");
  CSM_REQUIRE(sums && scores && (candidates || num_candidates == 0) && num_candidates >= 0,
              "candidates");
  Hook3D hk;
  Match3& x = hk.x;
  CSM_TRY(StartHook3D(hk, m, node, node_pose, submap_pose, full_submap, 0.f));
  CSM_TRY(ReadCtl3D(x));
  const int S = x.hp[kC3Scans];
  const List3* list = reinterpret_cast<const List3*>(candidates);
  const int n = num_candidates;
  for (int i = 0; i < n; ++i) {
    CSM_REQUIRE(list[i].scan >= 0 && list[i].scan < S, "candidate scan_index");
    CSM_REQUIRE(list[i].depth >= 0 && list[i].depth <= x.hmax, "candidate depth");
  }
  if (n == 0) return CSM_OK;
  cudaStream_t s = x.s;
  DevBuf *d_lc, *d_ls, *d_li;
  CSM_TRY(x.ctx->Reserve("m3_tie_c", sizeof(List3) * n, &d_lc));
  CSM_TRY(x.ctx->Reserve("m3_tie_s", sizeof(float) * n, &d_ls));
  CSM_TRY(x.ctx->Reserve("m3_probe_sums", sizeof(int) * n, &d_li));
  CSM_CUDA(cudaMemcpyAsync(d_lc->p, list, sizeof(List3) * n, cudaMemcpyHostToDevice, s));
  ProfBegin(x.ctx);
  k3_score_list<<<n, kT3, 0, s>>>(x.jb, d_lc->as<List3>(), d_ls->as<float>(), d_li->as<int>());
  CSM_LAUNCH_CHECK();
  ProfEnd(x.ctx, "k3_score_list", n);
  CSM_CUDA(cudaMemcpyAsync(scores, d_ls->p, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(sums, d_li->p, sizeof(int) * n, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

csm_status csm_score_top3d(const csm_matcher3d* m, const csm_node3d* node,
                           const double node_pose[7], const double submap_pose[7],
                           int32_t full_submap, float min_score, int32_t* num_scans,
                           int32_t lattice[2], int32_t* angle_index, float* rotational_scores,
                           int32_t* sums, int32_t* top_best, float* bound, int64_t counters[2]) {
  CSM_REQUIRE(num_scans && lattice, "null pointer");
  Hook3D hk;
  Match3& x = hk.x;
  CSM_TRY(StartHook3D(hk, m, node, node_pose, submap_pose, full_submap, min_score));
  CSM_TRY(TopDive3D(x));
  unsigned long long c[8];
  CSM_CUDA(cudaMemcpyAsync(c, x.ctr, sizeof(c), cudaMemcpyDeviceToHost, x.s));
  CSM_TRY(ReadCtl3D(x));
  const int S = x.hp[kC3Scans];
  *num_scans = S;
  lattice[0] = x.jb.nxc;
  lattice[1] = x.jb.nzc;
  if (S && angle_index)
    CSM_CUDA(cudaMemcpy(angle_index, x.d_sel->p, sizeof(int) * S, cudaMemcpyDeviceToHost));
  if (S && rotational_scores) {
    std::vector<Scan3> hs(S);
    CSM_CUDA(cudaMemcpy(hs.data(), x.d_scans->p, sizeof(Scan3) * S, cudaMemcpyDeviceToHost));
    for (int k = 0; k < S; ++k) rotational_scores[k] = hs[k].rot_score;
  }
  if (S && sums)
    CSM_CUDA(cudaMemcpy(sums, x.d_top->p, sizeof(int) * x.per_scan * S, cudaMemcpyDeviceToHost));
  if (top_best) *top_best = x.hp[kC3TopBest];
  if (bound) *bound = OrderedToFloat(static_cast<unsigned>(x.hp[kC3Bound]));
  if (counters) {
    counters[0] = static_cast<int64_t>(c[0]);
    counters[1] = static_cast<int64_t>(c[2]);
  }
  return CSM_OK;
}

csm_status csm_top_queue3d(const csm_matcher3d* m, const csm_node3d* node,
                           const double node_pose[7], const double submap_pose[7],
                           int32_t full_submap, float min_score, float dive_ratio, float* bound,
                           csm_bnb_node3d* queue, int32_t capacity, int32_t* count) {
  static_assert(sizeof(csm_bnb_node3d) == sizeof(Node3), "csm_bnb_node3d is Node3");
  CSM_REQUIRE(bound && count, "null pointer");
  CSM_REQUIRE(capacity >= 0, "capacity");
  CSM_REQUIRE(queue || capacity == 0, "null queue");
  CSM_REQUIRE(std::isfinite(dive_ratio) && dive_ratio >= 0.f, "dive_ratio");
  Hook3D hk;
  Match3& x = hk.x;
  x.dive_ratio = dive_ratio;
  CSM_TRY(StartHook3D(hk, m, node, node_pose, submap_pose, full_submap, min_score));
  CSM_TRY(TopDive3D(x));
  CSM_TRY(FilterTop3D(x, x.max_top));
  CSM_TRY(ReadCtl3D(x));
  const int n = x.hp[x.hmax];
  const int copy = std::min(n, capacity);
  if (copy > 0)
    CSM_CUDA(cudaMemcpy(queue, x.Queue(x.hmax), sizeof(Node3) * copy, cudaMemcpyDeviceToHost));
  *bound = OrderedToFloat(static_cast<unsigned>(x.hp[kC3Bound]));
  *count = n;
  return CSM_OK;
}

csm_status csm_branch_step3d(const csm_matcher3d* m, const csm_node3d* node,
                             const double node_pose[7], const double submap_pose[7],
                             int32_t full_submap, float min_score, int32_t level,
                             const csm_bnb_node3d* parents, int32_t num_parents, float bound,
                             csm_bnb_node3d* children, csm_bnb_leaf3d* leaves, int32_t* num_out,
                             float* final_bound, int64_t counters[3]) {
  static_assert(sizeof(csm_bnb_node3d) == sizeof(Node3), "csm_bnb_node3d is Node3");
  static_assert(sizeof(csm_bnb_leaf3d) == sizeof(Leaf3), "csm_bnb_leaf3d is Leaf3");
  CSM_REQUIRE(num_out && final_bound && counters, "null pointer");
  CSM_REQUIRE(num_parents >= 0 && (parents || num_parents == 0), "parents");
  CSM_REQUIRE(level >= 2 ? children != nullptr : leaves != nullptr, "output records");
  Hook3D hk;
  Match3& x = hk.x;
  CSM_TRY(StartHook3D(hk, m, node, node_pose, submap_pose, full_submap, min_score));
  cudaStream_t s = x.s;
  CSM_TRY(TopDive3D(x));
  CSM_TRY(FilterTop3D(x, std::max<long long>(x.max_top, num_parents)));
  // the level loop over the caller's parents only: its state is reset to them
  const int h = level, n = num_parents;
  CSM_REQUIRE(h >= 1 && h <= x.hmax, "level out of range");
  CSM_REQUIRE(h == x.hmax || n <= kQueueCap, "number of parents");
  CSM_TRY(ReadCtl3D(x));
  const int S = x.hp[kC3Scans];
  const Node3* ps = reinterpret_cast<const Node3*>(parents);
  const HostSearch3& sp = x.sp;
  for (int i = 0; i < n; ++i) {
    const Node3& p = ps[i];
    CSM_REQUIRE(p.scan >= 0 && p.scan < S, "parent scan_index");
    const int dx = p.ox + sp.wxy, dy = p.oy + sp.wxy, dz = p.oz + sp.wz;
    CSM_REQUIRE(dx >= 0 && dy >= 0 && dz >= 0 && ((dx | dy | dz) & ((1 << h) - 1)) == 0 &&
                    p.ox <= sp.wxy && p.oy <= sp.wxy && p.oz <= sp.wz,
                "parent is not a node of its level's lattice");
  }
  int* hp = x.hp;
  for (int l = 1; l <= x.hmax; ++l) hp[l] = 0;
  hp[h] = n;
  hp[kC3Leaf] = 0;
  hp[kC3Overflow] = 0;
  hp[kC3Bound] = static_cast<int>(FloatToOrdered(bound));
  CSM_CUDA(cudaMemcpyAsync(x.ictr, hp, kRbCtr, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemsetAsync(x.ctr, 0, 8 * 8, s));
  if (n) CSM_CUDA(cudaMemcpyAsync(x.Queue(h), ps, sizeof(Node3) * n, cudaMemcpyHostToDevice, s));
  for (int done = 0; done < n; done += kChunk) CSM_TRY(LevelStep3D(x, h));
  unsigned long long c[8];
  CSM_CUDA(cudaMemcpyAsync(c, x.ctr, sizeof(c), cudaMemcpyDeviceToHost, s));
  CSM_TRY(ReadCtl3D(x));
  if (hp[kC3Overflow]) { SetError("3D branch-and-bound capacity exceeded"); return CSM_E_CAPACITY; }
  *num_out = h >= 2 ? hp[h - 1] : hp[kC3Leaf];
  if (*num_out && h >= 2)
    CSM_CUDA(cudaMemcpy(children, x.Queue(h - 1), sizeof(Node3) * *num_out,
                        cudaMemcpyDeviceToHost));
  if (*num_out && h == 1)
    CSM_CUDA(cudaMemcpy(leaves, x.d_leaves->p, sizeof(Leaf3) * *num_out, cudaMemcpyDeviceToHost));
  *final_bound = OrderedToFloat(static_cast<unsigned>(hp[kC3Bound]));
  for (int k = 0; k < 3; ++k) counters[k] = static_cast<int64_t>(c[k]);
  return CSM_OK;
}

}  // extern "C"
