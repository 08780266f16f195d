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

#include "common.cuh"

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

__device__ __forceinline__ unsigned FloatToOrdered3(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float OrderedToFloat3(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

struct F3 { float x, y, z; };
__device__ __forceinline__ F3 Cross3(const F3& a, const F3& b) {
  return F3{__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
            __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
            __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
// Rigid3f * point: Eigen quaternion rotate, then + translation
// (transform/rigid_transform.h:192-196).
__device__ __forceinline__ F3 Apply3(float qw, const F3& qv, const F3& t, const F3& v) {
  F3 uv = Cross3(qv, v);
  uv.x = __fadd_rn(uv.x, uv.x);
  uv.y = __fadd_rn(uv.y, uv.y);
  uv.z = __fadd_rn(uv.z, uv.z);
  const F3 c = Cross3(qv, uv);
  return F3{__fadd_rn(__fadd_rn(__fadd_rn(v.x, __fmul_rn(qw, uv.x)), c.x), t.x),
            __fadd_rn(__fadd_rn(__fadd_rn(v.y, __fmul_rn(qw, uv.y)), c.y), t.y),
            __fadd_rn(__fadd_rn(__fadd_rn(v.z, __fmul_rn(qw, uv.z)), c.z), t.z)};
}
// HybridGridBase::GetCellIndex (hybrid_grid.h:428-433): lround(p / resolution) in float.
__device__ __forceinline__ int CellOf(float p, float resolution) {
  return static_cast<int>(lroundf(__fdiv_rn(p, resolution)));
}
// PrecomputationGrid3D::ToProbability(sum / float(N))  (precomputation_grid_3d.h:32-35)
__device__ __forceinline__ float ToScore3(int sum, int n) {
  const float kMin = 0.1f;
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
  const F3 qv{sc.qx, sc.qy, sc.qz}, t{sc.tx, sc.ty, sc.tz};
  const float res = jb.stack->resolution;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < jb.n_hi; p += gridDim.x * blockDim.x) {
    const F3 v{jb.hi_xyz[3 * p], jb.hi_xyz[3 * p + 1], jb.hi_xyz[3 * p + 2]};
    const F3 w = Apply3(sc.qw, qv, t, v);
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
  const F3 t{__fadd_rn(sc.tx, __fmul_rn(res, __int2float_rn(ox))),
             __fadd_rn(sc.ty, __fmul_rn(res, __int2float_rn(oy))),
             __fadd_rn(sc.tz, __fmul_rn(res, __int2float_rn(oz)))};
  const F3 qv{sc.nx, sc.ny, sc.nz};
  const Low3Dev& lg = *jb.low;
  __shared__ float s_sum;
  __syncthreads();  // a previous call's readers of s_sum are done
  if (threadIdx.x == 0) s_sum = 0.f;
  for (int p0 = 0; p0 < jb.n_lo; p0 += kT3) {
    const int p = p0 + threadIdx.x;
    if (p < jb.n_lo) {
      const F3 v{jb.lo_xyz[3 * p], jb.lo_xyz[3 * p + 1], jb.lo_xyz[3 * p + 2]};
      const F3 w = Apply3(sc.nw, qv, t, v);
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
      if (static_cast<double>(low) >= jb.min_low_d) atomicMax(lb, FloatToOrdered3(score));
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
  if (!(score > jb.min_score && score >= OrderedToFloat3(*lb))) return;
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
    if (threadIdx.x == 0) s_bound = OrderedToFloat3(*lb);
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
        if (threadIdx.x == 0) s_go = (sc > jb.min_score && sc >= OrderedToFloat3(*lb)) ? 1 : 0;
        __syncthreads();
        if (!s_go) continue;
        const int ox = nd.ox + (t & 1) * half, oy = nd.oy + ((t >> 1) & 1) * half,
                  oz = nd.oz + ((t >> 2) & 1) * half;
        const float low = LowResScore(jb, nd.scan, ox, oy, oz, s_buf);
        if (threadIdx.x == 0) {
          atomicAdd(&counters[2], 1ull);
          if (static_cast<double>(low) >= jb.min_low_d) {
            const unsigned o = FloatToOrdered3(sc);
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
      const float bound = OrderedToFloat3(*lb);
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
    if (FloatToOrdered3(l.score) != bound) continue;
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

// ---- Eigen semantics on the host (see oracle/oracle_3d.h for the provenance) ----
struct Qf { float w, x, y, z; };
struct Vf { float x, y, z; };
Vf HCross(const Vf& a, const Vf& b) {
  return Vf{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
Vf HRot(const Qf& q, const Vf& v) {  // QuaternionBase::_transformVector
  const Vf qv{q.x, q.y, q.z};
  Vf uv = HCross(qv, v);
  uv.x += uv.x; uv.y += uv.y; uv.z += uv.z;
  const Vf c = HCross(qv, uv);
  return Vf{(v.x + q.w * uv.x) + c.x, (v.y + q.w * uv.y) + c.y, (v.z + q.w * uv.z) + c.z};
}
Qf HMul(const Qf& a, const Qf& b) {  // Geometry_SSE.h quat_product<float>
  Qf r;
  r.x = (a.x * b.w - a.z * b.y) + (a.y * b.z + a.w * b.x);
  r.y = (a.y * b.w - a.x * b.z) + (a.z * b.x + a.w * b.y);
  r.z = (a.z * b.w - a.y * b.x) + (a.x * b.y + a.w * b.z);
  r.w = (a.w * b.w - a.x * b.x) + (-(a.z * b.z + a.y * b.y));
  return r;
}
float HSq(const Qf& q) { return (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w); }
Qf HNormalized(const Qf& q) {
  const float z = HSq(q);
  if (z > 0.f) {
    const float n = std::sqrt(z);
    return Qf{q.w / n, q.x / n, q.y / n, q.z / n};
  }
  return q;
}
Qf HConj(const Qf& q) { return Qf{q.w, -q.x, -q.y, -q.z}; }
Qf HInverse(const Qf& q) {
  const float n2 = HSq(q);
  if (n2 > 0.f) return Qf{q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
  return Qf{0.f, 0.f, 0.f, 0.f};
}
struct Rf { Vf t; Qf q; };
Rf RInverse(const Rf& r) {  // rigid_transform.h:148-152
  const Qf rot = HConj(r.q);
  const Vf v = HRot(rot, r.t);
  return Rf{Vf{-v.x, -v.y, -v.z}, rot};
}
Rf RMul(const Rf& a, const Rf& b) {  // rigid_transform.h:181-189
  const Vf v = HRot(a.q, b.t);
  return Rf{Vf{v.x + a.t.x, v.y + a.t.y, v.z + a.t.z}, HNormalized(HMul(a.q, b.q))};
}
float HYaw(const Qf& q) {  // transform/transform.h:42-47
  const Vf d = HRot(q, Vf{1.f, 0.f, 0.f});
  return std::atan2(d.y, d.x);
}
Qf HAngleAxisZ(float angle) {  // transform/transform.h:85-99 with (0, 0, angle)
  float scale = 0.5f, w = 1.f;
  const float sq = 0.f * 0.f + 0.f * 0.f + angle * angle;
  if (sq > 1e-8) {
    const float norm = std::sqrt(sq);
    scale = static_cast<float>(std::sin(norm / 2.) / norm);
    w = static_cast<float>(std::cos(norm / 2.));
  }
  return Qf{w, scale * 0.f, scale * 0.f, scale * angle};
}

struct HostSearch3 {
  int wxy, wz;
  double angular;
  Rf node, submap;
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

}  // namespace

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
  CSM_REQUIRE(options->branch_and_bound_depth >= 1 &&
              options->branch_and_bound_depth <= kMaxDepth3, "branch_and_bound_depth");  // :60
  CSM_REQUIRE(options->full_resolution_depth >= 1, "full_resolution_depth");            // :61
  CSM_REQUIRE(hist_n >= 0 && (hist_n == 0 || submap_hist), "histogram");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  cudaStream_t s = ctx->stream;
  std::unique_ptr<csm_matcher3d> m(new csm_matcher3d);
  m->ctx = ctx;
  m->opt = *options;
  m->hist.assign(submap_hist, submap_hist + hist_n);

  auto bbox = [](const int32_t* idx, int64_t n, int lo[3], int hi[3]) {
    for (int a = 0; a < 3; ++a) { lo[a] = INT_MAX; hi[a] = INT_MIN; }
    for (int64_t i = 0; i < n; ++i)
      for (int a = 0; a < 3; ++a) {
        lo[a] = std::min(lo[a], idx[3 * i + a]);
        hi[a] = std::max(hi[a], idx[3 * i + a]);
      }
    if (n == 0)
      for (int a = 0; a < 3; ++a) { lo[a] = 0; hi[a] = 0; }
  };
  int lo0[3], hi0[3];
  bbox(hi_idx, hi_n, lo0, hi0);
  for (int a = 0; a < 3; ++a)
    CSM_REQUIRE(lo0[a] >= -8192 && hi0[a] < 8192, "voxel index outside the 2^14 cube");  // :387
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
    const float kMin = 0.1f, kMax = 1.f - kMin;
    const float kScale = (kMax - kMin) / 32766.f;
    for (int v = 0; v < 65536; ++v) {
      const uint16_t value = static_cast<uint16_t>(v) & 0x7fff;
      const float p = value == 0 ? kMin : value * kScale + (kMin - kScale);
      const long q = std::lround((p - kMin) * (255.f / (kMax - kMin)));
      lut[v] = static_cast<uint8_t>(q < 0 ? 0 : (q > 255 ? 255 : q));
    }
  }
  DevBuf& d_idx = ctx->D("m3_idx");
  DevBuf& d_val = ctx->D("m3_val");
  DevBuf& d_lut = ctx->D("m3_lut");
  CSM_TRY(d_lut.Reserve(65536));
  CSM_CUDA(cudaMemcpyAsync(d_lut.p, lut.data(), 65536, cudaMemcpyHostToDevice, s));
  if (hi_n > 0) {
    CSM_TRY(d_idx.Reserve(sizeof(int) * 3 * hi_n));
    CSM_TRY(d_val.Reserve(sizeof(uint16_t) * hi_n));
    CSM_CUDA(cudaMemcpyAsync(d_idx.p, hi_idx, sizeof(int) * 3 * hi_n, cudaMemcpyHostToDevice, s));
    CSM_CUDA(cudaMemcpyAsync(d_val.p, hi_val, sizeof(uint16_t) * hi_n, cudaMemcpyHostToDevice, s));
    k3_scatter_u8<<<DivUp(hi_n, 256), 256, 0, s>>>(d_idx.as<int>(), d_val.as<uint16_t>(), hi_n,
                                                    d_lut.as<uint8_t>(), hs.level[0],
                                                    m->d_levels + off[0]);
    CSM_LAUNCH_CHECK();
  }
  for (int d = 1; d < hs.depth; ++d) {
    k3_precompute<<<ctx->sm_count * 16, 256, 0, s>>>(hs.level[d - 1], hs.level[d],
                                                     m->d_levels + off[d], shifts[d], halfs[d]);
    CSM_LAUNCH_CHECK();
  }
  CSM_CUDA(cudaStreamSynchronize(s));  // d_idx / d_val are reused below

  // ---- low-resolution grid ----
  Low3Dev& hl = m->hl;
  std::memset(&hl, 0, sizeof(hl));
  int llo[3], lhi[3];
  bbox(lo_idx, lo_n, llo, lhi);
  for (int a = 0; a < 3; ++a) {
    hl.lo[a] = llo[a];
    hl.n[a] = lhi[a] - llo[a] + 1;
  }
  const size_t lvox = static_cast<size_t>(hl.n[0]) * hl.n[1] * hl.n[2];
  CSM_REQUIRE(lvox < (size_t(4) << 30), "dense low-resolution volume too large");
  CSM_CUDA(cudaMalloc(&m->d_lowvol, std::max<size_t>(lvox * 2, 256)));
  CSM_CUDA(cudaMemsetAsync(m->d_lowvol, 0, std::max<size_t>(lvox * 2, 256), s));
  hl.p = m->d_lowvol;
  hl.resolution = lo_res;
  {
    const float kMin = 0.1f, kMax = 1.f - kMin;
    hl.k_scale = (kMax - kMin) / 32766.f;
    hl.bias = kMin - hl.k_scale;
    hl.min_probability = kMin;
  }
  if (lo_n > 0) {
    CSM_TRY(d_idx.Reserve(sizeof(int) * 3 * lo_n));
    CSM_TRY(d_val.Reserve(sizeof(uint16_t) * lo_n));
    CSM_CUDA(cudaMemcpyAsync(d_idx.p, lo_idx, sizeof(int) * 3 * lo_n, cudaMemcpyHostToDevice, s));
    CSM_CUDA(cudaMemcpyAsync(d_val.p, lo_val, sizeof(uint16_t) * lo_n, cudaMemcpyHostToDevice, s));
    k3_scatter_u16<<<DivUp(lo_n, 256), 256, 0, s>>>(d_idx.as<int>(), d_val.as<uint16_t>(), lo_n,
                                                     hl, m->d_lowvol);
    CSM_LAUNCH_CHECK();
  }
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
  const Rf node_to_submap = RMul(RInverse(sp.submap), sp.node);
  // gravity_alignment.inverse().cast<float>()
  const double* g = node->gravity_alignment;
  const double n2 = (g[1] * g[1] + g[3] * g[3]) + (g[2] * g[2] + g[0] * g[0]);
  Qf ginv{0.f, 0.f, 0.f, 0.f};
  if (n2 > 0.)
    ginv = Qf{static_cast<float>(g[0] / n2), static_cast<float>(-g[1] / n2),
              static_cast<float>(-g[2] / n2), static_cast<float>(-g[3] / n2)};
  *initial_angle = HYaw(HMul(node_to_submap.q, ginv));
  CSM_REQUIRE(node->histogram_size == static_cast<int>(m->hist.size()), "histogram sizes differ");
  plan->scans.clear();
  plan->scans.reserve(plan->num_angles);
  const Qf sub_inv = HInverse(sp.submap.q);
  for (int i = 0; i < plan->num_angles; ++i) {
    const Qf q = HMul(HMul(sub_inv, HAngleAxisZ(plan->angles[i])), sp.node.q);
    // GetPoseFromCandidate's rotation: (identity * q).normalized()
    const Qf nq = HNormalized(HMul(Qf{1.f, 0.f, 0.f, 0.f}, q));
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
    Rf r;
    r.t = rotation_only ? Vf{0.f, 0.f, 0.f}
                        : Vf{static_cast<float>(p[0]), static_cast<float>(p[1]),
                             static_cast<float>(p[2])};
    r.q = Qf{static_cast<float>(p[3]), static_cast<float>(p[4]), static_cast<float>(p[5]),
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
                                     x.d_sel->as<int>(), x.ictr, HostFloatToOrdered(x.min_score));
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
  k3_dive<<<x.plan.num_angles, kT3, 0, x.s>>>(x.jb, x.d_top->as<int>(), kDiveRatio, x.lb, x.ctr);
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
  k3_level_begin<<<1, 32, 0, x.s>>>(x.ictr, h, kChunk);
  CSM_LAUNCH_CHECK();
  ProfBegin(x.ctx);
  k3_expand<<<x.ctx->sm_count * 4, kT3, 0, x.s>>>(x.jb, x.Queue(h), x.ictr, h,
                                                   h - 1 >= 1 ? x.Queue(h - 1) : nullptr,
                                                   x.ictr + (h - 1 >= 1 ? h - 1 : 23), kQueueCap,
                                                   x.d_leaves->as<Leaf3>(), kLeafCap, x.ctr);
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
                                             x.d_sel->as<int>(), x.ictr, kLeafCap,
                                             x.d_best->as<BestLeaf3>(), kLeafCap);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaEventRecord(x.ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(pin, x.ictr, kRbCtr, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(pin + kRbCtr, x.ctr, 8 * 8, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(pin + kRbBest, x.d_best->p, sizeof(BestLeaf3) * kInlineBest,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  ++x.host_syncs;
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
    const float kMin = 0.1f, kMax = 1.f - kMin;
    for (long long i = 0; i < total_top; ++i)
      items[i] = Item{kMin + (static_cast<float>(sums[i]) / static_cast<float>(x.jb.n_hi)) *
                                 ((kMax - kMin) / 255.f),
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
  const float best_score = HostOrderedToFloat(static_cast<unsigned>(x.hp[kC3Bound]));
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
// node's clouds already on the device.
csm_status Match3D(Ctx* ctx, const csm_matcher3d* m, const csm_node3d* node,
                   const NodeDev3* dev, const double node_pose[7], const double submap_pose[7],
                   int full, float min_score, csm_result3d* result, csm_stats* stats) {
  Match3 x;
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
  std::vector<BestLeaf3> ties(x.best_inline, x.best_inline + std::min(n_best, kInlineBest));
  if (n_best > kInlineBest) {
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
csm_status csm_match3d_batch(const csm_matcher3d* const* matchers, int32_t num_matchers,
                             const csm_node3d* nodes, int32_t num_nodes, const csm_job3d* jobs,
                             int32_t num_jobs, int32_t max_concurrency, csm_result3d* results,
                             csm_stats* stats) {
  CSM_REQUIRE(num_jobs >= 0 && num_matchers >= 0 && num_nodes >= 0, "negative count");
  if (stats) std::memset(stats, 0, sizeof(*stats));
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
      csm_status rc;
      {
        LaneGuard guard;
        rc = AcquireLane(device, &guard);
        if (rc == CSM_OK)
          rc = Match3D(guard.lane, matchers[jb.matcher_index], &nodes[jb.node_index],
                       &ndev[jb.node_index], jb.global_node_pose, jb.global_submap_pose,
                       jb.full_submap, jb.min_score, &results[j], &st);
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
  if (bound) *bound = HostOrderedToFloat(static_cast<unsigned>(x.hp[kC3Bound]));
  if (counters) {
    counters[0] = static_cast<int64_t>(c[0]);
    counters[1] = static_cast<int64_t>(c[2]);
  }
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
  hp[kC3Bound] = static_cast<int>(HostFloatToOrdered(bound));
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
  *final_bound = HostOrderedToFloat(static_cast<unsigned>(hp[kC3Bound]));
  for (int k = 0; k < 3; ++k) counters[k] = static_cast<int64_t>(c[k]);
  return CSM_OK;
}

}  // extern "C"
