// FastCorrelativeScanMatcher2D on H100: precomputation-grid stack build,
// scan discretisation, candidate scoring and a batched, device-resident
// branch-and-bound.  Reference: cartographer/mapping/internal/2d/scan_matching/
// {correlative_scan_matcher_2d,fast_correlative_scan_matcher_2d}.{h,cc}.
//
// Exactness rules (DESIGN.md §Numerics): every float/double expression whose
// value reaches an output is written with explicit round-to-nearest intrinsics
// (__fmul_rn ...) so ptxas can never contract it into an FMA — the reference
// build has no FMA (cmake/functions.cmake:100-101).  Transcendentals are
// evaluated on the host with libm, like the reference.
#include "engine2d.cuh"
#include "rtgrid.cuh"

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <functional>

namespace csm {

// ---------------------------------------------------------------------------
// Small device helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ unsigned FloatToOrdered(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float OrderedToFloat(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// PrecomputationGrid2D::ToScore(sum / float(N))   (fast...2d.h:74-76, .cc:328-329)
__device__ __forceinline__ float ToScore(const StackDev& st, int sum, int n) {
  const float mean = __fdiv_rn(__int2float_rn(sum), __int2float_rn(n));
  return __fadd_rn(st.min_score, __fmul_rn(mean, st.k255));
}

// PrecomputationGrid2D::GetValue (fast...2d.h:56-71) on the row-major level.
__device__ __forceinline__ int GetValue(const uint8_t* __restrict__ g, int wx, int wy, int lx,
                                        int ly) {
  if (static_cast<unsigned>(lx) >= static_cast<unsigned>(wx) ||
      static_cast<unsigned>(ly) >= static_cast<unsigned>(wy))
    return 0;
  return __ldg(g + static_cast<size_t>(ly) * wx + lx);
}

__device__ __forceinline__ int WarpSum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Word index of lattice cell (X, Y) (both already shifted by +1) of phase `ph` in the
// child-window array of a level (StackDev::win): row-major per phase, so x-neighbours
// share 128-byte lines.
__host__ __device__ __forceinline__ long long WinPhaseWords(int jd, int ids) {
  return static_cast<long long>(jd) * ids;
}
__device__ __forceinline__ int WinCell(int X, int Y, int ids) { return Y * ids + X; }

// ---------------------------------------------------------------------------
// K1: precomputation grid stack
// ---------------------------------------------------------------------------
// Level 0: cells -> uint8 through the 64 Ki LUT
//   lut[v] = ComputeCellValue(1.f - |table[v]|)   (fast...2d.cc:110-111,163-169)
__global__ void k_stack_level0(const uint16_t* __restrict__ cells,
                               const uint8_t* __restrict__ lut, uint8_t* __restrict__ out,
                               int count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) out[i] = lut[cells[i]];
}

// Level h (window w = 2^h) from level h-1 (window w/2): a w x w window is the
// union of four (w/2) x (w/2) windows; max is exact and quantisation is
// monotone, so max-of-uint8 equals the reference's quantised float max
// (fast...2d.cc:108-160).  Coordinates are wide-grid local indices.
__global__ void k_stack_double(const uint8_t* __restrict__ prev, int pwx, int pwy,
                               uint8_t* __restrict__ out, int wx, int wy, int half) {
  int x = blockIdx.x * blockDim.x + threadIdx.x;
  int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= wx || y >= wy) return;
  auto at = [&](int px, int py) -> int {
    return (px >= 0 && py >= 0 && px < pwx && py < pwy) ? prev[static_cast<size_t>(py) * pwx + px]
                                                        : 0;
  };
  int v = max(max(at(x - half, y - half), at(x, y - half)), max(at(x - half, y), at(x, y)));
  out[static_cast<size_t>(y) * wx + x] = static_cast<uint8_t>(v);
}

// Four byte-shifted copies of the decimated lowest-resolution level
// (see StackDev::dec4).
__global__ void k_stack_decimate4(const uint8_t* __restrict__ lvl, int wx, int wy, int h,
                                  uint8_t* __restrict__ dec4, int lpad, int id, int jd,
                                  int ids) {
  const int s = 1 << h;
  const long long total = static_cast<long long>(s) * s * jd * ids;
  const long long n = 4LL * lpad;
  for (long long u = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; u < n;
       u += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(u / lpad);
    const long long t = u % lpad - 16 + k;  // index into D
    uint8_t v = 0;
    if (t >= 0 && t < total) {
      const int I = static_cast<int>(t % ids);
      long long r = t / ids;
      const int J = static_cast<int>(r % jd);
      r /= jd;
      const int ax = static_cast<int>(r % s);
      const int ay = static_cast<int>(r / s);
      const int x = s * I + ax, y = s * J + ay;
      if (I < id && x < wx && y < wy) v = lvl[static_cast<size_t>(y) * wx + x];
    }
    dec4[u] = v;
  }
}

// Child-window layout of parent level h (see StackDev::win): one 32-bit word per
// (phase, lattice cell) with the four children values of level h-1.
__global__ void k_stack_window(const uint8_t* __restrict__ lvl, int wx, int wy, int h,
                               unsigned* __restrict__ win, int jd, int ids) {
  const int S = 1 << h, s = S >> 1;
  const long long per_phase = WinPhaseWords(jd, ids);
  const long long total = static_cast<long long>(S) * S * per_phase;
  for (long long u = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; u < total;
       u += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ph = static_cast<int>(u / per_phase);
    const int c = static_cast<int>(u - ph * per_phase);
    const int X = c % ids, Y = c / ids;
    const int I = X - 1, J = Y - 1;
    const int ax = ph % S, ay = ph / S;
    const int x = S * I + ax, y = S * J + ay;
    auto at = [&](int px, int py) -> unsigned {
      return (px >= 0 && py >= 0 && px < wx && py < wy) ? lvl[static_cast<size_t>(py) * wx + px]
                                                        : 0u;
    };
    unsigned v = 0u;
    if (X < ids && Y < jd)
      v = at(x, y) | (at(x + s, y) << 8) | (at(x, y + s) << 16) | (at(x + s, y + s) << 24);
    win[u] = v;
  }
}

// ---------------------------------------------------------------------------
// K2: GenerateRotatedScans + DiscretizeScans + ShrinkToFit
// ---------------------------------------------------------------------------
struct V3 { float x, y, z; };
__device__ __forceinline__ V3 CrossRn(const V3& a, const V3& b) {
  return V3{__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
            __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
            __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
// Eigen QuaternionBase::_transformVector followed by "+ translation(0)"
// (transform/rigid_transform.h:192-196, sensor/point_cloud.cc:56-64).
__device__ __forceinline__ V3 RotateRn(float qw, const V3& qv, const V3& v) {
  V3 uv = CrossRn(qv, v);
  uv.x = __fadd_rn(uv.x, uv.x);
  uv.y = __fadd_rn(uv.y, uv.y);
  uv.z = __fadd_rn(uv.z, uv.z);
  const V3 c = CrossRn(qv, uv);
  V3 r{__fadd_rn(__fadd_rn(v.x, __fmul_rn(qw, uv.x)), c.x),
       __fadd_rn(__fadd_rn(v.y, __fmul_rn(qw, uv.y)), c.y),
       __fadd_rn(__fadd_rn(v.z, __fmul_rn(qw, uv.z)), c.z)};
  r.x = __fadd_rn(r.x, 0.f);
  r.y = __fadd_rn(r.y, 0.f);
  r.z = __fadd_rn(r.z, 0.f);
  return r;
}

// One CTA per (job, scan) of the scans from scan0 on.  Writes the scan's cell indices and
// its LinearBounds after ShrinkToFit (correlative_scan_matcher_2d.cc:73-127), plus the
// number of lowest-resolution candidates per axis (fast...2d.cc:281-292).
__global__ void __launch_bounds__(128)
k_discretize(const JobDev* __restrict__ jobs, const int* __restrict__ scan_job,
             short2* __restrict__ dscan, ScanInfo* __restrict__ info, int shrink,
             unsigned long long* __restrict__ counters, int scan0) {
  const int sg = scan0 + blockIdx.x;
  const int j = scan_job[sg];
  const JobDev jb = jobs[j];
  const StackDev& st = *jb.stack;
  const int k = sg - jb.scan_base;
  const float2 cs = jb.trig[k];
  // Quaternionf(AngleAxisf(a, UnitZ)): w = cos(ha), vec = sin(ha) * (0, 0, 1)
  const V3 qk{__fmul_rn(cs.y, 0.f), __fmul_rn(cs.y, 0.f), __fmul_rn(cs.y, 1.f)};
  const V3 q0{jb.q0x, jb.q0y, jb.q0z};
  short2* out = dscan + jb.dscan_off + static_cast<long long>(k) * jb.n;
  int min_ix = INT_MAX, max_ix = INT_MIN, min_iy = INT_MAX, max_iy = INT_MIN;
  for (int p = threadIdx.x; p < jb.n; p += blockDim.x) {
    const V3 v{jb.xyz[3 * p], jb.xyz[3 * p + 1], jb.xyz[3 * p + 2]};
    const V3 r0 = RotateRn(jb.q0w, q0, v);   // rotated_point_cloud   (fast...2d.cc:236-239)
    const V3 r1 = RotateRn(cs.x, qk, r0);    // GenerateRotatedScans  (corr...2d.cc:93-109)
    // Affine2f(Translation2f) * v = (1*x + 0*y) + t                    (corr...2d.cc:120-121)
    const float px = __fadd_rn(__fadd_rn(__fmul_rn(1.f, r1.x), __fmul_rn(0.f, r1.y)), jb.tx);
    const float py = __fadd_rn(__fadd_rn(__fmul_rn(0.f, r1.x), __fmul_rn(1.f, r1.y)), jb.ty);
    // MapLimits::GetCellIndex in double                               (2d/map_limits.h:69-76)
    const double fx = __dsub_rn(__ddiv_rn(__dsub_rn(st.max_y, static_cast<double>(py)),
                                          st.resolution), 0.5);
    const double fy = __dsub_rn(__ddiv_rn(__dsub_rn(st.max_x, static_cast<double>(px)),
                                          st.resolution), 0.5);
    const int ix = static_cast<int>(llround(fx));
    const int iy = static_cast<int>(llround(fy));
    // cells are kept as 2 x int16 (grids are < 32 k cells per axis; points farther
    // than 30 k cells from the origin read as 0 for every candidate either way)
    out[p] = make_short2(static_cast<short>(max(-30000, min(30000, ix))),
                         static_cast<short>(max(-30000, min(30000, iy))));
    if (shrink && (abs(ix) > 30000 || abs(iy) > 30000)) counters[7] = 1ull;  // reported as an error
    min_ix = min(min_ix, ix);
    max_ix = max(max_ix, ix);
    min_iy = min(min_iy, iy);
    max_iy = max(max_iy, iy);
  }
  __shared__ int red[4][4];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    min_ix = min(min_ix, __shfl_xor_sync(0xffffffffu, min_ix, o));
    max_ix = max(max_ix, __shfl_xor_sync(0xffffffffu, max_ix, o));
    min_iy = min(min_iy, __shfl_xor_sync(0xffffffffu, min_iy, o));
    max_iy = max(max_iy, __shfl_xor_sync(0xffffffffu, max_iy, o));
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[warp][0] = min_ix;
    red[warp][1] = max_ix;
    red[warp][2] = min_iy;
    red[warp][3] = max_iy;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 4; ++w) {
      red[0][0] = min(red[0][0], red[w][0]);
      red[0][1] = max(red[0][1], red[w][1]);
      red[0][2] = min(red[0][2], red[w][2]);
      red[0][3] = max(red[0][3], red[w][3]);
    }
    ScanInfo si;
    si.job = j;
    si.min_x = -jb.lin;
    si.max_x = jb.lin;
    si.min_y = -jb.lin;
    si.max_y = jb.lin;
    if (shrink) {
      // min_bound = min(0, min(-xy)); max_bound = max(0, max(limits - 1 - xy))
      const int min_bx = min(0, -red[0][1]), max_bx = max(0, st.nx - 1 - red[0][0]);
      const int min_by = min(0, -red[0][3]), max_by = max(0, st.ny - 1 - red[0][2]);
      si.min_x = max(si.min_x, min_bx);
      si.max_x = min(si.max_x, max_bx);
      si.min_y = max(si.min_y, min_by);
      si.max_y = min(si.max_y, max_by);
    }
    const int step = 1 << (st.depth - 1);
    si.nxc = (si.max_x - si.min_x + step) / step;
    si.nyc = (si.max_y - si.min_y + step) / step;
    si.pad = 0;
    if (shrink && (si.nyc > jb.cap_y || static_cast<long long>(si.nxc) * jb.cap_y > jb.cap)) {
      // the host's a-priori slot bound must cover the lattice (reported as an error)
      counters[6] = 1ull;
      si.nxc = si.nyc = 0;
    }
    info[sg] = si;
    const unsigned long long slots = static_cast<unsigned long long>(si.nxc) * si.nyc;
    atomicAdd(&counters[0], slots);  // every lowest-resolution candidate gets scored
    atomicAdd(&counters[3], slots);
  }
}

csm_status LaunchDiscretize2D(cudaStream_t stream, const JobDev* jobs, const int* scan_job,
                              int total_scans, short2* dscan, ScanInfo* info, int shrink,
                              unsigned long long* counters) {
  k_discretize<<<total_scans, 128, 0, stream>>>(jobs, scan_job, dscan, info, shrink, counters, 0);
  CSM_LAUNCH_CHECK();
  return CSM_OK;
}

// ---------------------------------------------------------------------------
// K3: candidate scoring
// ---------------------------------------------------------------------------
// Lowest-resolution pass, gather form: one warp per (scan, slot); slot = i*nyc+j
// follows the reference's generation order (x outer, y inner; fast...2d.cc:296-309).
__global__ void __launch_bounds__(256)
k_score_top_gather(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
                   const short2* __restrict__ dscan, int* __restrict__ top_sum,
                   const long long* __restrict__ scan_slot_base, int total_scans,
                   long long total_slots) {
  const int lane = threadIdx.x & 31;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= total_slots) return;
  // scan = last index with scan_slot_base[scan] <= w
  int lo = 0, hi = total_scans - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (scan_slot_base[mid] <= w) lo = mid; else hi = mid - 1;
  }
  const int sg = lo;
  const int slot = static_cast<int>(w - scan_slot_base[sg]);
  const ScanInfo si = info[sg];
  if (slot >= si.nxc * si.nyc) return;
  const JobDev& jb = jobs[si.job];
  const StackDev& st = *jb.stack;
  const int h = st.depth - 1;
  const int w1 = (1 << h) - 1;
  const uint8_t* __restrict__ g = st.level[h];
  const int wx = st.wx[h], wy = st.wy[h];
  const short2* __restrict__ pts = dscan + jb.dscan_off +
                                 static_cast<long long>(sg - jb.scan_base) * jb.n;
  const int i = slot / si.nyc, jy = slot - i * si.nyc;
  const int ox = si.min_x + (i << h) + w1, oy = si.min_y + (jy << h) + w1;
  int sum = 0;
  for (int p = lane; p < jb.n; p += 32) {
    const short2 c = pts[p];
    sum += GetValue(g, wx, wy, c.x + ox, c.y + oy);
  }
  sum = WarpSum(sum);
  if (lane == 0) top_sum[scan_slot_base[sg] + slot] = sum;
}

// Lowest-resolution pass, small-lattice form (local search windows: a few dozen
// candidates per scan).  `lanes` consecutive lanes of a warp share one scan; a lane
// owns one quad = 4 x-consecutive candidates of one lattice row and fetches their
// cells for a scan point with ONE aligned 32-bit load from the decimated level
// (as k_score_top_dense), so a warp works on 32 / lanes scans at once and nearly
// every lane is busy.  Packed u16 sums are flushed every 256 points.
__global__ void __launch_bounds__(128)
k_score_top_small(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
                  const short2* __restrict__ dscan, int* __restrict__ top_sum,
                  const long long* __restrict__ scan_slot_base, int total_scans, int lanes) {
  extern __shared__ __align__(16) int2 s_small[];  // [warp][scan of the warp][32 points]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int spw = 32 / lanes;                 // scans per warp
  const int sub = lane / lanes, ql = lane - sub * lanes;
  const long long gwarp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long sgl = gwarp * spw + sub;
  const bool has_scan = sub < spw && sgl < total_scans;
  const int sg = has_scan ? static_cast<int>(sgl) : 0;
  const ScanInfo si = info[sg];
  const JobDev& jb = jobs[si.job];
  const StackDev& st = *jb.stack;
  const int h = st.depth - 1;
  const int s1 = (1 << h) - 1;
  const int id = st.dec_id[h], jd = st.dec_jd[h], ids = st.dec_ids[h];
  const unsigned lpad1 = static_cast<unsigned>(st.dec_lpad[h]) - 1u;
  const uint8_t* __restrict__ dec = st.dec4[h] + 16;
  const int qr = (si.nxc + 3) >> 2;
  const bool owns = has_scan && ql < qr * si.nyc;   // this lane scores a quad
  const int jy = ql / qr, i0 = (ql - jy * qr) << 2;
  const int toff = jy * ids + i0;
  const int ox = si.min_x + s1, oy = si.min_y + s1;
  const short2* __restrict__ pts = dscan + jb.dscan_off +
                                 static_cast<long long>(sg - jb.scan_base) * jb.n;
  int2* __restrict__ s_pt = s_small + (warp * spw + (sub < spw ? sub : 0)) * 32;
  // all jobs of a batch have the same point count only per job: the warp walks the
  // longest of its scans, lanes of shorter scans idle
  int n_max = has_scan ? jb.n : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n_max = max(n_max, __shfl_xor_sync(0xffffffffu, n_max, o));
  unsigned sum0 = 0, sum1 = 0, sum2 = 0, sum3 = 0;
  unsigned a02 = 0, a13 = 0;
  for (int p0 = 0; p0 < n_max; p0 += 32) {
    // the scan's lanes stage {D index of the lattice origin, qy << 16 | qx} of 32 points
    __syncwarp();
    if (has_scan) {
      for (int t = ql; t < 32; t += lanes) {
        int2 d = make_int2(0, static_cast<int>(0x80008000u));  // never in range
        if (p0 + t < jb.n) {
          const short2 c = pts[p0 + t];
          const int bx = c.x + ox, by = c.y + oy;
          const int qx = bx >> h, qy = by >> h;  // floor division
          if (qx > -32000 && qx < 32000 && qy > -32000 && qy < 32000)
            d = make_int2(((((by & s1) << h) | (bx & s1)) * jd + qy) * ids + qx,
                          (qy << 16) | (qx & 0xffff));
        }
        s_pt[t] = d;
      }
    }
    __syncwarp();
    if (owns) {
#pragma unroll 8
      for (int t = 0; t < 32; t += 2) {
        const int4 d = *reinterpret_cast<const int4*>(s_pt + t);
        const int Ja = (d.y >> 16) + jy, ca = static_cast<short>(d.y & 0xffff) + i0 + 3;
        const int Jb = (d.w >> 16) + jy, cb = static_cast<short>(d.w & 0xffff) + i0 + 3;
        if (static_cast<unsigned>(Ja) < static_cast<unsigned>(jd) &&
            static_cast<unsigned>(ca) < static_cast<unsigned>(id + 3)) {
          const int a = d.x + toff;
          const unsigned k = static_cast<unsigned>(a) & 3u;
          const unsigned w = __ldg(reinterpret_cast<const unsigned*>(
              dec + static_cast<long long>(a) + static_cast<long long>(k * lpad1)));
          a02 += __byte_perm(w, 0u, 0x4240);  // bytes 0 and 2 in u16 lanes
          a13 += __byte_perm(w, 0u, 0x4341);  // bytes 1 and 3
        }
        if (static_cast<unsigned>(Jb) < static_cast<unsigned>(jd) &&
            static_cast<unsigned>(cb) < static_cast<unsigned>(id + 3)) {
          const int a = d.z + toff;
          const unsigned k = static_cast<unsigned>(a) & 3u;
          const unsigned w = __ldg(reinterpret_cast<const unsigned*>(
              dec + static_cast<long long>(a) + static_cast<long long>(k * lpad1)));
          a02 += __byte_perm(w, 0u, 0x4240);
          a13 += __byte_perm(w, 0u, 0x4341);
        }
      }
    }
    if (((p0 + 32) & 255) == 0 || p0 + 32 >= n_max) {  // flush the packed u16 sums
      sum0 += a02 & 0xffffu;
      sum2 += a02 >> 16;
      sum1 += a13 & 0xffffu;
      sum3 += a13 >> 16;
      a02 = a13 = 0u;
    }
  }
  if (!owns) return;
  int* __restrict__ out = top_sum + scan_slot_base[sg];
  const unsigned sums[4] = {sum0, sum1, sum2, sum3};
#pragma unroll
  for (int e = 0; e < 4; ++e)
    if (i0 + e < si.nxc) out[(i0 + e) * si.nyc + jy] = static_cast<int>(sums[e]);
}

// Lowest-resolution pass, dense form: one CTA per scan.  The candidates of one
// rotated scan form a lattice of stride s = 2^h, so for a scan point p the cells
// they read are one contiguous block of the decimated level (StackDev::dec4).
// A thread owns kQuads "quads" = 4 x-consecutive candidates of one lattice row
// and fetches their 4 cells with ONE aligned 32-bit load from the byte-shifted
// copy that matches the address' alignment; the four byte lanes are accumulated
// SIMD-in-register (2 x u16 per register, flushed every 256 points).  Point
// descriptors (tile base + lattice origin) are computed once per CTA into shared
// memory and broadcast to all threads.
constexpr int kDenseThreads = 128;
constexpr int kDenseChunk = 256;  // <= 257 so the packed u16 sums cannot overflow
template <int kQuads>
__global__ void __launch_bounds__(kDenseThreads)
k_score_top_dense(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
                  const short2* __restrict__ dscan, int* __restrict__ top_sum,
                  const long long* __restrict__ scan_slot_base, int total_scans) {
  __shared__ int4 s_pt[kDenseChunk];  // {D index of lattice origin, qx, qy, 0}
  for (int sg = blockIdx.x; sg < total_scans; sg += gridDim.x) {
    const ScanInfo si = info[sg];
    const JobDev& jb = jobs[si.job];
    const StackDev& st = *jb.stack;
    const int h = st.depth - 1;
    const int s = 1 << h;
    const int id = st.dec_id[h], jd = st.dec_jd[h], ids = st.dec_ids[h];
    const unsigned lpad1 = static_cast<unsigned>(st.dec_lpad[h]) - 1u;
    const uint8_t* __restrict__ dec = st.dec4[h] + 16;
    const int qr = (si.nxc + 3) >> 2;       // quads per lattice row
    const int quads = qr * si.nyc;
    const short2* __restrict__ pts = dscan + jb.dscan_off +
                                   static_cast<long long>(sg - jb.scan_base) * jb.n;
    int* __restrict__ out = top_sum + scan_slot_base[sg];
    for (int u0 = 0; u0 < quads; u0 += kDenseThreads * kQuads) {
      int jy[kQuads], i0[kQuads], toff[kQuads];
      unsigned sum[kQuads][4];
#pragma unroll
      for (int r = 0; r < kQuads; ++r) {
        const int u = u0 + threadIdx.x + r * kDenseThreads;
        jy[r] = u / qr;
        i0[r] = (u - jy[r] * qr) << 2;
        if (u >= quads) jy[r] = 1 << 20;    // never in range
        toff[r] = jy[r] * ids + i0[r];
        sum[r][0] = sum[r][1] = sum[r][2] = sum[r][3] = 0u;
      }
      for (int p0 = 0; p0 < jb.n; p0 += kDenseChunk) {
        __syncthreads();
        for (int t = threadIdx.x; t < kDenseChunk; t += kDenseThreads) {
          const int p = p0 + t;
          int4 d = make_int4(0, -(1 << 24), -(1 << 24), 0);
          if (p < jb.n) {
            const short2 c = pts[p];
            const int bx = c.x + si.min_x + s - 1, by = c.y + si.min_y + s - 1;
            const int qx = bx >> h, qy = by >> h;          // floor division
            const int ax = bx & (s - 1), ay = by & (s - 1);
            if (qx > -(1 << 20) && qx < (1 << 20) && qy > -(1 << 20) && qy < (1 << 20))
              d = make_int4(((ay * s + ax) * jd + qy) * ids + qx, qx, qy, 0);
          }
          s_pt[t] = d;
        }
        __syncthreads();
        const int cnt = min(kDenseChunk, jb.n - p0);
        unsigned a02[kQuads], a13[kQuads];
#pragma unroll
        for (int r = 0; r < kQuads; ++r) a02[r] = a13[r] = 0u;
#pragma unroll 4
        for (int t = 0; t < cnt; ++t) {
          const int4 d = s_pt[t];
#pragma unroll
          for (int r = 0; r < kQuads; ++r) {
            const int J = d.z + jy[r];
            const int c3 = d.y + i0[r] + 3;   // column of the quad's last byte
            if (static_cast<unsigned>(J) < static_cast<unsigned>(jd) &&
                static_cast<unsigned>(c3) < static_cast<unsigned>(id + 3)) {
              const int a = d.x + toff[r];    // D index of the quad's first byte (>= -3)
              const unsigned k = static_cast<unsigned>(a) & 3u;
              const unsigned w = __ldg(reinterpret_cast<const unsigned*>(
                  dec + static_cast<long long>(a) + static_cast<long long>(k * lpad1)));
              a02[r] += __byte_perm(w, 0u, 0x4240);  // bytes 0 and 2 in u16 lanes
              a13[r] += __byte_perm(w, 0u, 0x4341);  // bytes 1 and 3
            }
          }
        }
#pragma unroll
        for (int r = 0; r < kQuads; ++r) {
          sum[r][0] += a02[r] & 0xffffu;
          sum[r][2] += a02[r] >> 16;
          sum[r][1] += a13[r] & 0xffffu;
          sum[r][3] += a13[r] >> 16;
        }
      }
#pragma unroll
      for (int r = 0; r < kQuads; ++r) {
        if (jy[r] < si.nyc) {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (i0[r] + e < si.nxc) out[(i0[r] + e) * si.nyc + jy[r]] = static_cast<int>(sum[r][e]);
        }
      }
    }
  }
}

// ---- lowest-resolution pass, tile form ------------------------------------------
// For one scan point the candidates of a scan's lattice that fall inside the grid
// read exactly one tile of the decimated level: jd rows of ids bytes, contiguous in
// memory (phase (ax, ay) of StackDev::dec4).  MatchFullSubmap lattices are wider than
// that tile (most candidate/point pairs lie outside the grid), so instead of every
// candidate walking all points, ONE WARP walks the points of a scan and adds each
// point's tile into the lattice:
//   * lane l owns the tile words f = l - 1 + 32*it (fully coalesced 128 B loads);
//   * the word offset between tile and lattice, (qx, qy), only changes when the point
//     moves to another coarse cell; consecutive beams mostly stay in one, so the
//     lanes accumulate in REGISTERS (packed u16 pairs) across a run of points and add
//     the run into the 32-bit lattice in shared memory when (qx, qy) changes (or
//     after 256 points, before the u16 lanes can overflow);
//   * copy k = qx & 3 of dec4 aligns tile words with lattice quads.
// Integer sums are order independent, so the result equals k_score_top_dense's.
#ifndef CSM_TILE_THREADS
#define CSM_TILE_THREADS 128
#endif
constexpr int kTileThreads = CSM_TILE_THREADS;
constexpr int kTileWarps = kTileThreads / 32;
template <int kIters>
__global__ void __launch_bounds__(kTileThreads)
k_score_top_tile(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
                 const short2* __restrict__ dscan, int* __restrict__ top_sum,
                 const long long* __restrict__ scan_slot_base, int scan0, int scan_end,
                 int lat_ints) {
  extern __shared__ __align__(16) int s_lat_all[];
  __shared__ __align__(16) int s_key_all[kTileWarps][32], s_off_all[kTileWarps][32];
  constexpr int kNoKey = 0x7fff7fff;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* __restrict__ s_lat = s_lat_all + warp * lat_ints;  // [nyc][qr] quads of 4 ints
  int* __restrict__ s_key = s_key_all[warp];
  int* __restrict__ s_off = s_off_all[warp];
  const int nwarps = gridDim.x * kTileWarps;
  for (int sg = scan0 + blockIdx.x * kTileWarps + warp; sg < scan_end; sg += nwarps) {
    const ScanInfo si = info[sg];
    const JobDev& jb = jobs[si.job];
    const StackDev& st = *jb.stack;
    const int h = st.depth - 1;
    const int s1 = (1 << h) - 1;
    const int id = st.dec_id[h], jd = st.dec_jd[h], ids = st.dec_ids[h];
    const long long lpad = st.dec_lpad[h];
    const uint8_t* __restrict__ dec = st.dec4[h] + 16;
    const int rw = ids >> 2;         // words per tile row
    const int W = jd * rw + 1;       // tile words incl. the one before the tile (f = -1)
    const int qr = (si.nxc + 3) >> 2;
    const int lat_n = qr * 4 * si.nyc;
    const short2* __restrict__ pts = dscan + jb.dscan_off +
                                   static_cast<long long>(sg - jb.scan_base) * jb.n;
    int* __restrict__ out = top_sum + scan_slot_base[sg];
    for (int t = lane; t < lat_n; t += 32) s_lat[t] = 0;
    unsigned a02[kIters], a13[kIters];
#pragma unroll
    for (int it = 0; it < kIters; ++it) a02[it] = a13[it] = 0u;
    int cur_key = kNoKey;      // (qy << 16) | (qx & 0xffff) of the current run
    int run = 0;
    const uint8_t* cur_base = dec;
    // adds the run's register sums into the lattice
    // tile row and byte column (before the copy shift k) of this lane's words
    int f_row[kIters], f_col[kIters];
#pragma unroll
    for (int it = 0; it < kIters; ++it) {
      const int f = lane + 32 * it - 1;
      f_row[it] = (f + rw) / rw - 1;               // floor(f / rw) for f >= -1
      f_col[it] = (f - f_row[it] * rw) << 2;
      if (f + 1 >= W) f_row[it] = -(1 << 20);      // not a tile word: never valid
    }
    auto flush = [&]() {
      __syncwarp();
      const int qx = static_cast<short>(cur_key & 0xffff), qy = cur_key >> 16;
      const int k = qx & 3;
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        int r = f_row[it];
        int c0 = f_col[it] + k;                 // tile column of the word's first byte
        if (c0 + 3 >= ids) { ++r; c0 -= ids; }  // the word continues in the next row
        const int j = r - qy, i0 = c0 - qx;     // lattice row / first lattice column (multiple of 4)
        if (c0 < id && static_cast<unsigned>(r) < static_cast<unsigned>(jd) &&
            static_cast<unsigned>(j) < static_cast<unsigned>(si.nyc) &&
            static_cast<unsigned>(i0) < static_cast<unsigned>(qr << 2)) {
          int4* cell = reinterpret_cast<int4*>(s_lat) + (j * qr + (i0 >> 2));
          int4 v = *cell;
          v.x += static_cast<int>(a02[it] & 0xffffu);
          v.y += static_cast<int>(a13[it] & 0xffffu);
          v.z += static_cast<int>(a02[it] >> 16);
          v.w += static_cast<int>(a13[it] >> 16);
          *cell = v;
        }
        a02[it] = a13[it] = 0u;
      }
    };
    for (int p0 = 0; p0 < jb.n; p0 += 32) {
      int my_off = 0, my_key = kNoKey;
      if (p0 + lane < jb.n) {
        const short2 c = pts[p0 + lane];
        const int bx = c.x + si.min_x + s1, by = c.y + si.min_y + s1;
        const int qx = bx >> h, qy = by >> h;  // floor division
        if (qx > -32000 && qx < 32000 && qy > -32000 && qy < 32000) {
          my_off = ((((by & s1) << h) | (bx & s1)) * jd) * ids;
          my_key = (qy << 16) | (qx & 0xffff);
        }
      }
      __syncwarp();
      s_key[lane] = my_key;
      s_off[lane] = my_off;
      __syncwarp();
      for (int t = 0; t < 32; t += 4) {   // points past the end carry kNoKey
        const int4 key = *reinterpret_cast<const int4*>(s_key + t);
        const int4 off = *reinterpret_cast<const int4*>(s_off + t);
        if (key.x == cur_key && key.y == cur_key && key.z == cur_key && key.w == cur_key &&
            run <= 252 && cur_key != kNoKey) {
          // four points of the current run: 4 * kIters independent loads in flight
          run += 4;
          unsigned w[4][kIters];
#pragma unroll
          for (int it = 0; it < kIters; ++it) {
            const bool on = lane + 32 * it < W;
            w[0][it] = on ? __ldg(reinterpret_cast<const unsigned*>(cur_base + off.x) + 32 * it) : 0u;
            w[1][it] = on ? __ldg(reinterpret_cast<const unsigned*>(cur_base + off.y) + 32 * it) : 0u;
            w[2][it] = on ? __ldg(reinterpret_cast<const unsigned*>(cur_base + off.z) + 32 * it) : 0u;
            w[3][it] = on ? __ldg(reinterpret_cast<const unsigned*>(cur_base + off.w) + 32 * it) : 0u;
          }
#pragma unroll
          for (int it = 0; it < kIters; ++it) {
            a02[it] += (__byte_perm(w[0][it], 0u, 0x4240) + __byte_perm(w[1][it], 0u, 0x4240)) +
                       (__byte_perm(w[2][it], 0u, 0x4240) + __byte_perm(w[3][it], 0u, 0x4240));
            a13[it] += (__byte_perm(w[0][it], 0u, 0x4341) + __byte_perm(w[1][it], 0u, 0x4341)) +
                       (__byte_perm(w[2][it], 0u, 0x4341) + __byte_perm(w[3][it], 0u, 0x4341));
          }
          continue;
        }
#pragma unroll 1
        for (int u = 0; u < 4; ++u) {
          const int ku = s_key[t + u], ou = s_off[t + u];
          if (ku != cur_key || run == 256) {
            if (run) flush();
            cur_key = ku;
            run = 0;
            cur_base = dec + (cur_key & 3) * lpad - 4 + 4 * lane;
          }
          if (ku == kNoKey) continue;  // point cannot hit the grid / past the end
          ++run;
          const unsigned* __restrict__ q = reinterpret_cast<const unsigned*>(cur_base + ou);
#pragma unroll
          for (int it = 0; it < kIters; ++it) {
            if (lane + 32 * it < W) {
              const unsigned w = __ldg(q + 32 * it);
              a02[it] += __byte_perm(w, 0u, 0x4240);  // bytes 0 and 2 in u16 lanes
              a13[it] += __byte_perm(w, 0u, 0x4341);  // bytes 1 and 3
            }
          }
        }
      }
    }
    if (run) flush();
    __syncwarp();
    const int slots = si.nxc * si.nyc;
    for (int o = lane; o < slots; o += 32) {
      const int i = o / si.nyc, j = o - i * si.nyc;
      out[o] = s_lat[((j * qr + (i >> 2)) << 2) + (i & 3)];
    }
    __syncwarp();
  }
}

// Generic list scoring (test hook + tie resolution): one warp per candidate.
struct ListCand { int scan; int xo, yo, level; };
__global__ void __launch_bounds__(256)
k_score_list(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
             const short2* __restrict__ dscan, const ListCand* __restrict__ cands, int count,
             int* __restrict__ sums, float* __restrict__ scores) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= count) return;
  const ListCand c = cands[warp];
  const JobDev& jb = jobs[info[c.scan].job];
  const StackDev& st = *jb.stack;
  const int w1 = (1 << c.level) - 1;
  const uint8_t* __restrict__ g = st.level[c.level];
  const int wx = st.wx[c.level], wy = st.wy[c.level];
  const short2* __restrict__ pts = dscan + jb.dscan_off +
                                 static_cast<long long>(c.scan - jb.scan_base) * jb.n;
  int sum = 0;
  for (int p = lane; p < jb.n; p += 32) {
    const short2 q = pts[p];
    sum += GetValue(g, wx, wy, q.x + c.xo + w1, q.y + c.yo + w1);
  }
  sum = WarpSum(sum);
  if (lane == 0) {
    if (sums) sums[warp] = sum;
    if (scores) scores[warp] = ToScore(st, sum, jb.n);
  }
}

// Scores the (up to) four children of a node at level h-1 with one warp.
// Slot t = 2*ix + iy (ix, iy in {0,1}) is the child at offset (ix*half, iy*half);
// increasing t is the reference's generation order (x offset outer, y offset
// inner), and a slot is valid unless it is clipped by the scan's max bound
// (fast...2d.cc:352-367).  One aligned word of the child-window layout
// (StackDev::win) holds all four children values for a scan point; four points per
// lane are in flight per iteration (the loop is latency-bound otherwise).
// Returns the valid mask; sums[t] is 0 if invalid.
__device__ __forceinline__ unsigned ScoreChildren(const StackDev& st, const ScanInfo& si,
                                                  const short2* __restrict__ pts, int n, int xo,
                                                  int yo, int h, int lane, int sums[4]) {
  const int half = 1 << (h - 1);
  const bool x2 = !(xo + half > si.max_x);
  const bool y2 = !(yo + half > si.max_y);
  const int S1 = (1 << h) - 1;
  const unsigned* __restrict__ win = st.win[h];
  const int jd = st.win_jd[h], ids = st.win_ids[h];
  const long long per_phase = WinPhaseWords(jd, ids);
  const int bx = xo + half - 1, by = yo + half - 1;
  int s00 = 0, s01 = 0, s10 = 0, s11 = 0;
  constexpr int kU = 4;
  for (int p0 = lane; p0 < n; p0 += 32 * kU * 64) {
    // packed u16 pairs: r0 = (ix 0, ix 1) of iy 0, r1 = same of iy 1; at most
    // 64 * kU = 256 points per lane between flushes (256 * 255 < 2^16)
    unsigned r0 = 0, r1 = 0;
    const int pend = min(n, p0 + 32 * kU * 64);
    for (int p = p0; p < pend; p += 32 * kU) {
      short2 q[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int pp = p + 32 * u;
        q[u] = pp < pend ? pts[pp] : make_short2(0, 0);
      }
      unsigned w[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int lx = q[u].x + bx, ly = q[u].y + by;
        const int Qx = (lx >> h) + 1, Qy = (ly >> h) + 1;
        w[u] = 0u;
        if (p + 32 * u < pend && static_cast<unsigned>(Qx) < static_cast<unsigned>(ids) &&
            static_cast<unsigned>(Qy) < static_cast<unsigned>(jd))
          w[u] = __ldg(win + (static_cast<long long>((ly & S1) << h | (lx & S1)) * per_phase +
                              WinCell(Qx, Qy, ids)));
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        r0 += __byte_perm(w[u], 0u, 0x4140);
        r1 += __byte_perm(w[u], 0u, 0x4342);
      }
    }
    s00 += r0 & 0xffffu;
    s10 += r0 >> 16;
    s01 += r1 & 0xffffu;
    s11 += r1 >> 16;
  }
  sums[0] = WarpSum(s00);
  sums[1] = y2 ? WarpSum(s01) : 0;
  sums[2] = x2 ? WarpSum(s10) : 0;
  sums[3] = (x2 && y2) ? WarpSum(s11) : 0;
  return 1u | (y2 ? 2u : 0u) | (x2 ? 4u : 0u) | ((x2 && y2) ? 8u : 0u);
}

// scan -> job and scan -> first lowest-resolution slot, one CTA per job.
__global__ void k_scan_tables(const JobDev* __restrict__ jobs, int* __restrict__ scan_job,
                              long long* __restrict__ scan_slot_base, unsigned* __restrict__ lb,
                              int* __restrict__ job_best) {
  const JobDev& d = jobs[blockIdx.x];
  if (threadIdx.x == 0) {
    // the bound starts at min_score: only scores > min_score are ever accepted (fast...2d.cc:253)
    lb[blockIdx.x] = FloatToOrdered(d.min_score);
    job_best[blockIdx.x] = 0;
  }
  for (int k = threadIdx.x; k < d.num_scans; k += blockDim.x) {
    scan_job[d.scan_base + k] = blockIdx.x;
    scan_slot_base[d.scan_base + k] = d.top_off + static_cast<long long>(k) * d.cap;
  }
}

// Per-job maximum of the lowest-resolution sums (one warp per scan -> atomicMax).
__global__ void __launch_bounds__(256)
k_job_best(const ScanInfo* __restrict__ info, const int* __restrict__ top_sum,
           const long long* __restrict__ scan_slot_base, int total_scans,
           int* __restrict__ job_best) {
  const int lane = threadIdx.x & 31;
  const int sg = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (sg >= total_scans) return;
  const ScanInfo si = info[sg];
  const int slots = si.nxc * si.nyc;
  const int* __restrict__ ts = top_sum + scan_slot_base[sg];
  int best = 0;
  for (int s = lane; s < slots; s += 32) best = max(best, ts[s]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) atomicMax(&job_best[si.job], best);
}

// Greedy dives: one warp per scan starts at the scan's best lowest-resolution
// candidate and follows the best child down to a leaf.  Every leaf score is a
// valid lower bound of the job's optimum; the maximum over all scans seeds the
// branch-and-bound (the reference's DFS gets the same bound from its first dive,
// fast...2d.cc:335-378, only later).
__global__ void __launch_bounds__(256)
k_dive(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
       const short2* __restrict__ dscan, const int* __restrict__ top_sum,
       const long long* __restrict__ scan_slot_base, int total_scans,
       const int* __restrict__ job_best, float dive_ratio,
       unsigned* __restrict__ lb, unsigned long long* __restrict__ counters) {
  const int lane = threadIdx.x & 31;
  const int sg = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (sg >= total_scans) return;
  const ScanInfo si = info[sg];
  const JobDev& jb = jobs[si.job];
  const StackDev& st = *jb.stack;
  const int slots = si.nxc * si.nyc;
  const int* __restrict__ ts = top_sum + scan_slot_base[sg];
  int best = -1, best_slot = 0;
  for (int s = lane; s < slots; s += 32) {
    const int v = ts[s];
    if (v > best) { best = v; best_slot = s; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int os = __shfl_xor_sync(0xffffffffu, best_slot, o);
    if (ov > best || (ov == best && os < best_slot)) { best = ov; best_slot = os; }
  }
  if (!(ToScore(st, best, jb.n) > jb.min_score)) return;
  // only scans whose best bound is close to the job's best bound are worth a dive
  // (any subset keeps the bound valid; this one keeps it tight at a fraction of the cost)
  if (static_cast<float>(best) < dive_ratio * static_cast<float>(job_best[si.job])) return;
  int h = st.depth - 1;
  const int i = best_slot / si.nyc, jy = best_slot - i * si.nyc;
  int xo = si.min_x + (i << h), yo = si.min_y + (jy << h);
  const short2* __restrict__ pts = dscan + jb.dscan_off +
                                 static_cast<long long>(sg - jb.scan_base) * jb.n;
  int leaf_sum = best;
  unsigned long long scored = 0;
  while (h > 0) {
    int sums[4];
    const unsigned valid = ScoreChildren(st, si, pts, jb.n, xo, yo, h, lane, sums);
    scored += __popc(valid);
    const int half = 1 << (h - 1);
    int b = 0, bs = sums[0];
#pragma unroll
    for (int t = 1; t < 4; ++t)
      if (((valid >> t) & 1u) && sums[t] > bs) { b = t; bs = sums[t]; }
    xo += (b >> 1) * half;
    yo += (b & 1) * half;
    leaf_sum = bs;
    --h;
  }
  if (lane == 0) {
    const float score = ToScore(st, leaf_sum, jb.n);
    if (score > jb.min_score) atomicMax(&lb[si.job], FloatToOrdered(score));
    atomicAdd(&counters[0], scored);
    atomicAdd(&counters[2], 1ull);
  }
}

// Pushes every lowest-resolution candidate that can still contain the optimum
// (score > min_score and score >= current bound) onto the top-level queue.  One
// CTA per scan walks the scan's lattice ROW by ROW (y outer, x inner) and appends
// the survivors in that order with a block-wide ordered compaction, so queue
// neighbours are lattice neighbours along x — the direction the lattice branch
// kernel coalesces over.
__global__ void __launch_bounds__(256)
k_filter_top(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
             const int* __restrict__ top_sum, const long long* __restrict__ scan_slot_base,
             int total_scans, const unsigned* __restrict__ lb, Node* __restrict__ queue,
             int* __restrict__ qcount, int qcap, int* __restrict__ overflow) {
  __shared__ int s_warp[8];
  __shared__ int s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int sg = blockIdx.x; sg < total_scans; sg += gridDim.x) {
    const ScanInfo si = info[sg];
    const JobDev& jb = jobs[si.job];
    const StackDev& st = *jb.stack;
    const int h = st.depth - 1;
    const int slots = si.nxc * si.nyc;
    const float bound = OrderedToFloat(lb[si.job]);
    const int* __restrict__ ts = top_sum + scan_slot_base[sg];
    for (int q0 = 0; q0 < slots; q0 += blockDim.x) {
      const int q = q0 + threadIdx.x;  // row-major lattice index
      bool keep = false;
      float score = 0.f;
      int i = 0, jy = 0;
      if (q < slots) {
        jy = q / si.nxc;
        i = q - jy * si.nxc;
        score = ToScore(st, ts[i * si.nyc + jy], jb.n);
        keep = score > jb.min_score && score >= bound;
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) s_warp[warp] = __popc(m);
      __syncthreads();
      if (threadIdx.x == 0) {
        int tot = 0;
        for (int w = 0; w < 8; ++w) { const int c = s_warp[w]; s_warp[w] = tot; tot += c; }
        s_base = tot ? atomicAdd(qcount, tot) : 0;
      }
      __syncthreads();
      if (keep) {
        const int idx = s_base + s_warp[warp] + __popc(m & ((1u << lane) - 1));
        if (idx < qcap)
          queue[idx] = Node{sg, si.min_x + (i << h), si.min_y + (jy << h), score};
        else
          *overflow = 1;
      }
      __syncthreads();
    }
  }
}

// ---- device-resident control of the level loop ---------------------------------
// The branch-and-bound frontier sizes never visit the host between levels: every
// kernel of a level reads its chunk [start, start + n) of queue[h] and the kernel
// form (`mode`) from this block, which k_level_begin fills from the device-side queue
// counts.  Launch grids are sized for the worst case (or grid-stride), so a whole
// match batch is ONE stream of launches followed by ONE synchronisation.
enum : int {
  kCtlLeaf = 16,      // leaves recorded so far
  kCtlBest = 17,      // optimal leaves after compaction
  kCtlOverflow = 20,  // a queue / leaf buffer was too small
  kCtlItems = 24,     // work items of the current lattice launch
  kCtlStart = 25,     // first node of the current chunk in queue[h]
  kCtlCount = 26,     // nodes of the current chunk
  kCtlMode = 27,      // 0 = nothing to do, 1 = warp per parent, 2 = scan-grouped lattice
  kCtlInts = 32
};

// Branch step: one warp per parent node of level h.  Scores its children at
// level h-1, then either pushes the survivors to the next queue (h-1 >= 1) or,
// at h-1 == 0, raises the job's bound and records the leaf.
__device__ __forceinline__ void ExpandParentWarp(
    const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
    const short2* __restrict__ dscan, const Node nd, int h, unsigned* __restrict__ lb,
    Node* __restrict__ next, int* __restrict__ next_count, int next_cap,
    Node* __restrict__ leaves, int* __restrict__ leaf_count, int leaf_cap,
    int* __restrict__ overflow, unsigned long long* __restrict__ counters) {
  const int lane = threadIdx.x & 31;
  const ScanInfo si = info[nd.scan];
  const JobDev& jb = jobs[si.job];
  const StackDev& st = *jb.stack;
  // bound may have risen since the node was queued
  if (!(nd.score >= OrderedToFloat(lb[si.job]))) return;
  const short2* __restrict__ pts = dscan + jb.dscan_off +
                                 static_cast<long long>(nd.scan - jb.scan_base) * jb.n;
  int sums[4];
  const unsigned valid = ScoreChildren(st, si, pts, jb.n, nd.xo, nd.yo, h, lane, sums);
  if (lane != 0) return;
  atomicAdd(&counters[0], (unsigned long long)__popc(valid));
  atomicAdd(&counters[1], 1ull);
  const int half = 1 << (h - 1);
  float sc[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) sc[t] = ToScore(st, sums[t], jb.n);
  if (h - 1 == 0) {
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (!((valid >> t) & 1u) || !(sc[t] > jb.min_score)) continue;
      const unsigned o = FloatToOrdered(sc[t]);
      const unsigned old = atomicMax(&lb[si.job], o);
      if (o >= old) {
        const int idx = atomicAdd(leaf_count, 1);
        if (idx < leaf_cap)
          leaves[idx] = Node{nd.scan, nd.xo + (t >> 1) * half, nd.yo + (t & 1) * half, sc[t]};
        else
          *overflow = 1;
      }
    }
  } else {
    const float bound = OrderedToFloat(lb[si.job]);
    unsigned keep = 0;
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (((valid >> t) & 1u) && sc[t] > jb.min_score && sc[t] >= bound) keep |= 1u << t;
    if (keep) {
      int idx = atomicAdd(next_count, __popc(keep));
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if ((keep >> t) & 1u) {
          if (idx < next_cap)
            next[idx] = Node{nd.scan, nd.xo + (t >> 1) * half, nd.yo + (t & 1) * half, sc[t]};
          else
            *overflow = 1;
          ++idx;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256)
k_expand(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
         const short2* __restrict__ dscan, const Node* __restrict__ queue,
         const int* __restrict__ ctl, int h,
         unsigned* __restrict__ lb, Node* __restrict__ next, int* __restrict__ next_count,
         int next_cap, Node* __restrict__ leaves, int* __restrict__ leaf_count, int leaf_cap,
         int* __restrict__ overflow, unsigned long long* __restrict__ counters) {
  if (ctl[kCtlMode] != 1) return;
  const int count = ctl[kCtlCount];
  const Node* __restrict__ parents = queue + ctl[kCtlStart];
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; warp < count; warp += warps)
    ExpandParentWarp(jobs, info, dscan, parents[warp], h, lb, next, next_count, next_cap, leaves,
                     leaf_count, leaf_cap, overflow, counters);
}

// ---- scan-grouped branch step ------------------------------------------------
// The frontier nodes of ONE rotated scan lie on that scan's lattice of stride
// S = 2^h, so for one scan point the child-window words (StackDev::win) of lattice
// neighbours are neighbouring words of one phase tile.  Parents are first grouped by
// scan (counting sort), then one WARP handles a work item of up to 32 parents of a
// scan: point descriptors are staged once per item in shared memory and every lane
// fetches the 2 x 2 children of its parent with ONE aligned 32-bit load per point (vs.
// a point load + a scattered word per lane in the warp-per-parent form).
struct WorkItem { int scan, start, count; };

__global__ void k_level_begin(int* __restrict__ ctl, int h, int chunk_cap, int lattice_min) {
  if (threadIdx.x != 0) return;
  const int have = ctl[h];
  const int n = min(have, chunk_cap);
  ctl[h] = have - n;          // the chunk is taken from the END of the queue
  ctl[kCtlStart] = have - n;
  ctl[kCtlCount] = n;
  ctl[kCtlItems] = 0;
  ctl[kCtlMode] = n == 0 ? 0 : (n >= lattice_min ? 2 : 1);
}

// The producers push a scan's survivors in runs, so most warps see one or two scans: one
// atomic per scan per warp instead of one per node (with one per node, same-address
// atomics made this kernel half of the grouping's time).
__global__ void __launch_bounds__(256)
k_q_count(const Node* __restrict__ queue, const int* __restrict__ ctl,
          int* __restrict__ scan_cnt) {
  if (ctl[kCtlMode] != 2) return;
  const Node* __restrict__ nodes = queue + ctl[kCtlStart];
  const int count = ctl[kCtlCount];
  const int lane = threadIdx.x & 31;
  const int rounded = (count + 31) & ~31;  // whole warps take part in the match
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rounded; i += gridDim.x * blockDim.x) {
    const bool ok = i < count;
    const int scan = ok ? nodes[i].scan : -1 - lane;
    const unsigned peers = __match_any_sync(0xffffffffu, scan);
    if (ok && lane == __ffs(peers) - 1) atomicAdd(&scan_cnt[scan], __popc(peers));
  }
}

// Exclusive prefix sums of scan_cnt (node offsets) and of ceil(cnt / 32) (work
// items) in three steps: sums of 1024-scan blocks, a single-CTA scan of those block
// sums, and per-block scans that also emit the work items.
__device__ __forceinline__ void BlockScan2(int& ia, int& ib, int* s_wa, int* s_wb) {
  // inclusive scan of (ia, ib) over the 1024 threads of the CTA
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int va = __shfl_up_sync(0xffffffffu, ia, o), vb = __shfl_up_sync(0xffffffffu, ib, o);
    if (lane >= o) { ia += va; ib += vb; }
  }
  if (lane == 31) { s_wa[warp] = ia; s_wb[warp] = ib; }
  __syncthreads();
  if (warp == 0) {
    int wa = s_wa[lane], wb = s_wb[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int va = __shfl_up_sync(0xffffffffu, wa, o), vb = __shfl_up_sync(0xffffffffu, wb, o);
      if (lane >= o) { wa += va; wb += vb; }
    }
    s_wa[lane] = wa;
    s_wb[lane] = wb;
  }
  __syncthreads();
  if (warp) { ia += s_wa[warp - 1]; ib += s_wb[warp - 1]; }
}

__global__ void __launch_bounds__(1024)
k_q_block_sums(const int* __restrict__ ctl, const int* __restrict__ scan_cnt, int total_scans,
               int* __restrict__ part_a, int* __restrict__ part_b) {
  __shared__ int s_wa[32], s_wb[32];
  if (ctl[kCtlMode] != 2) return;
  const int i = blockIdx.x * 1024 + threadIdx.x;
  const int cnt = i < total_scans ? scan_cnt[i] : 0;
  int ia = cnt, ib = (cnt + 31) >> 5;
  BlockScan2(ia, ib, s_wa, s_wb);
  if (threadIdx.x == 1023) { part_a[blockIdx.x] = ia; part_b[blockIdx.x] = ib; }
}

// in-place exclusive scan of the block sums; single CTA, every thread owns a
// contiguous segment.  out[0] = total number of work items.
__global__ void __launch_bounds__(1024)
k_q_scan_parts(const int* __restrict__ ctl, int* __restrict__ part_a, int* __restrict__ part_b,
               int nb, int* __restrict__ out) {
  __shared__ int s_wa[32], s_wb[32];
  if (ctl[kCtlMode] != 2) return;
  const int seg = (nb + 1023) >> 10;
  const int lo = min(nb, static_cast<int>(threadIdx.x) * seg), hi = min(nb, lo + seg);
  int a = 0, b = 0;
  for (int i = lo; i < hi; ++i) { a += part_a[i]; b += part_b[i]; }
  int ia = a, ib = b;
  BlockScan2(ia, ib, s_wa, s_wb);
  int ea = ia - a, eb = ib - b;
  for (int i = lo; i < hi; ++i) {
    const int va = part_a[i], vb = part_b[i];
    part_a[i] = ea;
    part_b[i] = eb;
    ea += va;
    eb += vb;
  }
  if (threadIdx.x == 1023) out[0] = ib;
}

__global__ void __launch_bounds__(1024)
k_q_finish(const int* __restrict__ ctl, const int* __restrict__ scan_cnt, int total_scans,
           const int* __restrict__ part_a, const int* __restrict__ part_b,
           int* __restrict__ scan_off, WorkItem* __restrict__ items) {
  __shared__ int s_wa[32], s_wb[32];
  if (ctl[kCtlMode] != 2) return;
  const int i = blockIdx.x * 1024 + threadIdx.x;
  const int cnt = i < total_scans ? scan_cnt[i] : 0;
  int ia = cnt, ib = (cnt + 31) >> 5;
  BlockScan2(ia, ib, s_wa, s_wb);
  if (i >= total_scans) return;
  const int off = part_a[blockIdx.x] + ia - cnt;
  const int item0 = part_b[blockIdx.x] + ib - ((cnt + 31) >> 5);
  scan_off[i] = off;
  for (int k = 0; k * 32 < cnt; ++k)
    items[item0 + k] = WorkItem{i, off + k * 32, min(32, cnt - k * 32)};
}

// Stable within every 32-node run: lanes holding nodes of the same scan get
// consecutive slots in lane order (one atomic per scan per warp), so the x-ordered
// runs produced by the push code survive the grouping.
__global__ void __launch_bounds__(256)
k_q_scatter(const Node* __restrict__ queue, const int* __restrict__ ctl,
            const int* __restrict__ scan_off, int* __restrict__ cursor,
            Node* __restrict__ sorted) {
  if (ctl[kCtlMode] != 2) return;
  const Node* __restrict__ nodes = queue + ctl[kCtlStart];
  const int count = ctl[kCtlCount];
  const int lane = threadIdx.x & 31;
  const int rounded = (count + 31) & ~31;  // whole warps take part in the match
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rounded; i += gridDim.x * blockDim.x) {
    const bool ok = i < count;
    Node nd = Node{-1 - lane, 0, 0, 0.f};
    if (ok) nd = nodes[i];
    const unsigned peers = __match_any_sync(0xffffffffu, nd.scan);
    const int leader = __ffs(peers) - 1;
    int base = 0;
    if (ok && lane == leader) base = atomicAdd(&cursor[nd.scan], __popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (ok) sorted[scan_off[nd.scan] + base + __popc(peers & ((1u << lane) - 1))] = nd;
  }
}

#ifndef CSM_LAT_MINB
#define CSM_LAT_MINB 9   // CTAs per SM the register allocation aims for
#endif
#ifndef CSM_LAT_THREADS
#define CSM_LAT_THREADS 128
#endif
constexpr int kLatThreads = CSM_LAT_THREADS;   // every warp works on its own item
// Points staged per chunk, and the spacing of the early-exit tests below: on the config-2
// workload, with the bound at the optimum, tests every 128 points skip 31 % of the h = 6
// words and 48-52 % of the h = 5 words, every 256 points 27 % and 44-48 %
// (benchmarks/prototypes/early_exit_counts.py).  With the lanes re-mapped, tests every 64
// points would cut the warp passes by only about 5 % more, for twice the tests
// (benchmarks/prototypes/lane_remap_counts.py).
constexpr int kLatChunk = 128;

// Largest integer sum whose score is <= `score` (the node's own sum when `score` is
// ToScore of it), and smallest sum whose score passes both survival tests of a child
// (score > min_score and score >= bound; 255 n + 1 if none does).  ToScore is monotone in
// the sum, so a walk from the rounded estimate ends at the exact integer, in one or two
// steps in practice.  Without a score range (k255 = 0) they give the loosest values, which
// never rule a parent out.
__device__ __forceinline__ int SumAtMost(const StackDev& st, float score, int n) {
  const int top = 255 * n;
  if (!(st.k255 > 0.f)) return top;
  int e = __float2int_rn((score - st.min_score) / st.k255 * static_cast<float>(n));
  e = min(max(e, 0), top);
  while (e < top && ToScore(st, e + 1, n) <= score) ++e;
  while (e > 0 && ToScore(st, e, n) > score) --e;
  return e;
}
__device__ __forceinline__ int SumToSurvive(const StackDev& st, float min_score, float bound,
                                            int n) {
  const int top = 255 * n;
  auto pass = [&](int t) {
    const float sc = ToScore(st, t, n);
    return sc > min_score && sc >= bound;
  };
  if (!(st.k255 > 0.f)) return 0;
  int t = __float2int_rn((fmaxf(min_score, bound) - st.min_score) / st.k255 *
                         static_cast<float>(n));
  t = min(max(t, 0), top + 1);
  while (t > 0 && pass(t - 1)) --t;
  while (t <= top && !pass(t)) ++t;
  return t;
}

template <int kUnroll>
__global__ void __launch_bounds__(kLatThreads, CSM_LAT_MINB)
k_expand_lattice(const JobDev* __restrict__ jobs, const ScanInfo* __restrict__ info,
                 const short2* __restrict__ dscan, const Node* __restrict__ sorted,
                 const WorkItem* __restrict__ items, const int* __restrict__ num_items, int h,
                 unsigned* __restrict__ lb,
                 Node* __restrict__ next, int* __restrict__ next_count, int next_cap,
                 Node* __restrict__ leaves, int* __restrict__ leaf_count, int leaf_cap,
                 int* __restrict__ overflow, unsigned long long* __restrict__ counters) {
  __shared__ __align__(16) int2 s_all[kLatThreads / 32][kLatChunk];  // {window index of lattice origin, Qy << 16 | Qx}
  // (8 B per point: a smaller shared-memory carve-out leaves more L1 for the tiles)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // (one item per warp and a grid sized for the worst case: a capped grid with an item
  // loop measured 6 % slower — the hardware CTA scheduler balances uneven items better)
  const int item = blockIdx.x * (kLatThreads / 32) + warp;
  if (item >= *num_items) return;
  int2* s_pt = s_all[warp];
  const WorkItem it = items[item];
  // With few parents, G = 2^lg lanes share one parent and split the scan points
  // (lane = parent * G + sub, sub-lane `sub` takes the point pairs sub, sub + G, ...).
  // G grows when the early exit below leaves few parents running.
  int lg = 0;
  while ((it.count << (lg + 1)) <= 32) ++lg;
  int G = 1 << lg;
  int sub = lane & (G - 1);
  const int pidx = lane >> lg;
  const ScanInfo si = info[it.scan];
  const JobDev& jb = jobs[si.job];
  const StackDev& st = *jb.stack;
  const int lv = h - 1;            // level of the children
  const int s = 1 << lv;           // children stride = half the parents' stride
  const int S1 = (1 << h) - 1;
  const int jd = st.win_jd[h], ids = st.win_ids[h];
  const unsigned* __restrict__ win = st.win[h];
  const short2* __restrict__ pts = dscan + jb.dscan_off +
                                   static_cast<long long>(it.scan - jb.scan_base) * jb.n;
  const bool active = pidx < it.count;
  Node nd = Node{it.scan, si.min_x, si.min_y, 0.f};
  if (active) nd = sorted[it.start + pidx];
  // the bound may have risen since the node was queued
  const float bound0 = OrderedToFloat(lb[si.job]);
  const bool live = active && nd.score >= bound0;
  int i0 = (nd.xo - si.min_x) >> h, j0 = (nd.yo - si.min_y) >> h;  // parent lattice coords
  int toff = j0 * ids + i0;
  bool x2 = !(nd.xo + s > si.max_x), y2 = !(nd.yo + s > si.max_y);
  if (live && sub == 0) {
    // a parent ruled out early still counts: the bound decided all its children
    atomicAdd(&counters[0], 1ull + y2 + x2 + (x2 && y2));
    atomicAdd(&counters[1], 1ull);
  }
  unsigned sum0 = 0, sum1 = 0, sum2 = 0, sum3 = 0;  // slots 2*ix+iy: 00, 01, 10, 11
  // Early exit.  Every child window lies inside the parent's, so at each point the
  // largest byte of the word is <= the parent's level-h value there, and the parent's
  // sum is <= p_hi.  After some points, with partial child sums c_t and `mx` the partial
  // sum of the largest bytes, child t ends at most at c_t + p_hi - mx.  Once that is below
  // t_min (no sum below it survives: the bound only rises) for every valid child, the
  // parent is decided and its remaining words are not read.
  int p_hi = SumAtMost(st, nd.score, jb.n);
  const int t_min = SumToSurvive(st, jb.min_score, bound0, jb.n);
  unsigned mx = 0;
  bool run = live;       // live and not yet ruled out
  for (int p0 = 0; p0 < jb.n; p0 += kLatChunk) {
    __syncwarp();
    for (int t = lane; t < kLatChunk; t += 32) {
      const int p = p0 + t;
      int2 d = make_int2(0, static_cast<int>(0x80008000u));  // Qx = Qy = -32768: never in range
      if (p < jb.n) {
        const short2 c = pts[p];
        const int bx = c.x + si.min_x + s - 1, by = c.y + si.min_y + s - 1;
        const int qx = (bx >> h) + 1, qy = (by >> h) + 1;
        const int ax = bx & S1, ay = by & S1;
        if (qx > -32000 && qx < 32000 && qy > -32000 && qy < 32000)
          d = make_int2((((ay << h) | ax) * jd + qy) * ids + qx, (qy << 16) | (qx & 0xffff));
      }
      s_pt[t] = d;
    }
    __syncwarp();
    if (run) {
      const int cnt = min(kLatChunk, jb.n - p0);
      unsigned r0 = 0, r1 = 0;  // packed u16 pairs: (ix 0, ix 1) of iy 0 / iy 1
      auto add = [&](unsigned w) {
        const unsigned a = __byte_perm(w, 0u, 0x4140), b = __byte_perm(w, 0u, 0x4342);
        r0 += a;
        r1 += b;
        const unsigned ab = __vmaxu2(a, b);   // u16 pair (max(b0, b2), max(b1, b3))
        mx += max(ab & 0xffffu, ab >> 16);
      };
      // two staged points per 16-byte shared load (entries past cnt never pass the range test)
#pragma unroll(kUnroll / 2)
      for (int t = 2 * sub; t < cnt; t += 2 * G) {
        const int4 d = *reinterpret_cast<const int4*>(s_pt + t);
        const int Ja = (d.y >> 16) + j0, Ia = static_cast<short>(d.y & 0xffff) + i0;
        const int Jb = (d.w >> 16) + j0, Ib = static_cast<short>(d.w & 0xffff) + i0;
        if (static_cast<unsigned>(Ia) < static_cast<unsigned>(ids) &&
            static_cast<unsigned>(Ja) < static_cast<unsigned>(jd)) {
          add(__ldg(win + (d.x + toff)));
        }
        if (static_cast<unsigned>(Ib) < static_cast<unsigned>(ids) &&
            static_cast<unsigned>(Jb) < static_cast<unsigned>(jd)) {
          add(__ldg(win + (d.z + toff)));
        }
      }
      sum0 += r0 & 0xffffu;   // (ix 0, iy 0)
      sum2 += r0 >> 16;       // (ix 1, iy 0)
      sum1 += r1 & 0xffffu;   // (ix 0, iy 1)
      sum3 += r1 >> 16;       // (ix 1, iy 1)
    }
    if (p0 + kLatChunk < jb.n) {
      // c_t - mx summed over the G sub-lanes of the parent (G is the same on every lane)
      int d0 = static_cast<int>(sum0 - mx), d1 = static_cast<int>(sum1 - mx);
      int d2 = static_cast<int>(sum2 - mx), d3 = static_cast<int>(sum3 - mx);
      for (int o = 1; o < G; o <<= 1) {
        d0 += __shfl_xor_sync(0xffffffffu, d0, o);
        d1 += __shfl_xor_sync(0xffffffffu, d1, o);
        d2 += __shfl_xor_sync(0xffffffffu, d2, o);
        d3 += __shfl_xor_sync(0xffffffffu, d3, o);
      }
      const int lim = t_min - p_hi;
      run = run && (d0 >= lim || (y2 && d1 >= lim) || (x2 && d2 >= lim) ||
                    (x2 && y2 && d3 >= lim));
      const unsigned leads = __ballot_sync(0xffffffffu, run && sub == 0);  // running parents
      if (!leads) break;
      const int L = __popc(leads);
      if ((L << (lg + 1)) <= 32) {
        // Re-map: the L running parents move, in lane (lattice) order, to groups of the
        // largest G with L * G <= 32, so the lanes of ruled-out parents share the remaining
        // points.  A group's partials are first summed over its old sub-lanes; the new
        // sub-lane 0 takes the totals over and the other sub-lanes start from zero.  Lanes
        // left without a running parent hold nothing.
        for (int o = 1; o < G; o <<= 1) {
          sum0 += __shfl_xor_sync(0xffffffffu, sum0, o);
          sum1 += __shfl_xor_sync(0xffffffffu, sum1, o);
          sum2 += __shfl_xor_sync(0xffffffffu, sum2, o);
          sum3 += __shfl_xor_sync(0xffffffffu, sum3, o);
          mx += __shfl_xor_sync(0xffffffffu, mx, o);
        }
        ++lg;
        while ((L << (lg + 1)) <= 32) ++lg;
        G = 1 << lg;
        sub = lane & (G - 1);
        const int k = lane >> lg;       // rank of the lane's new parent among the running ones
        unsigned m = leads;
        for (int i = 0; i < k && m; ++i) m &= m - 1;   // lowest bit: the k-th leader's lane
        const int src = m ? __ffs(m) - 1 : 0;
        const bool own = m && sub == 0;
        const unsigned v0 = __shfl_sync(0xffffffffu, sum0, src), v1 = __shfl_sync(0xffffffffu, sum1, src);
        const unsigned v2 = __shfl_sync(0xffffffffu, sum2, src), v3 = __shfl_sync(0xffffffffu, sum3, src);
        const unsigned vm = __shfl_sync(0xffffffffu, mx, src);
        sum0 = own ? v0 : 0u; sum1 = own ? v1 : 0u; sum2 = own ? v2 : 0u; sum3 = own ? v3 : 0u;
        mx = own ? vm : 0u;
        nd.xo = __shfl_sync(0xffffffffu, nd.xo, src);
        nd.yo = __shfl_sync(0xffffffffu, nd.yo, src);
        p_hi = __shfl_sync(0xffffffffu, p_hi, src);
        const int f = __shfl_sync(0xffffffffu, (x2 ? 1 : 0) | (y2 ? 2 : 0), src);
        x2 = f & 1;
        y2 = f & 2;
        run = m != 0;
        i0 = (nd.xo - si.min_x) >> h;
        j0 = (nd.yo - si.min_y) >> h;
        toff = j0 * ids + i0;
      }
    }
  }
  // totals of the G sub-lanes (all lanes of the warp take part)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned v0 = __shfl_xor_sync(0xffffffffu, sum0, o), v1 = __shfl_xor_sync(0xffffffffu, sum1, o);
    const unsigned v2 = __shfl_xor_sync(0xffffffffu, sum2, o), v3 = __shfl_xor_sync(0xffffffffu, sum3, o);
    if (o < G) { sum0 += v0; sum1 += v1; sum2 += v2; sum3 += v3; }
  }
  // one lane per running parent carries on (the lanes of a parent ruled out early hold
  // partial sums that never reach the queues)
  const bool lead = run && sub == 0;
  const unsigned emit = lead ? (1u | (y2 ? 2u : 0u) | (x2 ? 4u : 0u) | ((x2 && y2) ? 8u : 0u)) : 0u;
  const int sums[4] = {static_cast<int>(sum0), static_cast<int>(sum1), static_cast<int>(sum2),
                       static_cast<int>(sum3)};
  float sc[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) sc[t] = ToScore(st, sums[t], jb.n);
  if (lv == 0) {
    if (!lead) return;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (!((emit >> t) & 1u) || !(sc[t] > jb.min_score)) continue;
      const unsigned o = FloatToOrdered(sc[t]);
      const unsigned old = atomicMax(&lb[si.job], o);
      if (o >= old) {
        const int idx = atomicAdd(leaf_count, 1);
        if (idx < leaf_cap)
          leaves[idx] = Node{nd.scan, nd.xo + (t >> 1) * s, nd.yo + (t & 1) * s, sc[t]};
        else
          *overflow = 1;
      }
    }
    return;
  }
  // Survivors are appended row by row (all lanes' children of lattice row 2*j0, then
  // row 2*j0+1; within a row in lane order, x ascending) with one atomic per warp.
  const float bound = OrderedToFloat(lb[si.job]);
  unsigned keep = 0;
#pragma unroll
  for (int t = 0; t < 4; ++t)
    if (((emit >> t) & 1u) && sc[t] > jb.min_score && sc[t] >= bound) keep |= 1u << t;
  // slot t = 2*ix + iy
  const unsigned m00 = __ballot_sync(0xffffffffu, keep & 1u), m10 = __ballot_sync(0xffffffffu, keep & 4u);
  const unsigned m01 = __ballot_sync(0xffffffffu, keep & 2u), m11 = __ballot_sync(0xffffffffu, keep & 8u);
  const int row0 = __popc(m00) + __popc(m10), row1 = __popc(m01) + __popc(m11);
  int base = 0;
  if (lane == 0 && row0 + row1) base = atomicAdd(next_count, row0 + row1);
  base = __shfl_sync(0xffffffffu, base, 0);
  const unsigned lt = (1u << lane) - 1u;
  int p = base + __popc(m00 & lt) + __popc(m10 & lt);
  if (keep & 1u) {
    if (p < next_cap) next[p] = Node{nd.scan, nd.xo, nd.yo, sc[0]}; else *overflow = 1;
    ++p;
  }
  if (keep & 4u) {
    if (p < next_cap) next[p] = Node{nd.scan, nd.xo + s, nd.yo, sc[2]}; else *overflow = 1;
  }
  p = base + row0 + __popc(m01 & lt) + __popc(m11 & lt);
  if (keep & 2u) {
    if (p < next_cap) next[p] = Node{nd.scan, nd.xo, nd.yo + s, sc[1]}; else *overflow = 1;
    ++p;
  }
  if (keep & 8u) {
    if (p < next_cap) next[p] = Node{nd.scan, nd.xo + s, nd.yo + s, sc[3]}; else *overflow = 1;
  }
}

// Keeps the leaves whose score equals their job's final optimum.  The leaf count is
// read on the device (grid-stride).
__global__ void __launch_bounds__(256)
k_compact_leaves(const ScanInfo* __restrict__ info, const Node* __restrict__ in,
                 const int* __restrict__ count_ptr, int cap_in, const unsigned* __restrict__ lb,
                 Node* __restrict__ out, int* __restrict__ out_count, int cap,
                 int* __restrict__ overflow) {
  const int count = min(*count_ptr, cap_in);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const Node nd = in[i];
    if (FloatToOrdered(nd.score) >= lb[info[nd.scan].job]) {
      const int idx = atomicAdd(out_count, 1);
      if (idx < cap) out[idx] = nd;
      else *overflow = 1;
    }
  }
}

// depth 1: the lowest resolution IS the leaf level (fast...2d.cc:339-343): every queued
// candidate raises its job's bound and becomes a leaf.
__global__ void __launch_bounds__(256)
k_top_as_leaves(const ScanInfo* __restrict__ info, const Node* __restrict__ queue,
                int* __restrict__ ctl, unsigned* __restrict__ lb, Node* __restrict__ leaves,
                int leaf_cap) {
  const int count = ctl[0];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const Node nd = queue[i];
    atomicMax(&lb[info[nd.scan].job], FloatToOrdered(nd.score));
    if (i < leaf_cap) leaves[i] = nd;
    else ctl[kCtlOverflow] = 1;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) ctl[kCtlLeaf] = min(count, leaf_cap);
}

}  // namespace csm

// ===========================================================================
// Host side
// ===========================================================================
using namespace csm;

namespace {

// mapping/value_conversion_tables.cc:29-51 and fast...2d.cc:97-98,110-111,163-169:
// lut[v] = lround(((1 - |cost(v)|) - min_score) * (255 / (max_score - min_score)))
void BuildLut(float min_cost, float max_cost, uint8_t* lut, float* min_score, float* max_score) {
  const float lo = 1.f - max_cost;  // min_score_
  const float hi = 1.f - min_cost;  // max_score_
  *min_score = lo;
  *max_score = hi;
  const float kScale = (max_cost - min_cost) / 32766.f;
  for (int v = 0; v < 65536; ++v) {
    const uint16_t value = static_cast<uint16_t>(v) & static_cast<uint16_t>(~(1u << 15));
    float cost;
    if (value == 0) cost = max_cost;  // unknown -> max_correspondence_cost (grid_2d.cc:69-71)
    else cost = value * kScale + (min_cost - kScale);
    const float probability = 1.f - std::abs(cost);
    const long q = std::lround((probability - lo) * (255.f / (hi - lo)));
    lut[v] = static_cast<uint8_t>(q < 0 ? 0 : (q > 255 ? 255 : q));
  }
}

}  // namespace

// Fills every layout of the stack (levels, decimated copies, child windows) from the
// grid's cells; caller holds ctx->mu.  Shared by csm_stack2d_create and csm_stack2d_update.
// `cells` are host memory with row pitch nx, or (device_pitch > 0) a device array with row
// pitch device_pitch cells (csm_stack2d_create_from_rt_grid2d).
static csm_status BuildStack2D(csm_stack2d* st, const uint16_t* cells, int device_pitch = 0) {
  Ctx* ctx = st->ctx;
  const StackDev& h = st->h;
  const int nx = h.nx, ny = h.ny, depth = h.depth, top = depth - 1;
  std::vector<uint8_t> lut(65536);
  float lo, hi;
  BuildLut(st->min_cost, st->max_cost, lut.data(), &lo, &hi);
  const size_t* win_off = st->win_off;
  // upload cells + LUT into scratch
  DevBuf& d_cells = ctx->D("stack_cells");
  DevBuf& d_lut = ctx->D("stack_lut");
  const size_t ncell = static_cast<size_t>(nx) * ny;
  CSM_TRY(d_cells.Reserve(ncell * sizeof(uint16_t)));
  CSM_TRY(d_lut.Reserve(65536));
  if (device_pitch > 0)
    CSM_CUDA(cudaMemcpy2DAsync(d_cells.p, static_cast<size_t>(nx) * 2, cells,
                               static_cast<size_t>(device_pitch) * 2, static_cast<size_t>(nx) * 2,
                               ny, cudaMemcpyDeviceToDevice, ctx->stream));
  else
    CSM_CUDA(cudaMemcpyAsync(d_cells.p, cells, ncell * sizeof(uint16_t), cudaMemcpyHostToDevice,
                             ctx->stream));
  CSM_CUDA(cudaMemcpyAsync(d_lut.p, lut.data(), 65536, cudaMemcpyHostToDevice, ctx->stream));
  k_stack_level0<<<DivUp(ncell, 256), 256, 0, ctx->stream>>>(
      d_cells.as<uint16_t>(), d_lut.as<uint8_t>(), st->d_levels + st->level_off[0],
      static_cast<int>(ncell));
  CSM_LAUNCH_CHECK();
  for (int l = 1; l < depth; ++l) {
    dim3 block(32, 8), grid(DivUp(h.wx[l], 32), DivUp(h.wy[l], 8));
    k_stack_double<<<grid, block, 0, ctx->stream>>>(st->d_levels + st->level_off[l - 1],
                                                    h.wx[l - 1], h.wy[l - 1],
                                                    st->d_levels + st->level_off[l], h.wx[l],
                                                    h.wy[l], 1 << (l - 1));
    CSM_LAUNCH_CHECK();
  }
  k_stack_decimate4<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(
      h.level[top], h.wx[top], h.wy[top], top, st->d_dec, h.dec_lpad[top], h.dec_id[top],
      h.dec_jd[top], h.dec_ids[top]);
  CSM_LAUNCH_CHECK();
  for (int l = 1; l < depth; ++l) {
    k_stack_window<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(
        h.level[l - 1], h.wx[l - 1], h.wy[l - 1], l, st->d_win + win_off[l], h.win_jd[l],
        h.win_ids[l]);
    CSM_LAUNCH_CHECK();
  }
  return CSM_OK;
}

// csm_stack2d_create over host cells (device_pitch == 0) or over a device array of row
// pitch device_pitch cells; `locked` says the caller already holds the device's ctx->mu.
static csm_status CreateStack2D(const uint16_t* cells, int device_pitch, bool locked, int32_t nx,
                                int32_t ny, double resolution, double max_x, double max_y,
                                float min_cost, float max_cost, int32_t depth, int32_t device,
                                csm_stack2d** out) {
  CSM_REQUIRE(out != nullptr && cells != nullptr, "null pointer");
  CSM_REQUIRE(nx >= 1 && ny >= 1, "cell limits must be >= 1");  // fast...2d.cc:100-102
  CSM_REQUIRE(depth >= 1 && depth <= kMaxDepth, "branch_and_bound_depth out of range");  // :174
  CSM_REQUIRE(resolution > 0., "resolution must be > 0");
  CSM_REQUIRE(min_cost < max_cost, "min cost must be < max cost");  // grid_2d.cc:73
  CSM_REQUIRE(static_cast<long long>(nx) + (1 << (depth - 1)) < 32000 &&
              static_cast<long long>(ny) + (1 << (depth - 1)) < 32000, "grid too large");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::unique_lock<std::mutex> lock(ctx->mu, std::defer_lock);
  if (!locked) lock.lock();
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_stack2d> st(new csm_stack2d);
  st->ctx = ctx;
  st->min_cost = min_cost;
  st->max_cost = max_cost;
  StackDev& h = st->h;
  std::memset(&h, 0, sizeof(h));
  h.nx = nx;
  h.ny = ny;
  h.depth = depth;
  h.resolution = resolution;
  h.max_x = max_x;
  h.max_y = max_y;
  std::vector<uint8_t> lut(65536);
  BuildLut(min_cost, max_cost, lut.data(), &h.min_score, &h.max_score);
  h.k255 = (h.max_score - h.min_score) / 255.f;
  size_t total = 0;
  for (int l = 0; l < depth; ++l) {
    const int w = 1 << l;
    h.wx[l] = nx + w - 1;
    h.wy[l] = ny + w - 1;
    st->level_off[l] = total;
    total += (static_cast<size_t>(h.wx[l]) * h.wy[l] + 255) / 256 * 256;
  }
  CSM_CUDA(cudaMalloc(&st->d_levels, total));
  for (int l = 0; l < depth; ++l) h.level[l] = st->d_levels + st->level_off[l];
  // decimated, 4x byte-shifted copies of the lowest-resolution level (dense pass)
  const int top = depth - 1;
  {
    const int s = 1 << top;
    h.dec_id[top] = (h.wx[top] + s - 1) / s;
    h.dec_jd[top] = (h.wy[top] + s - 1) / s;
    h.dec_ids[top] = (h.dec_id[top] + 3 + 3) / 4 * 4;  // >= 3 zero bytes after every row
    const long long bytes = static_cast<long long>(s) * s * h.dec_jd[top] * h.dec_ids[top];
    CSM_REQUIRE(bytes < (1LL << 29), "decimated level too large");
    h.dec_lpad[top] = static_cast<int>((bytes + 32 + 15) / 16 * 16);
    CSM_CUDA(cudaMalloc(&st->d_dec, 4 * static_cast<size_t>(h.dec_lpad[top])));
    h.dec4[top] = st->d_dec;
  }
  // child-window words for every parent level (branch steps and dives)
  std::vector<size_t> win_off(depth, 0);
  size_t win_total = 0;
  for (int l = 1; l < depth; ++l) {
    const int S = 1 << l;
    h.win_ids[l] = (h.wx[l - 1] + S - 1) / S + 1;
    h.win_jd[l] = (h.wy[l - 1] + S - 1) / S + 1;
    const long long words = static_cast<long long>(S) * S * WinPhaseWords(h.win_jd[l], h.win_ids[l]);
    CSM_REQUIRE(words < (1LL << 31), "window level too large");
    win_off[l] = win_total;
    win_total += (static_cast<size_t>(words) + 63) / 64 * 64;
  }
  if (win_total) CSM_CUDA(cudaMalloc(&st->d_win, win_total * sizeof(unsigned)));
  for (int l = 1; l < depth; ++l) h.win[l] = st->d_win + win_off[l];
  for (int l = 1; l < depth; ++l) st->win_off[l] = win_off[l];
  CSM_TRY(BuildStack2D(st.get(), cells, device_pitch));
  CSM_CUDA(cudaMalloc(&st->d, sizeof(StackDev)));
  CSM_CUDA(cudaMemcpyAsync(st->d, &h, sizeof(StackDev), cudaMemcpyHostToDevice, ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = st.release();
  return CSM_OK;
}

extern "C" {

csm_status csm_stack2d_create(const uint16_t* cells, int32_t nx, int32_t ny, double resolution,
                              double max_x, double max_y, float min_cost, float max_cost,
                              int32_t depth, int32_t device, csm_stack2d** out) {
  return CreateStack2D(cells, 0, false, nx, ny, resolution, max_x, max_y, min_cost, max_cost,
                       depth, device, out);
}

// The PrecomputationGridStack2D constructor over a ProbabilityGrid handle: level 0 is built
// from the handle's device cells (one device-to-device copy into the stack's scratch), with
// the ProbabilityGrid's cost bounds (probability_grid.cc:27-31).
csm_status csm_stack2d_create_from_rt_grid2d(const csm_rt_grid2d* grid, int32_t depth,
                                             csm_stack2d** out) {
  CSM_REQUIRE(grid != nullptr && out != nullptr, "null pointer");
  CSM_REQUIRE(grid->d_wcells == nullptr, "a TSDF2D handle has no precomputation stack");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  const float kMinCorrespondenceCost = 1.f - (1.f - 0.1f);   // probability_values.h:64-67
  const float kMaxCorrespondenceCost = 1.f - 0.1f;
  return CreateStack2D(grid->d_cells, grid->g.pitch, true, grid->g.nx, grid->g.ny,
                       grid->g.resolution, grid->g.max_x, grid->g.max_y, kMinCorrespondenceCost,
                       kMaxCorrespondenceCost, depth, grid->ctx->device, out);
}

csm_status csm_stack2d_destroy(csm_stack2d* stack) {
  if (!stack) return CSM_OK;
  std::lock_guard<std::mutex> lock(stack->ctx->mu);
  cudaSetDevice(stack->ctx->device);
  cudaStreamSynchronize(stack->ctx->stream);
  delete stack;  // the destructor frees the device buffers
  return CSM_OK;
}

// Incremental refresh: the submap's grid received new range data (same limits, same cost
// bounds); rebuilds every layout in place.  No match may be in flight on this stack
// (ConstraintBuilder only matches against finished submaps; a trimmed or updated submap
// goes through DeleteScanMatcher, constraints/constraint_builder_2d.cc:307-316).
csm_status csm_stack2d_update(csm_stack2d* stack, const uint16_t* cells) {
  CSM_REQUIRE(stack != nullptr && cells != nullptr, "null pointer");
  std::lock_guard<std::mutex> lock(stack->ctx->mu);
  CSM_CUDA(cudaSetDevice(stack->ctx->device));
  CSM_TRY(BuildStack2D(stack, cells));
  CSM_CUDA(cudaStreamSynchronize(stack->ctx->stream));
  return CSM_OK;
}

csm_status csm_stack2d_read_level(const csm_stack2d* stack, int32_t level, uint8_t* out,
                                  int32_t* wide_num_x, int32_t* wide_num_y) {
  CSM_REQUIRE(stack != nullptr, "null stack");
  CSM_REQUIRE(level >= 0 && level < stack->h.depth, "level out of range");
  if (wide_num_x) *wide_num_x = stack->h.wx[level];
  if (wide_num_y) *wide_num_y = stack->h.wy[level];
  if (out) {
    std::lock_guard<std::mutex> lock(stack->ctx->mu);
    CSM_CUDA(cudaSetDevice(stack->ctx->device));
    CSM_CUDA(cudaMemcpy(out, stack->h.level[level],
                        static_cast<size_t>(stack->h.wx[level]) * stack->h.wy[level],
                        cudaMemcpyDeviceToHost));
  }
  return CSM_OK;
}

csm_status csm_cloud_create(const float* xyz, int32_t n, int32_t device, csm_cloud** out) {
  CSM_REQUIRE(out != nullptr && xyz != nullptr, "null pointer");
  CSM_REQUIRE(n >= 1, "empty point cloud");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_cloud> c(new csm_cloud);
  c->ctx = ctx;
  c->n = n;
  c->h_xyz.assign(xyz, xyz + 3 * static_cast<size_t>(n));
  float m = 0.f;
  for (int i = 0; i < n; ++i) {
    const float x = xyz[3 * i], y = xyz[3 * i + 1];
    const float range = std::sqrt(x * x + y * y);  // head<2>().norm()
    m = std::max(range, m);
  }
  c->max_norm = m;
  const size_t need = sizeof(float) * 3 * static_cast<size_t>(n);
  for (size_t i = 0; i < ctx->cloud_pool.size(); ++i) {
    if (ctx->cloud_pool[i].second >= need && ctx->cloud_pool[i].second <= 2 * need + 4096) {
      c->d_xyz = static_cast<float*>(ctx->cloud_pool[i].first);
      c->d_bytes = ctx->cloud_pool[i].second;
      ctx->cloud_pool_bytes -= c->d_bytes;
      ctx->cloud_pool[i] = ctx->cloud_pool.back();
      ctx->cloud_pool.pop_back();
      break;
    }
  }
  if (!c->d_xyz) {
    c->d_bytes = (need + 4095) / 4096 * 4096;
    CSM_CUDA(cudaMalloc(&c->d_xyz, c->d_bytes));
  }
  CSM_CUDA(cudaMemcpyAsync(c->d_xyz, xyz, need, cudaMemcpyHostToDevice, ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = c.release();
  return CSM_OK;
}

csm_status csm_cloud_destroy(csm_cloud* cloud) {
  if (!cloud) return CSM_OK;
  std::lock_guard<std::mutex> lock(cloud->ctx->mu);
  cudaSetDevice(cloud->ctx->device);
  Ctx* ctx = cloud->ctx;
  // No match is in flight on this cloud (caller contract), so the buffer can be
  // handed to the next csm_cloud_create without a device-wide cudaFree.
  if (cloud->d_xyz && ctx->cloud_pool.size() < 4096 &&
      ctx->cloud_pool_bytes + cloud->d_bytes <= (256u << 20)) {
    ctx->cloud_pool.emplace_back(cloud->d_xyz, cloud->d_bytes);
    ctx->cloud_pool_bytes += cloud->d_bytes;
    cloud->d_xyz = nullptr;  // now owned by the pool
  } else {
    cudaStreamSynchronize(ctx->stream);
  }
  delete cloud;  // frees d_xyz unless it was pooled
  return CSM_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// Batched matcher
// ---------------------------------------------------------------------------
namespace {

// SearchParameters(linear, angular, cloud, resolution)   (corr...2d.cc:27-55)
struct HostSearch {
  int num_angular;
  int num_scans;
  int lin;
  double step;
  double angular;  // the angular window it was made for (rotation tables are shared by it)
};
HostSearch MakeSearch(double linear_window, double angular_window, float cloud_max_norm,
                      double resolution) {
  float max_scan_range = 3.f * resolution;
  max_scan_range = std::max(cloud_max_norm, max_scan_range);
  const double kSafetyMargin = 1. - 1e-3;
  HostSearch s;
  s.step = kSafetyMargin *
           std::acos(1. - (resolution * resolution) / (2. * (max_scan_range * max_scan_range)));
  s.num_angular = static_cast<int>(std::ceil(angular_window / s.step));
  s.num_scans = 2 * s.num_angular + 1;
  s.lin = static_cast<int>(std::ceil(linear_window / resolution));
  s.angular = angular_window;
  return s;
}

// The search of one job: MatchFullSubmap searches the whole submap (fast...2d.cc:210-225).
HostSearch JobSearch(const csm_stack2d* st, const csm_cloud* cl, const csm_job2d& jb,
                     double linear_window, double angular_window) {
  const double res = st->h.resolution;
  return jb.full_submap ? MakeSearch(1e6 * res, M_PI, cl->max_norm, res)
                        : MakeSearch(linear_window, angular_window, cl->max_norm, res);
}

struct TrigKey {
  const csm_cloud* cloud;
  double resolution, angular;
  bool operator<(const TrigKey& o) const {
    if (cloud != o.cloud) return cloud < o.cloud;
    if (resolution != o.resolution) return resolution < o.resolution;
    return angular < o.angular;
  }
};

// One rotation table: (cos, sin) of the float half angle of every rotated scan of a
// search, at pair offset `off` of the batch's table.
struct TrigTable {
  long long off;
  HostSearch sp;
};

// Tables [t0, t1) into out (pairs).  GenerateRotatedScans: delta_theta accumulates in
// double, is cast to float for AngleAxisf, Quaternionf takes cos/sin of the float half angle.
void FillTrigTables(const std::vector<TrigTable>& tables, size_t t0, size_t t1, float* out) {
  for (size_t t = t0; t < t1; ++t) {
    const HostSearch& sp = tables[t].sp;
    float* o = out + 2 * tables[t].off;
    double delta_theta = -sp.num_angular * sp.step;
    for (int k = 0; k < sp.num_scans; ++k, delta_theta += sp.step) {
      const float ha = 0.5f * static_cast<float>(delta_theta);
      o[2 * k] = std::cos(ha);
      o[2 * k + 1] = std::sin(ha);
    }
  }
}

struct BatchPlan {
  std::vector<JobDev> jobs;
  std::vector<HostSearch> search;
  std::vector<double> init_x, init_y, init_theta;
  long long total_scans = 0, total_points = 0, total_slots = 0;
};

struct TieLeaf { int scan, xo, yo; };

// Kernel forms that can be forced.  A match takes them from CSM_NO_LATTICE / CSM_LAT_UNROLL,
// the test hooks csm_score_top2d / csm_branch_step2d from their arguments.
struct Forms2D {
  const char* top = nullptr;  // "small" | "gather" | "tile" | "dense"; nullptr = by size
  int lattice_min = INT_MAX;  // smallest frontier the lattice kernel takes (INT_MAX: none)
  int unroll = 8;             // k_expand_lattice<4 | 8 | 16>
};

// The branch-and-bound sweep.  The first sweep hmax -> 1 is a static stream of launches:
// every level takes a chunk of <= kChunk nodes from the end of its queue (k_level_begin),
// picks the kernel form on the device and appends the survivors to the next queue; nothing
// is read back in between.  A queue below the top starts the sweep empty and receives
// <= 4 * kChunk children, so it cannot overflow.  Only if a level held more than one chunk
// (frontiers > 8 M nodes) does the host continue, deepest non-empty level first, with one
// read-back per extra chunk.
constexpr int kChunk = 1 << 23;
constexpr int kQueueCap = 4 * kChunk;
constexpr int kLeafCap = 1 << 22;
constexpr int kLatticeMin = 16384;  // smaller frontiers: the warp-per-parent kernel has a
                                    // 34-iteration critical path, the lattice kernel a 1081-iteration one
constexpr int kInlineBest = 4096;   // optimal leaves read back with the first (usually only) sync
// Dives start only from scans whose best lowest-resolution sum is within 3 % of their job's best.
constexpr float kDiveRatio = 0.97f;

double NowMs() {
  return std::chrono::duration<double, std::milli>(
             std::chrono::steady_clock::now().time_since_epoch()).count();
}

// One batch call: its plan, workspaces, control block and read-back area.  MatchBatch2D
// runs the phases below over it in order; the test hooks run the prefix they need.
struct Batch2D {
  Ctx* ctx = nullptr;
  cudaStream_t s = nullptr;
  const csm_stack2d* const* stacks = nullptr;  // indexed by csm_job2d::stack_index
  const csm_cloud* const* clouds = nullptr;    // indexed by csm_job2d::cloud_index
  const csm_job2d* jobs = nullptr;
  int num_jobs = 0;
  Forms2D forms;
  // plan
  BatchPlan plan;
  std::vector<TrigTable> trig_tables;  // in the order of the jobs that first use them
  std::vector<size_t> tables_before;   // tables first used by jobs < j
  std::vector<long long> trig_off;     // per job: offset (in float2) of its table
  long long trig_pairs = 0;            // (cos, sin) pairs of all tables
  std::vector<int> scan_bases;         // scan -> job on the host (optimal leaves only)
  int total_scans = 0;
  // workspaces
  DevBuf *d_trig = nullptr, *d_jobs = nullptr, *d_scan_job = nullptr, *d_slot_base = nullptr,
         *d_info = nullptr, *d_dscan = nullptr, *d_top = nullptr, *d_lb = nullptr,
         *d_ctr = nullptr, *d_job_best = nullptr;
  DevBuf *d_qtop = nullptr, *d_q = nullptr, *d_leaves = nullptr, *d_best = nullptr,
         *d_scan_cnt = nullptr, *d_scan_off = nullptr, *d_items = nullptr, *d_sorted = nullptr;
  float* up_trig = nullptr;           // rotation tables in the pinned upload staging
  unsigned long long* ctr = nullptr;  // counters
  int* ictr = nullptr;                // the level-loop control block (kCtl*)
  int top_kernel = 0;                 // lowest-resolution form that ran: 1 small, 2 gather,
  int tile_iters = 0;                 // 3 tile, 4 dense; K of k_score_top_tile<K>
  int hmax = 0, top_cap = 0;
  // read-back area (pinned): control block | counters | per-job bound | first optimal leaves
  PinnedBuf* pin = nullptr;
  size_t rb_ctr = 0, rb_lb = 0, rb_best = 0;
  const int* hp = nullptr;
  const unsigned long long* hctr = nullptr;
  const unsigned* lbh = nullptr;
  const Node* best_inline = nullptr;
  int host_syncs = 0;
  unsigned long long prof_c0 = 0;
  double t_phase = 0.;

  Batch2D() = default;
  Batch2D(Ctx* c, const csm_stack2d* const* st, const csm_cloud* const* cl, const csm_job2d* jb,
          int n, const Forms2D& f)
      : ctx(c), s(c->stream), stacks(st), clouds(cl), jobs(jb), num_jobs(n), forms(f) {}
  Node* Queue(int h) const {
    return h == hmax ? d_qtop->as<Node>() : d_q->as<Node>() + static_cast<size_t>(kQueueCap) * h;
  }
  int QueueCap(int h) const { return h == hmax ? top_cap : kQueueCap; }
  int JobOfScan(int scan) const {
    return static_cast<int>(std::upper_bound(scan_bases.begin(), scan_bases.end(), scan) -
                            scan_bases.begin()) - 1;
  }
  const StackDev& Stack(int j) const { return stacks[jobs[j].stack_index]->h; }
  int ScanEnd(int j1) const { return j1 < num_jobs ? plan.jobs[j1].scan_base : total_scans; }
  // CSM_TIMING: every phase ends in a synchronise and prints its host time
  void Phase(const char* name) {
    static const bool timing = getenv("CSM_TIMING") != nullptr;
    if (!timing) return;
    cudaStreamSynchronize(s);
    const double t = NowMs();
    fprintf(stderr, "[csm timing] %-14s %8.3f ms\n", name, t - t_phase);
    t_phase = t;
  }
  // candidates scored since the last call (profiling only)
  double ProfScored() {
    unsigned long long c0 = 0;
    cudaStreamSynchronize(s);
    cudaMemcpy(&c0, ctr, sizeof(c0), cudaMemcpyDeviceToHost);
    const double d = static_cast<double>(c0 - prof_c0);
    prof_c0 = c0;
    return d;
  }
};

// Host plan: the jobs' records, the rotation-table layout and the slots each scan's
// lowest-resolution lattice may need.  `search` holds the jobs' searches (JobSearch).
csm_status Plan2D(Batch2D& b, const HostSearch* search) {
  b.t_phase = NowMs();
  const int num_jobs = b.num_jobs;
  BatchPlan& plan = b.plan;
  plan.jobs.resize(num_jobs);
  plan.search.assign(search, search + num_jobs);
  plan.init_x.resize(num_jobs);
  plan.init_y.resize(num_jobs);
  plan.init_theta.resize(num_jobs);
  std::map<TrigKey, long long> trig_index;  // -> offset (in float2) into trig table
  b.tables_before.assign(num_jobs + 1, 0);
  for (int j = 0; j < num_jobs; ++j) {
    const csm_job2d& jb = b.jobs[j];
    const csm_stack2d* st = b.stacks[jb.stack_index];
    const csm_cloud* cl = b.clouds[jb.cloud_index];
    CSM_REQUIRE(st->ctx->device == b.ctx->device && cl->ctx->device == b.ctx->device,
                "handles must share one device");
    const StackDev& h = st->h;
    double ix = jb.initial_pose[0], iy = jb.initial_pose[1], ith = jb.initial_pose[2];
    if (jb.full_submap) {  // fast...2d.cc:210-225
      ix = h.max_x - 0.5 * h.resolution * h.ny;
      iy = h.max_y - 0.5 * h.resolution * h.nx;
      ith = 0.;
    }
    const HostSearch& sp = search[j];
    CSM_REQUIRE(sp.num_scans > 0 && sp.num_scans < (1 << 22), "angular window / step");
    plan.init_x[j] = ix;
    plan.init_y[j] = iy;
    plan.init_theta[j] = ith;
    const TrigKey key{cl, h.resolution, sp.angular};
    auto it = trig_index.find(key);
    if (it == trig_index.end()) {
      b.trig_tables.push_back(TrigTable{b.trig_pairs, sp});
      it = trig_index.emplace(key, b.trig_pairs).first;
      b.trig_pairs += sp.num_scans;
    }
    b.tables_before[j + 1] = b.trig_tables.size();
    JobDev& d = plan.jobs[j];
    d.stack = st->d;
    d.xyz = cl->d_xyz;
    d.trig = nullptr;  // set once the table is uploaded
    b.trig_off.push_back(it->second);
    d.n = cl->n;
    d.num_scans = sp.num_scans;
    d.scan_base = static_cast<int>(plan.total_scans);
    d.lin = sp.lin;
    {
      const float ha = 0.5f * static_cast<float>(ith);
      const float sn = std::sin(ha);
      d.q0w = std::cos(ha);
      d.q0x = sn * 0.f;
      d.q0y = sn * 0.f;
      d.q0z = sn * 1.f;
    }
    d.tx = static_cast<float>(ix);
    d.ty = static_cast<float>(iy);
    d.min_score = jb.min_score;
    // upper bound of lowest-resolution candidates per axis after ShrinkToFit
    // (corr...2d.cc:73-91): with c = cell of the sensor origin and e = scan radius in
    // cells, every point index lies in [c - e, c + e], so the window is at most
    //   min(lin, max(0, cells - 1 - (c - e))) + min(lin, max(0, c + e)).
    // (k_discretize re-checks the bound on the device and reports a violation.)
    const int step = 1 << (h.depth - 1);
    const long long e = static_cast<long long>(std::ceil(cl->max_norm / h.resolution)) + 4;
    auto clampll = [](double v) {
      return static_cast<long long>(std::max(-4e9, std::min(4e9, std::floor(v))));
    };
    const long long c_x = clampll((h.max_y - iy) / h.resolution - 0.5);  // index x <- world y
    const long long c_y = clampll((h.max_x - ix) / h.resolution - 0.5);
    auto span = [&](long long cells, long long c) {
      const long long lin = sp.lin;
      return std::min(lin, std::max<long long>(0, cells - 1 - (c - e))) +
             std::min(lin, std::max<long long>(0, c + e));
    };
    const long long span_x = span(h.nx, c_x), span_y = span(h.ny, c_y);
    const long long cx = (span_x + step) / step, cy = (span_y + step) / step;
    d.cap_y = static_cast<int>(cy);
    d.cap = static_cast<int>(cx * cy);
    d.dscan_off = plan.total_points;
    d.top_off = plan.total_slots;
    plan.total_scans += sp.num_scans;
    plan.total_points += static_cast<long long>(sp.num_scans) * cl->n;
    plan.total_slots += static_cast<long long>(sp.num_scans) * d.cap;
    CSM_REQUIRE(plan.total_scans < (1LL << 30), "too many scans in one batch");
  }
  b.total_scans = static_cast<int>(plan.total_scans);
  for (int j = 0; j < num_jobs; ++j)
    CSM_REQUIRE(b.Stack(j).depth == b.Stack(0).depth,
                "internal: sub-batches are grouped by branch_and_bound_depth");
  b.hmax = b.Stack(0).depth - 1;
  b.top_cap = static_cast<int>(std::min<long long>(plan.total_slots, 1LL << 30));
  // the per-scan tables themselves are written on the device (k_scan_tables)
  b.scan_bases.resize(num_jobs);
  for (int j = 0; j < num_jobs; ++j) b.scan_bases[j] = plan.jobs[j].scan_base;
  return CSM_OK;
}

// Workspaces, the job records' upload and the per-scan tables (k_scan_tables).
csm_status Upload2D(Batch2D& b) {
  Ctx* ctx = b.ctx;
  cudaStream_t s = b.s;
  const int num_jobs = b.num_jobs;
  BatchPlan& plan = b.plan;
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_TRY(ctx->Reserve("trig", sizeof(float2) * b.trig_pairs, &b.d_trig));
  CSM_TRY(ctx->Reserve("jobs", sizeof(JobDev) * num_jobs, &b.d_jobs));
  CSM_TRY(ctx->Reserve("scan_job", sizeof(int) * plan.total_scans, &b.d_scan_job));
  CSM_TRY(ctx->Reserve("slot_base", sizeof(long long) * plan.total_scans, &b.d_slot_base));
  CSM_TRY(ctx->Reserve("info", sizeof(ScanInfo) * plan.total_scans, &b.d_info));
  CSM_TRY(ctx->Reserve("dscan", sizeof(short2) * plan.total_points, &b.d_dscan));
  CSM_TRY(ctx->Reserve("lb", sizeof(unsigned) * num_jobs, &b.d_lb));
  CSM_TRY(ctx->Reserve("counters", sizeof(unsigned long long) * 8 + sizeof(int) * kCtlInts,
                       &b.d_ctr));
  CSM_TRY(ctx->Reserve("job_best", sizeof(int) * num_jobs, &b.d_job_best));
  for (int j = 0; j < num_jobs; ++j) plan.jobs[j].trig = b.d_trig->as<float2>() + b.trig_off[j];

  // uploads go through pinned staging so that they are truly asynchronous (the
  // previous call on this lane has completed: every call ends with a synchronise)
  PinnedBuf& up = ctx->P("upload");
  const size_t up_trig_off = (sizeof(JobDev) * num_jobs + 255) / 256 * 256;
  CSM_TRY(up.Reserve(up_trig_off + sizeof(float2) * b.trig_pairs));
  b.up_trig = reinterpret_cast<float*>(up.as<char>() + up_trig_off);
  std::memcpy(up.as<char>(), plan.jobs.data(), sizeof(JobDev) * num_jobs);
  CSM_CUDA(cudaMemcpyAsync(b.d_jobs->p, up.as<char>(), sizeof(JobDev) * num_jobs,
                           cudaMemcpyHostToDevice, s));
  k_scan_tables<<<num_jobs, 256, 0, s>>>(b.d_jobs->as<JobDev>(), b.d_scan_job->as<int>(),
                                         b.d_slot_base->as<long long>(), b.d_lb->as<unsigned>(),
                                         b.d_job_best->as<int>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemsetAsync(b.d_ctr->p, 0, sizeof(unsigned long long) * 8 + sizeof(int) * kCtlInts, s));
  b.ctr = b.d_ctr->as<unsigned long long>();
  b.ictr = reinterpret_cast<int*>(b.ctr + 8);
  return CSM_OK;
}

// Jobs [j0, j1): the rotation tables they use first are computed into the staging buffer
// and uploaded, then their scans are discretised.
csm_status Discretize2D(Batch2D& b, int j0, int j1) {
  cudaStream_t s = b.s;
  const size_t t0 = b.tables_before[j0], t1 = b.tables_before[j1];
  if (t1 > t0) FillTrigTables(b.trig_tables, t0, t1, b.up_trig);
  // device time counts from the first table upload: the host's table work is not in it
  if (j0 == 0) CSM_CUDA(cudaEventRecord(b.ctx->ev0, s));
  if (t1 > t0) {
    const long long p0 = b.trig_tables[t0].off;
    const long long p1 = t1 < b.trig_tables.size() ? b.trig_tables[t1].off : b.trig_pairs;
    CSM_CUDA(cudaMemcpyAsync(b.d_trig->as<float2>() + p0, b.up_trig + 2 * p0,
                             sizeof(float2) * (p1 - p0), cudaMemcpyHostToDevice, s));
  }
  const int s0 = b.plan.jobs[j0].scan_base, s1 = b.ScanEnd(j1);
  ProfBegin(b.ctx);
  if (s1 > s0) {
    k_discretize<<<s1 - s0, 128, 0, s>>>(b.d_jobs->as<JobDev>(), b.d_scan_job->as<int>(),
                                         b.d_dscan->as<short2>(), b.d_info->as<ScanInfo>(), 1,
                                         b.ctr, s0);
    CSM_LAUNCH_CHECK();
  }
  const long long pt0 = b.plan.jobs[j0].dscan_off;
  const long long pt1 = j1 < b.num_jobs ? b.plan.jobs[j1].dscan_off : b.plan.total_points;
  ProfEnd(b.ctx, "k_discretize", static_cast<double>(pt1 - pt0));
  return CSM_OK;
}

// Tile form of the lowest-resolution pass over scans [s0, s1): persistent warps, exactly the
// resident CTAs, every warp walks (s1 - s0) / warps scans.
csm_status LaunchTile2D(Batch2D& b, int s0, int s1, int tile_words, int lat_ints) {
  const size_t smem = static_cast<size_t>(lat_ints) * 4 * kTileWarps;  // one lattice per warp
#define CSM_TILE(K)                                                                          \
  do {                                                                                       \
    if (smem > 48 * 1024)                                                                    \
      CSM_CUDA(cudaFuncSetAttribute(k_score_top_tile<K>,                                     \
                                    cudaFuncAttributeMaxDynamicSharedMemorySize,             \
                                    static_cast<int>(smem)));                                \
    int per_sm = 0;                                                                          \
    CSM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_score_top_tile<K>,     \
                                                           kTileThreads, smem));             \
    const int grid = std::min(DivUp(s1 - s0, kTileWarps), b.ctx->sm_count * std::max(1, per_sm)); \
    k_score_top_tile<K><<<grid, kTileThreads, smem, b.s>>>(                                  \
        b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(),           \
        b.d_top->as<int>(), b.d_slot_base->as<long long>(), s0, s1, lat_ints);               \
    b.tile_iters = K;                                                                        \
  } while (0)
  if (tile_words <= 32) CSM_TILE(1);
  else if (tile_words <= 64) CSM_TILE(2);
  else if (tile_words <= 96) CSM_TILE(3);
  else CSM_TILE(4);
#undef CSM_TILE
  CSM_LAUNCH_CHECK();
  return CSM_OK;
}

// Discretisation and the lowest-resolution pass in form b.forms.top (nullptr: the size-based
// choice).  Wide lattices (MatchFullSubmap) take the dense decimated-grid kernel; narrow
// ones (local windows: a few dozen candidates per scan) the gather kernel.
csm_status TopPass2D(Batch2D& b) {
  Ctx* ctx = b.ctx;
  const char* force = b.forms.top;
  cudaStream_t s = b.s;
  const int num_jobs = b.num_jobs, total_scans = b.total_scans;
  const BatchPlan& plan = b.plan;
  CSM_TRY(ctx->Reserve("top_sum", sizeof(int) * plan.total_slots, &b.d_top));
  int max_cap = 0, max_cap_x = 0, max_cap_y = 0;
  for (const JobDev& d : plan.jobs) {
    max_cap = std::max(max_cap, d.cap);
    max_cap_y = std::max(max_cap_y, d.cap_y);
    max_cap_x = std::max(max_cap_x, d.cap / std::max(1, d.cap_y));
  }
  bool use_gather_top = max_cap < 128;
  if (force && !strcmp(force, "gather")) use_gather_top = true;
  if (force && !strcmp(force, "dense")) use_gather_top = false;
  // Tile form of the dense pass: needs the whole tile in <= 4 words per lane and the
  // lattice of one scan per warp in shared memory.
  int tile_words = 0;
  for (int j = 0; j < num_jobs; ++j) {
    const StackDev& sh = b.Stack(j);
    const int t = sh.depth - 1;
    tile_words = std::max(tile_words, sh.dec_jd[t] * (sh.dec_ids[t] / 4) + 1);
  }
  const int lat_ints = (max_cap_x + 3) / 4 * 4 * max_cap_y;
  bool use_tile_top = !use_gather_top && tile_words <= 128 && lat_ints * 4 * kTileWarps <= 96 * 1024;
  const int small_lanes = (max_cap_x + 3) / 4 * max_cap_y;  // quads per scan, a-priori bound
  bool use_small_top = small_lanes <= 32;
  if (force && !strcmp(force, "small"))
    CSM_REQUIRE(use_small_top, "form small: more than 32 quads per scan");
  if (force && strcmp(force, "small")) use_small_top = false;
  if (use_small_top) use_gather_top = use_tile_top = false;
  if (force && !strcmp(force, "dense")) use_tile_top = false;
  if (force && !strcmp(force, "tile"))
    CSM_REQUIRE(use_tile_top, "form tile: lattice or tile too large");
  const char* top_name = use_small_top    ? "k_score_top_small"
                         : use_gather_top ? "k_score_top_gather"
                         : use_tile_top   ? "k_score_top_tile" : "k_score_top_dense";
  // The rotation tables of a MatchFullSubmap batch are a libm cos and sin per rotated scan,
  // about 2 ms of host time for 64 searches.  With the tile form, the batch is staged in
  // groups of jobs, each group's tables, discretisation and tile pass before the next
  // group's tables, so the host computes tables while the device scores the groups before.
  // A group takes the device several times longer than its tables take the host, so groups
  // grow 4x and the host stays ahead; the first one is small so that the device starts early.
  std::vector<int> group_end;
  {
    const bool split = use_tile_top && !g_profile_on.load();
    long long prev = 0, acc = 0;
    for (int j = 0; j < num_jobs; ++j) {
      acc += plan.search[j].num_scans;
      if (split && acc >= std::max(4096LL, 4 * prev)) {
        group_end.push_back(j + 1);
        prev = acc;
        acc = 0;
      }
    }
    if (group_end.empty() || group_end.back() != num_jobs) group_end.push_back(num_jobs);
  }
  for (size_t g = 0, j0 = 0; g < group_end.size(); j0 = group_end[g++]) {
    const int j1 = group_end[g];
    CSM_TRY(Discretize2D(b, static_cast<int>(j0), j1));
    if (use_tile_top) {
      ProfBegin(ctx);
      CSM_TRY(LaunchTile2D(b, plan.jobs[j0].scan_base, b.ScanEnd(j1), tile_words, lat_ints));
    }
  }
  b.Phase(use_tile_top ? "upload+discr+top" : "upload+discr");
  if (!use_tile_top) ProfBegin(ctx);
  if (use_small_top) {
    const int spw = 32 / small_lanes;
    k_score_top_small<<<DivUp(DivUp(total_scans, spw), 4), 128, 4 * spw * 32 * sizeof(int2), s>>>(
        b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(),
        b.d_top->as<int>(), b.d_slot_base->as<long long>(), total_scans, small_lanes);
  } else if (use_gather_top) {
    k_score_top_gather<<<DivUp(plan.total_slots * 32, 256), 256, 0, s>>>(
        b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(),
        b.d_top->as<int>(), b.d_slot_base->as<long long>(), total_scans, plan.total_slots);
  } else if (!use_tile_top) {
    const int grid = std::min(total_scans, ctx->sm_count * 128);
    // one quad per thread and extra passes for larger lattices (the real lattice is
    // only known on the device after ShrinkToFit; more quads per thread would execute
    // predicated-off work)
    k_score_top_dense<1><<<grid, kDenseThreads, 0, s>>>(
        b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(),
        b.d_top->as<int>(), b.d_slot_base->as<long long>(), total_scans);
  }
  CSM_LAUNCH_CHECK();
  b.top_kernel = use_small_top ? 1 : use_gather_top ? 2 : use_tile_top ? 3 : 4;
  if (g_profile_on.load()) {
    unsigned long long c3 = 0;
    ProfStop(ctx);
    CSM_CUDA(cudaStreamSynchronize(s));
    CSM_CUDA(cudaMemcpy(&c3, b.ctr + 3, sizeof(c3), cudaMemcpyDeviceToHost));
    ProfCommit(ctx, top_name, static_cast<double>(c3));
  }
  return CSM_OK;
}

// Greedy dives seed the per-job bound.
csm_status Dives2D(Batch2D& b) {
  const int grid = DivUp(static_cast<long long>(b.total_scans) * 32, 256);  // a warp per scan
  if (g_profile_on.load()) b.ProfScored();
  ProfBegin(b.ctx);
  k_job_best<<<grid, 256, 0, b.s>>>(b.d_info->as<ScanInfo>(), b.d_top->as<int>(),
                                    b.d_slot_base->as<long long>(), b.total_scans,
                                    b.d_job_best->as<int>());
  CSM_LAUNCH_CHECK();
  k_dive<<<grid, 256, 0, b.s>>>(
      b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(),
      b.d_top->as<int>(), b.d_slot_base->as<long long>(), b.total_scans, b.d_job_best->as<int>(),
      kDiveRatio, b.d_lb->as<unsigned>(), b.ctr);
  CSM_LAUNCH_CHECK();
  if (g_profile_on.load()) {
    ProfStop(b.ctx);
    ProfCommit(b.ctx, "k_dive", b.ProfScored());
  }
  return CSM_OK;
}

// Queues, leaf lists and the read-back area of the level loop.
csm_status PrepareLevels2D(Batch2D& b) {
  Ctx* ctx = b.ctx;
  const size_t n = static_cast<size_t>(b.total_scans);
  CSM_TRY(ctx->Reserve("queue_top", sizeof(Node) * b.top_cap, &b.d_qtop));
  CSM_TRY(ctx->Reserve("queues", sizeof(Node) * kQueueCap * std::max(1, b.hmax), &b.d_q));
  CSM_TRY(ctx->Reserve("leaves", sizeof(Node) * kLeafCap, &b.d_leaves));
  CSM_TRY(ctx->Reserve("best_leaves", sizeof(Node) * kLeafCap, &b.d_best));
  CSM_TRY(ctx->Reserve("scan_cnt", sizeof(int) * 2 * n, &b.d_scan_cnt));
  CSM_TRY(ctx->Reserve("scan_off", sizeof(int) * (n + 2 * (n / 1024 + 2)), &b.d_scan_off));
  CSM_TRY(ctx->Reserve("work_items", sizeof(WorkItem) * (kChunk / 32 + n + 2), &b.d_items));
  CSM_TRY(ctx->Reserve("sorted_nodes", sizeof(Node) * kChunk, &b.d_sorted));
  b.pin = &ctx->P("readback");
  b.rb_ctr = sizeof(int) * kCtlInts;
  b.rb_lb = b.rb_ctr + sizeof(unsigned long long) * 8;
  b.rb_best = (b.rb_lb + sizeof(unsigned) * b.num_jobs + 15) / 16 * 16;
  CSM_TRY(b.pin->Reserve(b.rb_best + sizeof(Node) * kInlineBest));
  const char* pin = b.pin->as<char>();
  b.hp = reinterpret_cast<const int*>(pin);
  b.hctr = reinterpret_cast<const unsigned long long*>(pin + b.rb_ctr);
  b.lbh = reinterpret_cast<const unsigned*>(pin + b.rb_lb);
  b.best_inline = reinterpret_cast<const Node*>(pin + b.rb_best);
  // The lattice kernel's shared-memory carve-out: just what CSM_LAT_MINB CTAs need, so the
  // rest of the unified L1 caches the window tables, which its loads are bound by.  On an
  // H100 80GB HBM3 (700 W) this took k_expand_lattice from 26.64-26.81 ms per config-2 step
  // with the driver's own choice to 26.42-26.53 ms; the largest carve-out gave 31.1 ms.
  int dev = 0, smem_sm = 0, rsv = 0;
  CSM_CUDA(cudaGetDevice(&dev));
  CSM_CUDA(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
  CSM_CUDA(cudaDeviceGetAttribute(&rsv, cudaDevAttrReservedSharedMemoryPerBlock, dev));
  const int need = CSM_LAT_MINB * (static_cast<int>(sizeof(int2)) * kLatThreads / 32 * kLatChunk + rsv);
  const int pct = std::min(100, DivUp(100LL * need, std::max(1, smem_sm)));
  CSM_CUDA(cudaFuncSetAttribute(k_expand_lattice<4>, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
  CSM_CUDA(cudaFuncSetAttribute(k_expand_lattice<8>, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
  CSM_CUDA(cudaFuncSetAttribute(k_expand_lattice<16>, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
  return CSM_OK;
}

// The lowest-resolution candidates above their job's bound become the top queue (or, with
// a single level, the leaves).
csm_status FilterTop2D(Batch2D& b) {
  const int hmax = b.hmax;
  k_filter_top<<<std::min(b.total_scans, b.ctx->sm_count * 16), 256, 0, b.s>>>(
      b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_top->as<int>(),
      b.d_slot_base->as<long long>(), b.total_scans, b.d_lb->as<unsigned>(), b.Queue(hmax),
      b.ictr + hmax, b.QueueCap(hmax), b.ictr + kCtlOverflow);
  CSM_LAUNCH_CHECK();
  if (hmax == 0) {
    k_top_as_leaves<<<b.ctx->sm_count * 4, 256, 0, b.s>>>(b.d_info->as<ScanInfo>(), b.Queue(0),
                                                          b.ictr, b.d_lb->as<unsigned>(),
                                                          b.d_leaves->as<Node>(), kLeafCap);
    CSM_LAUNCH_CHECK();
  }
  return CSM_OK;
}

// One level step: chunk bookkeeping, grouping by scan, both kernel forms predicated on
// the device-side mode.
csm_status LevelStep2D(Batch2D& b, int h) {
  Ctx* ctx = b.ctx;
  cudaStream_t s = b.s;
  const int total_scans = b.total_scans;
  const int nb = DivUp(total_scans, 1024);
  const int sort_grid = ctx->sm_count * 8;
  const int max_items = kChunk / 32 + std::min(kChunk, total_scans) + 1;
  int* ictr = b.ictr;
  int* scan_cnt = b.d_scan_cnt->as<int>();
  int* cursor = scan_cnt + total_scans;
  int* scan_off = b.d_scan_off->as<int>();
  int* part_a = scan_off + total_scans;   // block sums (DivUp(total_scans, 1024) each)
  int* part_b = part_a + nb;
  Node* next = h - 1 >= 1 ? b.Queue(h - 1) : nullptr;
  int* next_count = ictr + (h - 1 >= 1 ? h - 1 : 31);
  k_level_begin<<<1, 32, 0, s>>>(ictr, h, kChunk, b.forms.lattice_min);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemsetAsync(b.d_scan_cnt->p, 0, sizeof(int) * 2 * total_scans, s));
  ProfBegin(ctx);
  k_q_count<<<sort_grid, 256, 0, s>>>(b.Queue(h), ictr, scan_cnt);
  CSM_LAUNCH_CHECK();
  k_q_block_sums<<<nb, 1024, 0, s>>>(ictr, scan_cnt, total_scans, part_a, part_b);
  CSM_LAUNCH_CHECK();
  k_q_scan_parts<<<1, 1024, 0, s>>>(ictr, part_a, part_b, nb, ictr + kCtlItems);
  CSM_LAUNCH_CHECK();
  k_q_finish<<<nb, 1024, 0, s>>>(ictr, scan_cnt, total_scans, part_a, part_b, scan_off,
                                 b.d_items->as<WorkItem>());
  CSM_LAUNCH_CHECK();
  k_q_scatter<<<sort_grid, 256, 0, s>>>(b.Queue(h), ictr, scan_off, cursor,
                                        b.d_sorted->as<Node>());
  CSM_LAUNCH_CHECK();
  if (g_profile_on.load()) {
    ProfStop(ctx);
    ProfCommit(ctx, "k_q_sort", 0.);
  }
  ProfBegin(ctx);
#define CSM_LATTICE(U)                                                                        \
  k_expand_lattice<U><<<DivUp(max_items, kLatThreads / 32), kLatThreads, 0, s>>>(             \
      b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(),              \
      b.d_sorted->as<Node>(), b.d_items->as<WorkItem>(), ictr + kCtlItems, h,                 \
      b.d_lb->as<unsigned>(), next, next_count, kQueueCap, b.d_leaves->as<Node>(),            \
      ictr + kCtlLeaf, kLeafCap, ictr + kCtlOverflow, b.ctr)
  if (b.forms.unroll <= 4) CSM_LATTICE(4);
  else if (b.forms.unroll <= 8) CSM_LATTICE(8);
  else CSM_LATTICE(16);
#undef CSM_LATTICE
  CSM_LAUNCH_CHECK();
  if (g_profile_on.load()) {
    ProfStop(ctx);
    const double c = b.ProfScored();
    if (c > 0.) ProfCommit(ctx, "k_expand_lattice", c);
  }
  ProfBegin(ctx);
  k_expand<<<kLatticeMin * 32 / 256, 256, 0, s>>>(
      b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(), b.Queue(h),
      ictr, h, b.d_lb->as<unsigned>(), next, next_count, kQueueCap, b.d_leaves->as<Node>(),
      ictr + kCtlLeaf, kLeafCap, ictr + kCtlOverflow, b.ctr);
  CSM_LAUNCH_CHECK();
  if (g_profile_on.load()) {
    ProfStop(ctx);
    const double c = b.ProfScored();
    if (c > 0.) ProfCommit(ctx, "k_expand", c);
  }
  return CSM_OK;
}

// Compaction of the optimal leaves + read-back of everything the host needs.
csm_status Collect2D(Batch2D& b) {
  cudaStream_t s = b.s;
  int* best_count = b.ictr + kCtlBest;
  char* pin = b.pin->as<char>();
  CSM_CUDA(cudaMemsetAsync(best_count, 0, sizeof(int), s));
  k_compact_leaves<<<b.ctx->sm_count * 4, 256, 0, s>>>(
      b.d_info->as<ScanInfo>(), b.d_leaves->as<Node>(), b.ictr + kCtlLeaf, kLeafCap,
      b.d_lb->as<unsigned>(), b.d_best->as<Node>(), best_count, kLeafCap, b.ictr + kCtlOverflow);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaEventRecord(b.ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(pin, b.ictr, b.rb_ctr, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(pin + b.rb_ctr, b.ctr, sizeof(unsigned long long) * 8,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(pin + b.rb_lb, b.d_lb->p, sizeof(unsigned) * b.num_jobs,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(pin + b.rb_best, b.d_best->p, sizeof(Node) * kInlineBest,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  ++b.host_syncs;
  return CSM_OK;
}

// The sweep hmax -> 1, then (frontiers larger than one chunk, rare) continuation sweeps
// from the deepest non-empty level, each ended by a collect.
csm_status Sweep2D(Batch2D& b) {
  for (int h = b.hmax; h >= 1; --h) CSM_TRY(LevelStep2D(b, h));
  CSM_TRY(Collect2D(b));
  for (;;) {
    if (b.hp[kCtlOverflow]) {
      SetError("branch-and-bound queue overflow (more than 2^22 tied optimal leaves, or more "
               "than 2^30 lowest-resolution candidates in one batch)");
      return CSM_E_CAPACITY;
    }
    int h = -1;
    for (int l = 1; l <= b.hmax; ++l)
      if (b.hp[l] > 0) { h = l; break; }
    if (h < 0) break;
    if (b.hp[kCtlLeaf] > kLeafCap / 2) {
      // drop the leaves that are already below their job's bound (d_best holds them
      // after Collect2D); more than kLeafCap / 2 exactly tied optima are not supported
      if (b.hp[kCtlBest] > kLeafCap / 2) { SetError("too many tied leaves"); return CSM_E_CAPACITY; }
      CSM_CUDA(cudaMemcpyAsync(b.d_leaves->p, b.d_best->p, sizeof(Node) * b.hp[kCtlBest],
                               cudaMemcpyDeviceToDevice, b.s));
      CSM_CUDA(cudaMemcpyAsync(b.ictr + kCtlLeaf, b.ictr + kCtlBest, sizeof(int),
                               cudaMemcpyDeviceToDevice, b.s));
    }
    CSM_TRY(LevelStep2D(b, h));
    for (int l = h - 1; l >= 1; --l) CSM_TRY(LevelStep2D(b, l));  // its children fit one chunk each
    CSM_TRY(Collect2D(b));
  }
  return CSM_OK;
}

// Tie resolution of job j: the reference returns the first optimal leaf in DFS order, which
// is moved to ties[0].  h_info holds every scan's ScanInfo.
csm_status ResolveTies2D(Batch2D& b, int j, const std::vector<ScanInfo>& h_info,
                         std::vector<TieLeaf>& ties, int* host_resolves) {
  cudaStream_t s = b.s;
  const int hmax = b.hmax;
  const int T = static_cast<int>(ties.size());
  // ancestor scores at levels 1..hmax
  std::vector<ListCand> lc;
  lc.reserve(static_cast<size_t>(T) * hmax);
  for (const TieLeaf& t : ties) {
    const ScanInfo& si = h_info[t.scan];
    for (int l = 1; l <= hmax; ++l) {
      const int ax = si.min_x + (((t.xo - si.min_x) >> l) << l);
      const int ay = si.min_y + (((t.yo - si.min_y) >> l) << l);
      lc.push_back(ListCand{t.scan, ax, ay, l});
    }
  }
  std::vector<float> anc(lc.size());
  if (!lc.empty()) {
    DevBuf *d_lc, *d_ls;
    CSM_TRY(b.ctx->Reserve("tie_cands", sizeof(ListCand) * lc.size(), &d_lc));
    CSM_TRY(b.ctx->Reserve("tie_scores", sizeof(float) * lc.size(), &d_ls));
    CSM_CUDA(cudaMemcpyAsync(d_lc->p, lc.data(), sizeof(ListCand) * lc.size(),
                             cudaMemcpyHostToDevice, s));
    k_score_list<<<DivUp(static_cast<long long>(lc.size()) * 32, 256), 256, 0, s>>>(
        b.d_jobs->as<JobDev>(), b.d_info->as<ScanInfo>(), b.d_dscan->as<short2>(),
        d_lc->as<ListCand>(), static_cast<int>(lc.size()), nullptr, d_ls->as<float>());
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cudaMemcpyAsync(anc.data(), d_ls->p, sizeof(float) * lc.size(),
                             cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaStreamSynchronize(s));
  }
  const JobDev& jd = b.plan.jobs[j];
  // lazily computed rank of every lowest-resolution candidate of this job in
  // the reference's std::sort order (fast...2d.cc:331-332)
  std::vector<int> top_rank;
  std::vector<long long> scan_first;  // first generation index of each scan
  auto ensure_top_rank = [&]() -> csm_status {
    if (!top_rank.empty()) return CSM_OK;
    ++*host_resolves;
    std::vector<int> sums(static_cast<size_t>(jd.num_scans) * jd.cap);
    CSM_CUDA(cudaMemcpy(sums.data(), b.d_top->as<int>() + jd.top_off, sizeof(int) * sums.size(),
                        cudaMemcpyDeviceToHost));
    const StackDev& sh = b.Stack(j);
    struct Item { float score; int gen; };
    std::vector<Item> items;
    scan_first.assign(jd.num_scans, 0);
    for (int k = 0; k < jd.num_scans; ++k) {
      const ScanInfo& si = h_info[jd.scan_base + k];
      scan_first[k] = static_cast<long long>(items.size());
      for (int q = 0; q < si.nxc * si.nyc; ++q) {
        const float mean = static_cast<float>(sums[static_cast<size_t>(k) * jd.cap + q]) /
                           static_cast<float>(jd.n);
        items.push_back(Item{sh.min_score + mean * sh.k255, static_cast<int>(items.size())});
      }
    }
    std::sort(items.begin(), items.end(),
              [](const Item& a, const Item& b) { return a.score > b.score; });
    top_rank.resize(items.size());
    for (size_t r = 0; r < items.size(); ++r) top_rank[items[r].gen] = static_cast<int>(r);
    return CSM_OK;
  };
  // returns true if leaf a precedes leaf b in the reference's DFS order
  csm_status err = CSM_OK;
  auto before = [&](int a, int b) -> bool {
    const TieLeaf& A = ties[a];
    const TieLeaf& B = ties[b];
    const ScanInfo& sa = h_info[A.scan];
    const ScanInfo& sb = h_info[B.scan];
    for (int l = hmax; l >= 0; --l) {
      const int ax = (A.xo - sa.min_x) >> l, ay = (A.yo - sa.min_y) >> l;
      const int bx = (B.xo - sb.min_x) >> l, by = (B.yo - sb.min_y) >> l;
      if (A.scan == B.scan && ax == bx && ay == by) continue;  // same ancestor
      const float fa = l == 0 ? 0.f : anc[static_cast<size_t>(a) * hmax + (l - 1)];
      const float fb = l == 0 ? 0.f : anc[static_cast<size_t>(b) * hmax + (l - 1)];
      if (l > 0 && fa != fb) return fa > fb;
      if (l == hmax) {
        // equal lowest-resolution scores: replay the reference's std::sort
        if (ensure_top_rank() != CSM_OK) { err = CSM_E_CUDA; return false; }
        const long long ga = scan_first[A.scan - jd.scan_base] + static_cast<long long>(ax) * sa.nyc + ay;
        const long long gb = scan_first[B.scan - jd.scan_base] + static_cast<long long>(bx) * sb.nyc + by;
        return top_rank[ga] < top_rank[gb];
      }
      // siblings: stable insertion sort keeps generation order (x outer, y inner)
      if ((ax & 1) != (bx & 1)) return (ax & 1) < (bx & 1);
      return (ay & 1) < (by & 1);
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

// Results of every job from its first optimal leaf, and the call's statistics.
void Results2D(const Batch2D& b, const std::vector<std::vector<TieLeaf>>& per_job,
               int host_resolves, csm_result2d* results, csm_stats* total) {
  for (int j = 0; j < b.num_jobs; ++j) {
    csm_result2d& r = results[j];
    const float best_score = HostOrderedToFloat(b.lbh[j]);
    r.found = 0;
    r.leaves_tied = static_cast<int32_t>(per_job[j].size());
    if (!per_job[j].empty() && best_score > b.jobs[j].min_score) {
      const TieLeaf& t = per_job[j][0];
      const JobDev& jd = b.plan.jobs[j];
      const HostSearch& sp = b.plan.search[j];
      const double res = b.Stack(j).resolution;
      const int scan_index = t.scan - jd.scan_base;
      // Candidate2D (corr...2d.h:77-86): x = -y_off * res, y = -x_off * res
      const double cx = -t.yo * res, cy = -t.xo * res;
      const double orientation = (scan_index - sp.num_angular) * sp.step;
      r.found = 1;
      r.score = best_score;
      r.pose_estimate[0] = b.plan.init_x[j] + cx;
      r.pose_estimate[1] = b.plan.init_y[j] + cy;
      r.pose_estimate[2] = b.plan.init_theta[j] + orientation;
      r.best_scan_index = scan_index;
      r.best_x_offset = t.xo;
      r.best_y_offset = t.yo;
    }
  }
  if (!total) return;
  float ms = 0.f;
  cudaEventElapsedTime(&ms, b.ctx->ev0, b.ctx->ev1);
  total->candidates_scored += static_cast<int64_t>(b.hctr[0]);
  total->nodes_expanded += static_cast<int64_t>(b.hctr[1]);
  total->lowest_resolution_candidates += static_cast<long long>(b.hctr[3]);
  total->host_tie_resolves += host_resolves;
  total->host_syncs += b.host_syncs;
  total->device_ms += ms;
  if (b.num_jobs == 1) {
    total->num_scans = b.plan.search[0].num_scans;
    total->leaves_tied = results[0].leaves_tied;
    total->best_scan_index = results[0].best_scan_index;
    total->best_x_offset = results[0].best_x_offset;
    total->best_y_offset = results[0].best_y_offset;
  }
}

// Runs a batch of independent matches of one branch_and_bound_depth; `search` holds the
// jobs' searches.
csm_status MatchBatch2D(Batch2D& b, const HostSearch* search, csm_result2d* results,
                        csm_stats* total) {
  CSM_TRY(Plan2D(b, search));
  b.Phase("host plan");
  CSM_TRY(Upload2D(b));
  CSM_TRY(TopPass2D(b));
  b.Phase("top pass");
  CSM_TRY(Dives2D(b));
  b.Phase("dives");
  CSM_TRY(PrepareLevels2D(b));
  CSM_TRY(FilterTop2D(b));
  CSM_TRY(Sweep2D(b));
  b.Phase("branch&bound");
  const int n_best = b.hp[kCtlBest];
  if (b.hctr[7]) {
    SetError("a scan point lies more than 30000 cells from the grid origin (int16 cell indices)");
    return CSM_E_CAPACITY;
  }
  if (b.hctr[6]) {
    SetError("internal: a scan's lowest-resolution lattice exceeds its reserved slots");
    return CSM_E_CAPACITY;
  }
  std::vector<Node> best(b.best_inline, b.best_inline + std::min(n_best, kInlineBest));
  if (n_best > kInlineBest) {  // many exactly tied optima
    best.resize(n_best);
    CSM_CUDA(cudaMemcpyAsync(best.data(), b.d_best->p, sizeof(Node) * n_best,
                             cudaMemcpyDeviceToHost, b.s));
    CSM_CUDA(cudaStreamSynchronize(b.s));
    ++b.host_syncs;
  }
  // group optimal leaves by job
  std::vector<std::vector<TieLeaf>> per_job(b.num_jobs);
  for (const Node& nd : best) per_job[b.JobOfScan(nd.scan)].push_back(TieLeaf{nd.scan, nd.xo, nd.yo});
  int host_resolves = 0;
  std::vector<ScanInfo> h_info;
  for (int j = 0; j < b.num_jobs; ++j) {
    if (per_job[j].size() <= 1) continue;
    if (h_info.empty()) {
      h_info.resize(b.total_scans);
      CSM_CUDA(cudaMemcpy(h_info.data(), b.d_info->p, sizeof(ScanInfo) * b.total_scans,
                          cudaMemcpyDeviceToHost));
    }
    CSM_TRY(ResolveTies2D(b, j, h_info, per_job[j], &host_resolves));
  }
  b.Phase("collect+ties");
  Results2D(b, per_job, host_resolves, results, total);
  return CSM_OK;
}

// One test-hook call: the one-job batch csm_match2d would run with the same arguments.
struct Hook2D {
  const csm_stack2d* stack = nullptr;
  csm_cloud* cloud = nullptr;
  csm_job2d job;
  HostSearch search;
  LaneGuard guard;
  Batch2D b;
  ~Hook2D() {  // a call that failed after a launch must not pool the cloud while it is read
    if (guard.lane) cudaStreamSynchronize(guard.lane->stream);
    csm_cloud_destroy(cloud);
  }
};

// The hook's cloud, job and search.
csm_status MakeHook2D(Hook2D& hk, const csm_stack2d* stack, const float* xyz, int32_t n,
                      const double initial_pose[3], int32_t full_submap, double linear_window,
                      double angular_window, float min_score) {
  CSM_REQUIRE(stack && xyz, "null pointer");
  hk.stack = stack;
  CSM_TRY(csm_cloud_create(xyz, n, stack->ctx->device, &hk.cloud));
  std::memset(&hk.job, 0, sizeof(hk.job));
  hk.job.full_submap = full_submap;
  if (initial_pose) std::memcpy(hk.job.initial_pose, initial_pose, sizeof(double) * 3);
  hk.job.min_score = min_score;
  hk.search = JobSearch(stack, hk.cloud, hk.job, linear_window, angular_window);
  return CSM_OK;
}

// Plans the hook's batch on a lane; nothing is launched yet.
csm_status PlanHook2D(Hook2D& hk, const Forms2D& forms) {
  CSM_TRY(AcquireLane(hk.stack->ctx->device, &hk.guard));
  hk.b = Batch2D(hk.guard.lane, &hk.stack, &hk.cloud, &hk.job, 1, forms);
  return Plan2D(hk.b, &hk.search);
}

// Every scan's ScanInfo, after the work queued so far (one synchronise).
csm_status ReadInfo2D(const Batch2D& b, std::vector<ScanInfo>* info) {
  info->resize(b.total_scans);
  CSM_CUDA(cudaMemcpyAsync(info->data(), b.d_info->p, sizeof(ScanInfo) * b.total_scans,
                           cudaMemcpyDeviceToHost, b.s));
  CSM_CUDA(cudaStreamSynchronize(b.s));
  return CSM_OK;
}

}  // namespace

extern "C" {

csm_status csm_match2d_batch(const csm_stack2d* const* stacks, int32_t num_stacks,
                             const csm_cloud* const* clouds, int32_t num_clouds,
                             const csm_job2d* jobs, int32_t num_jobs, double linear_window,
                             double angular_window, csm_result2d* results, csm_stats* total) {
  CSM_REQUIRE(stacks && clouds && jobs && results, "null pointer");
  CSM_REQUIRE(num_jobs >= 1 && num_stacks >= 1 && num_clouds >= 1, "empty batch");
  CSM_REQUIRE(stacks[0] != nullptr, "null stack");
  bool one_depth = true;
  for (int j = 0; j < num_jobs; ++j) {
    const csm_job2d& jb = jobs[j];
    CSM_REQUIRE(jb.stack_index >= 0 && jb.stack_index < num_stacks, "stack index");
    CSM_REQUIRE(jb.cloud_index >= 0 && jb.cloud_index < num_clouds, "cloud index");
    CSM_REQUIRE(stacks[jb.stack_index] && clouds[jb.cloud_index], "null handle");
    one_depth = one_depth &&
                stacks[jb.stack_index]->h.depth == stacks[jobs[0].stack_index]->h.depth;
  }
  static const Forms2D env_forms{nullptr, getenv("CSM_NO_LATTICE") ? INT_MAX : kLatticeMin,
                                 getenv("CSM_LAT_UNROLL") ? atoi(getenv("CSM_LAT_UNROLL")) : 8};
  LaneGuard guard;
  CSM_TRY(AcquireLane(stacks[0]->ctx->device, &guard));
  Ctx* ctx = guard.lane;
  if (total) std::memset(total, 0, sizeof(*total));
  // Runs jobs[0..n) (one branch_and_bound_depth) in sub-batches whose discrete-scan buffer
  // stays below ~4 GB.
  auto run = [&](const csm_job2d* js, int n, csm_result2d* rs) -> csm_status {
    const long long kMaxPoints = 1LL << 30;
    std::vector<HostSearch> search(n);
    for (int j = 0; j < n; ++j)
      search[j] = JobSearch(stacks[js[j].stack_index], clouds[js[j].cloud_index], js[j],
                            linear_window, angular_window);
    int j0 = 0;
    while (j0 < n) {
      long long pts = 0;
      int j1 = j0;
      while (j1 < n) {
        const long long add =
            static_cast<long long>(search[j1].num_scans) * clouds[js[j1].cloud_index]->n;
        if (j1 > j0 && pts + add > kMaxPoints) break;
        pts += add;
        ++j1;
      }
      Batch2D b(ctx, stacks, clouds, js + j0, j1 - j0, env_forms);
      CSM_TRY(MatchBatch2D(b, search.data() + j0, rs + j0, total));
      j0 = j1;
    }
    return CSM_OK;
  };
  if (one_depth) return run(jobs, num_jobs, results);
  // Stacks of different branch_and_bound_depth (the level loop is per depth): one pass per
  // depth, results scattered back into job order.
  std::map<int, std::vector<int>> by_depth;
  for (int j = 0; j < num_jobs; ++j) by_depth[stacks[jobs[j].stack_index]->h.depth].push_back(j);
  for (const auto& kv : by_depth) {
    const std::vector<int>& idx = kv.second;
    std::vector<csm_job2d> js(idx.size());
    std::vector<csm_result2d> rs(idx.size());
    for (size_t i = 0; i < idx.size(); ++i) js[i] = jobs[idx[i]];
    CSM_TRY(run(js.data(), static_cast<int>(js.size()), rs.data()));
    for (size_t i = 0; i < idx.size(); ++i) results[idx[i]] = rs[i];
  }
  return CSM_OK;
}

csm_status csm_match2d(const csm_stack2d* stack, const float* xyz, int32_t n,
                       const double initial_pose[3], int32_t full_submap, double linear_window,
                       double angular_window, float min_score, int32_t* found, float* score,
                       double pose_estimate[3], csm_stats* stats) {
  CSM_REQUIRE(stack && xyz && found && score && pose_estimate, "null pointer");  // :232-233
  CSM_REQUIRE(full_submap || initial_pose, "null initial pose");
  csm_cloud* cloud = nullptr;
  CSM_TRY(csm_cloud_create(xyz, n, stack->ctx->device, &cloud));
  csm_job2d job;
  std::memset(&job, 0, sizeof(job));
  job.full_submap = full_submap;
  if (initial_pose) std::memcpy(job.initial_pose, initial_pose, sizeof(double) * 3);
  job.min_score = min_score;
  csm_result2d res;
  std::memset(&res, 0, sizeof(res));
  const csm_cloud* cl = cloud;
  const csm_status st = csm_match2d_batch(&stack, 1, &cl, 1, &job, 1, linear_window,
                                          angular_window, &res, stats);
  csm_cloud_destroy(cloud);
  if (st != CSM_OK) return st;
  *found = res.found;
  if (res.found) {
    *score = res.score;
    std::memcpy(pose_estimate, res.pose_estimate, sizeof(double) * 3);
  }
  return CSM_OK;
}

csm_status csm_discretize2d(const csm_stack2d* stack, const float* xyz, int32_t n,
                            const double initial_pose[3], int32_t full_submap,
                            double linear_window, double angular_window, int32_t* num_scans,
                            int32_t* discrete_scans, int32_t* bounds) {
  CSM_REQUIRE(num_scans, "null pointer");
  Hook2D hk;
  CSM_TRY(MakeHook2D(hk, stack, xyz, n, initial_pose, full_submap, linear_window, angular_window,
                     0.f));
  *num_scans = hk.search.num_scans;
  if (!discrete_scans && !bounds) return CSM_OK;
  CSM_TRY(PlanHook2D(hk, Forms2D()));
  Batch2D& b = hk.b;
  CSM_TRY(Upload2D(b));
  CSM_TRY(Discretize2D(b, 0, 1));
  std::vector<short2> h_ds(discrete_scans ? b.plan.total_points : 0);
  if (discrete_scans)
    CSM_CUDA(cudaMemcpyAsync(h_ds.data(), b.d_dscan->p, sizeof(short2) * h_ds.size(),
                             cudaMemcpyDeviceToHost, b.s));
  std::vector<ScanInfo> info;
  CSM_TRY(ReadInfo2D(b, &info));
  for (size_t i = 0; i < h_ds.size(); ++i) {
    discrete_scans[2 * i] = h_ds[i].x;
    discrete_scans[2 * i + 1] = h_ds[i].y;
  }
  for (int i = 0; bounds && i < b.total_scans; ++i) {
    const int32_t v[4] = {info[i].min_x, info[i].max_x, info[i].min_y, info[i].max_y};
    std::memcpy(bounds + 4 * i, v, sizeof(v));
  }
  return CSM_OK;
}

csm_status csm_score_top2d(const csm_stack2d* stack, const float* xyz, int32_t n,
                           const double initial_pose[3], int32_t full_submap,
                           double linear_window, double angular_window, int32_t form,
                           int32_t* num_scans, int32_t* slots_per_scan, int32_t* sums,
                           int32_t* lattices, int32_t* kernel) {
  static const char* const kForms[] = {nullptr, "small", "gather", "tile", "dense"};
  CSM_REQUIRE(num_scans && slots_per_scan, "null pointer");
  CSM_REQUIRE(form >= 0 && form <= 4, "form");
  CSM_REQUIRE(full_submap || initial_pose, "null initial pose");
  Hook2D hk;
  CSM_TRY(MakeHook2D(hk, stack, xyz, n, initial_pose, full_submap, linear_window, angular_window,
                     0.f));
  Forms2D forms;
  forms.top = kForms[form];
  CSM_TRY(PlanHook2D(hk, forms));
  Batch2D& b = hk.b;
  CSM_TRY(Upload2D(b));
  CSM_TRY(TopPass2D(b));
  unsigned long long err[2] = {0, 0};
  CSM_CUDA(cudaMemcpyAsync(err, b.ctr + 6, sizeof(err), cudaMemcpyDeviceToHost, b.s));
  std::vector<ScanInfo> info;
  CSM_TRY(ReadInfo2D(b, &info));
  if (err[0] || err[1]) {
    SetError("a scan's lattice or cell indices exceed the engine's limits");
    return CSM_E_CAPACITY;
  }
  if (sums)
    CSM_CUDA(cudaMemcpy(sums, b.d_top->p, sizeof(int) * b.plan.total_slots, cudaMemcpyDeviceToHost));
  *num_scans = b.total_scans;
  *slots_per_scan = b.plan.jobs[0].cap;
  for (int i = 0; lattices && i < b.total_scans; ++i) {
    const ScanInfo& si = info[i];
    const int32_t v[6] = {si.min_x, si.max_x, si.min_y, si.max_y, si.nxc, si.nyc};
    std::memcpy(lattices + 6 * i, v, sizeof(v));
  }
  if (kernel) {
    kernel[0] = b.top_kernel;
    kernel[1] = b.tile_iters;
  }
  return CSM_OK;
}

csm_status csm_branch_step2d(const csm_stack2d* stack, const float* xyz, int32_t n,
                             const double initial_pose[3], int32_t full_submap,
                             double linear_window, double angular_window, float min_score,
                             int32_t level, const csm_node2d* parents, int32_t num_parents,
                             float bound, int32_t form, int32_t unroll, csm_node2d* children,
                             int32_t* num_children, float* final_bound, int64_t counters[2]) {
  static_assert(sizeof(csm_node2d) == sizeof(Node), "csm_node2d is Node");
  CSM_REQUIRE(children && num_children && final_bound && counters, "null pointer");
  CSM_REQUIRE(parents || num_parents == 0, "null parents");
  CSM_REQUIRE(level >= 1, "level out of range");
  CSM_REQUIRE(form == 0 || form == 1, "form");
  CSM_REQUIRE(unroll == 4 || unroll == 8 || unroll == 16, "unroll");
  CSM_REQUIRE(full_submap || initial_pose, "null initial pose");
  Hook2D hk;
  CSM_TRY(MakeHook2D(hk, stack, xyz, n, initial_pose, full_submap, linear_window, angular_window,
                     min_score));
  Forms2D forms;
  forms.lattice_min = form == 1 ? 1 : INT_MAX;
  forms.unroll = unroll;
  CSM_TRY(PlanHook2D(hk, forms));
  Batch2D& b = hk.b;
  cudaStream_t s = b.s;
  const int h = level;
  CSM_REQUIRE(h <= b.hmax, "level out of range");
  CSM_REQUIRE(num_parents >= 0 && num_parents <= std::min(b.QueueCap(h), kChunk),
              "number of parents");
  // the batch's own launches up to the level loop, whose state is then reset to the
  // caller's parents for one level step
  CSM_TRY(Upload2D(b));
  CSM_TRY(TopPass2D(b));
  CSM_TRY(PrepareLevels2D(b));
  std::vector<ScanInfo> info;
  CSM_TRY(ReadInfo2D(b, &info));
  for (int i = 0; i < num_parents; ++i) {
    const csm_node2d& p = parents[i];
    CSM_REQUIRE(p.scan_index >= 0 && p.scan_index < b.total_scans, "parent scan_index");
    const ScanInfo& si = info[p.scan_index];
    const int dx = p.x_index_offset - si.min_x, dy = p.y_index_offset - si.min_y;
    CSM_REQUIRE(dx >= 0 && dy >= 0 && (dx & ((1 << h) - 1)) == 0 && (dy & ((1 << h) - 1)) == 0 &&
                p.x_index_offset <= si.max_x && p.y_index_offset <= si.max_y,
                "parent is not a node of its scan's level lattice");
  }
  const unsigned lb_in = HostFloatToOrdered(bound);
  CSM_CUDA(cudaMemsetAsync(b.ictr, 0, sizeof(int) * kCtlInts, s));
  CSM_CUDA(cudaMemsetAsync(b.ctr, 0, sizeof(unsigned long long) * 2, s));
  CSM_CUDA(cudaMemcpyAsync(b.ictr + h, &num_parents, sizeof(int), cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(b.d_lb->p, &lb_in, sizeof(unsigned), cudaMemcpyHostToDevice, s));
  if (num_parents)
    CSM_CUDA(cudaMemcpyAsync(b.Queue(h), parents, sizeof(Node) * num_parents,
                             cudaMemcpyHostToDevice, s));
  CSM_TRY(LevelStep2D(b, h));
  int ctl[kCtlInts];
  unsigned long long c[8];
  unsigned lb_out = 0;
  CSM_CUDA(cudaMemcpyAsync(ctl, b.ictr, sizeof(ctl), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(c, b.ctr, sizeof(c), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(&lb_out, b.d_lb->p, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  if (c[6] || c[7]) {
    SetError("a scan's lattice or cell indices exceed the engine's limits");
    return CSM_E_CAPACITY;
  }
  const int cnt = h >= 2 ? ctl[h - 1] : ctl[kCtlLeaf];
  if (ctl[kCtlOverflow] || cnt > 4 * num_parents) {
    SetError("internal: more children than 4 per parent");
    return CSM_E_CAPACITY;
  }
  if (cnt)
    CSM_CUDA(cudaMemcpy(children, h >= 2 ? b.Queue(h - 1) : b.d_leaves->as<Node>(),
                        sizeof(Node) * cnt, cudaMemcpyDeviceToHost));
  *num_children = cnt;
  *final_bound = HostOrderedToFloat(lb_out);
  counters[0] = static_cast<int64_t>(c[0]);
  counters[1] = static_cast<int64_t>(c[1]);
  return CSM_OK;
}

csm_status csm_score_candidates2d(const csm_stack2d* stack, int32_t level,
                                  const int32_t* discrete_scans, int32_t num_scans,
                                  int32_t n, const int32_t* candidates, int32_t num_candidates,
                                  float* scores, int32_t* sums) {
  CSM_REQUIRE(stack && discrete_scans && candidates && scores, "null pointer");
  CSM_REQUIRE(level >= 0 && level < stack->h.depth, "level out of range");
  CSM_REQUIRE(num_scans >= 1 && n >= 1 && num_candidates >= 0, "sizes");
  if (num_candidates == 0) return CSM_OK;
  LaneGuard guard;
  CSM_TRY(AcquireLane(stack->ctx->device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  // one synthetic job whose discrete scans are supplied by the caller
  JobDev jd;
  std::memset(&jd, 0, sizeof(jd));
  jd.stack = stack->d;
  jd.n = n;
  jd.num_scans = num_scans;
  std::vector<ScanInfo> info(num_scans);
  for (int k = 0; k < num_scans; ++k) {
    std::memset(&info[k], 0, sizeof(ScanInfo));
    info[k].job = 0;
  }
  std::vector<ListCand> lc(num_candidates);
  for (int c = 0; c < num_candidates; ++c) {
    CSM_REQUIRE(candidates[3 * c] >= 0 && candidates[3 * c] < num_scans, "scan_index");
    lc[c] = ListCand{candidates[3 * c], candidates[3 * c + 1], candidates[3 * c + 2], level};
  }
  DevBuf *d_jobs, *d_info, *d_dscan, *d_lc, *d_sc, *d_su;
  const size_t npts = static_cast<size_t>(num_scans) * n;
  CSM_TRY(ctx->Reserve("hook_jobs", sizeof(JobDev), &d_jobs));
  CSM_TRY(ctx->Reserve("hook_info", sizeof(ScanInfo) * num_scans, &d_info));
  CSM_TRY(ctx->Reserve("hook_dscan", sizeof(short2) * npts, &d_dscan));
  std::vector<short2> h_ds(npts);
  for (size_t i = 0; i < npts; ++i)
    h_ds[i] = make_short2(
        static_cast<short>(std::max(-30000, std::min(30000, discrete_scans[2 * i]))),
        static_cast<short>(std::max(-30000, std::min(30000, discrete_scans[2 * i + 1]))));
  CSM_TRY(ctx->Reserve("hook_cands", sizeof(ListCand) * num_candidates, &d_lc));
  CSM_TRY(ctx->Reserve("hook_scores", sizeof(float) * num_candidates, &d_sc));
  CSM_TRY(ctx->Reserve("hook_sums", sizeof(int) * num_candidates, &d_su));
  CSM_CUDA(cudaMemcpyAsync(d_jobs->p, &jd, sizeof(jd), cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(d_info->p, info.data(), sizeof(ScanInfo) * num_scans,
                           cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(d_dscan->p, h_ds.data(), sizeof(short2) * npts,
                           cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(d_lc->p, lc.data(), sizeof(ListCand) * num_candidates,
                           cudaMemcpyHostToDevice, s));
  k_score_list<<<DivUp(static_cast<long long>(num_candidates) * 32, 256), 256, 0, s>>>(
      d_jobs->as<JobDev>(), d_info->as<ScanInfo>(), d_dscan->as<short2>(), d_lc->as<ListCand>(),
      num_candidates, d_su->as<int>(), d_sc->as<float>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(scores, d_sc->p, sizeof(float) * num_candidates,
                           cudaMemcpyDeviceToHost, s));
  if (sums)
    CSM_CUDA(cudaMemcpyAsync(sums, d_su->p, sizeof(int) * num_candidates, cudaMemcpyDeviceToHost,
                             s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

}  // extern "C"
