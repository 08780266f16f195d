// RealTimeCorrelativeScanMatcher2D::Match on the device
// (cartographer/mapping/internal/2d/scan_matching/real_time_correlative_scan_matcher_2d.cc:61-176).
//
// Shape of the work: for every rotated scan the candidates are the (2L+1)^2 integer
// offsets of a small window, and every candidate's score is an ORDERED float32 sum of
// one probability per scan point (:64-72).  One WARP owns one (job, rotated scan):
//   * the lanes discretise 32 scan points at a time (rotate, translate, GetCellIndex —
//     the same float / double expression order as the reference) and hand them round
//     with warp shuffles, so neither the rotated scans nor their cell indices ever
//     touch global memory;
//   * lane r accumulates candidate r of the window in point order (4 independent
//     candidates per lane for windows of more than 32 offsets);
//   * the probability grid (or the part of it the scan can reach) is staged ONCE per
//     CTA into shared memory by the TMA engine: one cp.async.bulk.tensor.2d of a
//     (BW x BH) uint16 box, completion signalled through an mbarrier; gathers then hit
//     shared memory (a 5 x 5 window of one point is 5 rows of <= 3 words: no bank
//     conflicts).  Grids / reach areas larger than the box use the same kernel with
//     read-only global gathers instead;
//   * score * exp(-(...)^2) (:170-174): the exp / hypot factors are evaluated in double
//     on the host with libm (like every transcendental of the path; DESIGN.md
//     §Numerics) — one value per (|scan - n|, {|xo|, |yo|}) class — and multiplied in
//     double on the device;
//   * std::max_element's "first maximum in generation order" (:142-143) becomes a 64-bit
//     atomicMax of (score bits << 32 | ~candidate index) per job.
// Many scans per call (csm_rt_match2d_batch) share one grid-resident handle
// (csm_rt_grid2d); a persistent grid of CTAs walks the (job, scan) items.
#include <cuda.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <thread>

#include "engine2d.cuh"
#include "rtgrid.cuh"

namespace csm {

constexpr int kRtThreads = 256;
constexpr int kRtWarps = kRtThreads / 32;
// candidates per lane and pass: 1 for windows of <= 32 offsets (the default +-0.1 m window
// has 25), 4 for larger ones — a template parameter, so the common case carries no
// predicated-off accumulator code (executing all four costs several times the instructions
// per warp and point)
constexpr int kRtTileBytes = 100 * 1024;     // staged box (2 CTAs in an H100 SM's 228 KB)

struct RtParams {
  int lin, width, per_scan, npair;
  float k_scale, cost_bias, max_cost, min_probability;
  // TSDF variant: value -> tsd / weight (tsd_value_converter.cc:24-34)
  float tsd_scale, tsd_bias, min_tsd, w_scale, w_bias, truncation;
};

struct RtJobDev {
  long long xyz_off;   // first float of the job's (pre-rotated) cloud
  int trig_off;        // first float2 of the job's rotation table
  int w_off;           // first double of the job's weight table
  int n, num_scans, num_angular;
  int item_base;       // index of the job's scan 0 among all (job, scan) items
  float tx, ty;        // Translation2f(initial translation)
  int x0, y0;          // origin of the staged box in grid cells (shared-memory form)
};

// ---- mbarrier / TMA wrappers (PTX ISA: mbarrier, cp.async.bulk.tensor) -------------
__device__ __forceinline__ unsigned SmemAddr(const void* p) {
  return static_cast<unsigned>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void MbarInit(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(SmemAddr(bar)), "r"(count));
}
__device__ __forceinline__ void MbarExpectTx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(SmemAddr(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void MbarWait(uint64_t* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(SmemAddr(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void TmaLoad2D(void* dst, const CUtensorMap* map, int x, int y,
                                          uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%2, %3}], [%4];" ::"r"(SmemAddr(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(SmemAddr(bar))
      : "memory");
}

// Eigen quaternion * vector for a rotation about z (transform/rigid_transform.h:192-196):
// q = (w, 0, 0, s).  Same operation order as engine2d.cu's RotateRn.
__device__ __forceinline__ void RotateZ(float w, float s, float vx, float vy, float vz, float& ox,
                                        float& oy) {
  const float qx = __fmul_rn(s, 0.f), qy = __fmul_rn(s, 0.f), qz = __fmul_rn(s, 1.f);
  float ux = __fsub_rn(__fmul_rn(qy, vz), __fmul_rn(qz, vy));
  float uy = __fsub_rn(__fmul_rn(qz, vx), __fmul_rn(qx, vz));
  float uz = __fsub_rn(__fmul_rn(qx, vy), __fmul_rn(qy, vx));
  ux = __fadd_rn(ux, ux);
  uy = __fadd_rn(uy, uy);
  uz = __fadd_rn(uz, uz);
  const float cx = __fsub_rn(__fmul_rn(qy, uz), __fmul_rn(qz, uy));
  const float cy = __fsub_rn(__fmul_rn(qz, ux), __fmul_rn(qx, uz));
  ox = __fadd_rn(__fadd_rn(__fadd_rn(vx, __fmul_rn(w, ux)), cx), 0.f);
  oy = __fadd_rn(__fadd_rn(__fadd_rn(vy, __fmul_rn(w, uy)), cy), 0.f);
}

// kForm: 0 = ProbabilityGrid staged in shared memory by TMA, 1 = ProbabilityGrid through
// read-only global gathers, 2 = TSDF2D (two global cell arrays).
template <int kForm, int kRtAcc>
__global__ void __launch_bounds__(kRtThreads, 2)
k_rt_match(const __grid_constant__ CUtensorMap tmap, const RtGridDev G, const RtParams P,
           const RtJobDev* __restrict__ jobs, int num_jobs, int total_items,
           const float* __restrict__ xyz, const float2* __restrict__ trig,
           const double* __restrict__ weights, unsigned long long* __restrict__ best) {
  extern __shared__ __align__(128) unsigned char s_raw[];
  uint16_t* s_tile = reinterpret_cast<uint16_t*>(s_raw);
  __shared__ __align__(8) uint64_t s_bar;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // contiguous item range of this CTA (items are (job, scan) pairs in job order)
  const long long per_cta = (static_cast<long long>(total_items) + gridDim.x - 1) / gridDim.x;
  const int it_lo = static_cast<int>(min(static_cast<long long>(total_items), per_cta * blockIdx.x));
  const int it_hi = static_cast<int>(min(static_cast<long long>(total_items), per_cta * (blockIdx.x + 1)));
  if (it_lo >= it_hi) return;
  // job of the first item (binary search over item_base)
  int j = 0;
  {
    int lo = 0, hi = num_jobs - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (jobs[mid].item_base <= it_lo) lo = mid; else hi = mid - 1;
    }
    j = lo;
  }
  unsigned phase = 0;
  int tile_x0 = INT_MIN, tile_y0 = INT_MIN;
  if (kForm == 0) {
    if (threadIdx.x == 0) {
      MbarInit(&s_bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
  }
  int it = it_lo;
  while (it < it_hi) {
    const RtJobDev jb = jobs[j];
    const int job_end = min(it_hi, jb.item_base + jb.num_scans);
    if (kForm == 0 && (jb.x0 != tile_x0 || jb.y0 != tile_y0)) {
      // (re)stage the box this job reads; all warps are done with the previous one
      __syncthreads();
      if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        MbarExpectTx(&s_bar, static_cast<unsigned>(G.bw) * G.bh * 2u);
        TmaLoad2D(s_tile, &tmap, jb.x0, jb.y0, &s_bar);
      }
      MbarWait(&s_bar, phase);
      phase ^= 1u;
      tile_x0 = jb.x0;
      tile_y0 = jb.y0;
    }
    const float* __restrict__ pts = xyz + jb.xyz_off;
    const float n_f = __int2float_rn(jb.n);
    for (int item = it + warp; item < job_end; item += kRtWarps) {
      const int k = item - jb.item_base;       // rotated scan of the job
      const float2 cs = trig[jb.trig_off + k];
      const int ak = abs(k - jb.num_angular);
      for (int r0 = 0; r0 < P.per_scan; r0 += 32 * kRtAcc) {
        int xo[kRtAcc], yo[kRtAcc];
        float sum[kRtAcc], wsum[kRtAcc];
#pragma unroll
        for (int a = 0; a < kRtAcc; ++a) {
          const int r = r0 + lane + 32 * a;    // generation order: x outer, y inner (:98-111)
          xo[a] = -P.lin + r / P.width;
          yo[a] = -P.lin + r % P.width;
          sum[a] = 0.f;
          wsum[a] = 0.f;
        }
        const int acc_n = min(kRtAcc, (P.per_scan - r0 + 31) >> 5);  // warp-uniform
        for (int p0 = 0; p0 < jb.n; p0 += 32) {
          int cell = 0;
          if (p0 + lane < jb.n) {
            const float vx = pts[3 * (p0 + lane)], vy = pts[3 * (p0 + lane) + 1],
                        vz = pts[3 * (p0 + lane) + 2];
            float rx, ry;
            RotateZ(cs.x, cs.y, vx, vy, vz, rx, ry);   // GenerateRotatedScans (corr...2d.cc:93-109)
            // Affine2f(Translation2f) * v                                    (corr...2d.cc:120-121)
            const float px = __fadd_rn(__fadd_rn(__fmul_rn(1.f, rx), __fmul_rn(0.f, ry)), jb.tx);
            const float py = __fadd_rn(__fadd_rn(__fmul_rn(0.f, rx), __fmul_rn(1.f, ry)), jb.ty);
            // MapLimits::GetCellIndex in double                              (2d/map_limits.h:69-76)
            const double fx = __dsub_rn(__ddiv_rn(__dsub_rn(G.max_y, static_cast<double>(py)),
                                                  G.resolution), 0.5);
            const double fy = __dsub_rn(__ddiv_rn(__dsub_rn(G.max_x, static_cast<double>(px)),
                                                  G.resolution), 0.5);
            const long long ix = llround(fx), iy = llround(fy);
            // far-away points read "outside" for every candidate either way
            const int cx = static_cast<int>(max(-30000LL, min(30000LL, ix)));
            const int cy = static_cast<int>(max(-30000LL, min(30000LL, iy)));
            cell = (cy << 16) | (cx & 0xffff);
          }
          const int cnt = min(32, jb.n - p0);
#pragma unroll 8
          for (int t = 0; t < cnt; ++t) {
            const int c = __shfl_sync(0xffffffffu, cell, t);
            const int cx = static_cast<short>(c & 0xffff), cy = c >> 16;
#pragma unroll
            for (int a = 0; a < kRtAcc; ++a) {
              if (a >= acc_n) continue;   // warp-uniform
              // branch-free: an out-of-range candidate reads cell 0 of the staged box /
              // the grid and discards it
              const int x = cx + xo[a], y = cy + yo[a];
              const bool in = static_cast<unsigned>(x) < static_cast<unsigned>(G.nx) &&
                              static_cast<unsigned>(y) < static_cast<unsigned>(G.ny);
              if (kForm == 2) {
                // TSDF (real_time...2d.cc:38-59): outside the limits tsd = min, weight = 0
                const size_t flat = in ? static_cast<size_t>(y) * G.pitch + x : 0;
                const int tv = __ldg(G.cells + flat) & 0x7fff, wv = __ldg(G.wcells + flat) & 0x7fff;
                const float tsd_in =
                    tv == 0 ? P.min_tsd
                            : __fadd_rn(__fmul_rn(__int2float_rn(tv), P.tsd_scale), P.tsd_bias);
                const float w_in =
                    wv == 0 ? 0.f : __fadd_rn(__fmul_rn(__int2float_rn(wv), P.w_scale), P.w_bias);
                const float tsd = in ? tsd_in : P.min_tsd, w = in ? w_in : 0.f;
                const float normalized = __fdiv_rn(__fsub_rn(P.truncation, fabsf(tsd)), P.truncation);
                sum[a] = __fadd_rn(sum[a], __fmul_rn(normalized, w));
                wsum[a] = __fadd_rn(wsum[a], w);
              } else {
                // ProbabilityGrid::GetProbability (2d/probability_grid.cc:78-82)
                int value;
                if (kForm == 0) {
                  const int idx = in ? (y - tile_y0) * G.bw + (x - tile_x0) : 0;
                  value = s_tile[idx] & 0x7fff;
                } else {
                  const size_t flat = in ? static_cast<size_t>(y) * G.pitch + x : 0;
                  value = __ldg(G.cells + flat) & 0x7fff;
                }
                const float cost = value == 0 ? P.max_cost
                                              : __fadd_rn(__fmul_rn(__int2float_rn(value), P.k_scale),
                                                          P.cost_bias);
                const float prob = in ? __fsub_rn(1.f, cost) : P.min_probability;
                sum[a] = __fadd_rn(sum[a], prob);
              }
            }
          }
        }
        // score, weight, first-maximum key
        unsigned long long key = 0ull;
#pragma unroll
        for (int a = 0; a < kRtAcc; ++a) {
          const int r = r0 + lane + 32 * a;
          if (r >= P.per_scan) continue;
          float score;
          if (kForm == 2) score = wsum[a] == 0.f ? 0.f : __fdiv_rn(sum[a], wsum[a]);
          else score = __fdiv_rn(sum[a], n_f);
          const int i = min(abs(xo[a]), abs(yo[a])), jj = max(abs(xo[a]), abs(yo[a]));
          const double w = weights[jb.w_off + ak * P.npair + (jj * (jj + 1) / 2 + i)];
          // candidate.score *= exp(...): float *= double                 (:170-174)
          score = __double2float_rn(__dmul_rn(static_cast<double>(score), w));
          const unsigned c_index = static_cast<unsigned>(k * P.per_scan + r);
          // scores are >= 0, so their bit patterns order like the floats; ties go to the
          // smaller generation index (std::max_element returns the first maximum)
          const unsigned long long kk =
              (static_cast<unsigned long long>(__float_as_uint(fmaxf(score, 0.f))) << 32) |
              (0xffffffffu - c_index);
          key = max(key, kk);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
        if (lane == 0) atomicMax(&best[j], key);
      }
    }
    it = job_end;
    if (it >= jb.item_base + jb.num_scans) ++j;
  }
}

// Public ScoreCandidates (real_time_correlative_scan_matcher_2d.h:75, .cc:151-176) for
// caller-supplied discrete scans and candidates: one thread per candidate, ordered sum.
__global__ void __launch_bounds__(128)
k_rt_score_list(const RtGridDev G, const RtParams P, const int2* __restrict__ dscan, int n,
                const int4* __restrict__ cands /* scan, xo, yo, _ */,
                const double* __restrict__ weight, int count, float* __restrict__ scores) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= count) return;
  const int4 cd = cands[c];
  const int2* __restrict__ pts = dscan + static_cast<size_t>(cd.x) * n;
  float sum = 0.f;
  for (int p = 0; p < n; ++p) {
    const int2 q = pts[p];
    const int x = q.x + cd.y, y = q.y + cd.z;
    float prob = P.min_probability;
    if (static_cast<unsigned>(x) < static_cast<unsigned>(G.nx) &&
        static_cast<unsigned>(y) < static_cast<unsigned>(G.ny)) {
      const int value = __ldg(G.cells + static_cast<size_t>(y) * G.pitch + x) & 0x7fff;
      const float cost = value == 0 ? P.max_cost
                                    : __fadd_rn(__fmul_rn(__int2float_rn(value), P.k_scale), P.cost_bias);
      prob = __fsub_rn(1.f, cost);
    }
    sum = __fadd_rn(sum, prob);
  }
  const float score = __fdiv_rn(sum, __int2float_rn(n));
  scores[c] = __double2float_rn(__dmul_rn(static_cast<double>(score), weight[c]));
}

}  // namespace csm

using namespace csm;

// A ProbabilityGrid (or TSDF2D) resident on the device, with the TMA descriptor of its
// cell array.  LocalTrajectoryBuilder2D matches every scan against the active submap's
// grid (local_trajectory_builder_2d.cc:77-82); the handle lets many scans share one copy.
namespace {

struct HV3 { float x, y, z; };
inline HV3 HCross(const HV3& a, const HV3& b) {
  return HV3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
// Same Eigen formula as the device RotateRn (transform/rigid_transform.h:192-196).
inline HV3 HRotate(float qw, const HV3& qv, const HV3& v) {
  HV3 uv = HCross(qv, v);
  uv.x += uv.x; uv.y += uv.y; uv.z += uv.z;
  const HV3 c = HCross(qv, uv);
  HV3 r{(v.x + qw * uv.x) + c.x, (v.y + qw * uv.y) + c.y, (v.z + qw * uv.z) + c.z};
  r.x += 0.f; r.y += 0.f; r.z += 0.f;
  return r;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn GetEncodeTiled() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

void FillParams(RtParams* P, int lin, float truncation, float max_weight) {
  std::memset(P, 0, sizeof(*P));
  P->lin = lin;
  P->width = 2 * lin + 1;
  P->per_scan = P->width * P->width;
  P->npair = (lin + 1) * (lin + 2) / 2;
  // probability_values.h:64-67 and .cc:29-37 evaluated in float
  const float kMinProbability = 0.1f;
  const float kMaxProbability = 1.f - kMinProbability;
  const float kMinCost = 1.f - kMaxProbability;
  const float kMaxCost = 1.f - kMinProbability;
  P->k_scale = (kMaxCost - kMinCost) / 32766.f;
  P->cost_bias = kMinCost - P->k_scale;
  P->max_cost = kMaxCost;
  P->min_probability = kMinProbability;
  if (truncation > 0.f) {
    const TsdfConversion c = MakeTsdfConversion(truncation, max_weight);
    P->tsd_scale = c.tsd_scale;
    P->tsd_bias = c.tsd_bias;
    P->min_tsd = c.min_tsd;
    P->w_scale = c.w_scale;
    P->w_bias = c.w_bias;
    P->truncation = truncation;
  }
}

// Uploads `cells` (host pitch nx) into the handle's padded device array.
csm_status UploadCells(csm_rt_grid2d* g, const uint16_t* cells, const uint16_t* wcells,
                       cudaStream_t s) {
  CSM_CUDA(cudaMemcpy2DAsync(g->d_cells, static_cast<size_t>(g->g.pitch) * 2, cells,
                             static_cast<size_t>(g->g.nx) * 2, static_cast<size_t>(g->g.nx) * 2,
                             g->g.ny, cudaMemcpyHostToDevice, s));
  if (wcells)
    CSM_CUDA(cudaMemcpy2DAsync(g->d_wcells, static_cast<size_t>(g->g.pitch) * 2, wcells,
                               static_cast<size_t>(g->g.nx) * 2, static_cast<size_t>(g->g.nx) * 2,
                               g->g.ny, cudaMemcpyHostToDevice, s));
  return CSM_OK;
}

csm_status GridCreate(const uint16_t* cells, const uint16_t* wcells, float truncation,
                      float max_weight, int32_t nx, int32_t ny, double resolution, double max_x,
                      double max_y, int32_t device, csm_rt_grid2d** out) {
  CSM_REQUIRE(out != nullptr && cells != nullptr, "null pointer");
  CSM_REQUIRE(nx >= 1 && ny >= 1 && resolution > 0., "sizes");
  CSM_REQUIRE(nx < 30000 && ny < 30000, "grid too large");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_rt_grid2d> g(new csm_rt_grid2d);
  g->ctx = ctx;
  g->truncation = truncation;
  g->max_weight = max_weight;
  RtGridDev& d = g->g;
  d.nx = nx;
  d.ny = ny;
  d.pitch = (nx + 7) / 8 * 8;  // rows are multiples of 16 bytes (TMA global strides)
  d.resolution = resolution;
  d.max_x = max_x;
  d.max_y = max_y;
  const size_t bytes = static_cast<size_t>(d.pitch) * ny * 2;
  CSM_CUDA(cudaMalloc(&g->d_cells, bytes));
  CSM_CUDA(cudaMemsetAsync(g->d_cells, 0, bytes, ctx->stream));
  if (wcells) {
    CSM_CUDA(cudaMalloc(&g->d_wcells, bytes));
    CSM_CUDA(cudaMemsetAsync(g->d_wcells, 0, bytes, ctx->stream));
  }
  d.cells = g->d_cells;
  d.wcells = g->d_wcells;
  CSM_TRY(UploadCells(g.get(), cells, wcells, ctx->stream));
  CSM_TRY(RtGridEncodeTmap(g.get()));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = g.release();
  return CSM_OK;
}

struct RtHostJob {
  const float* xyz;
  int n;
  double init[3];
};

struct RtPlan {          // per job, host side
  int num_angular = 0, num_scans = 0;
  double step = 0.;
  bool smem = false;
};

// Host preparation of one job into the staging buffers: rotated cloud, SearchParameters,
// rotation table, weight classes (all libm, like the reference).
void PrepareJob(const RtHostJob& job, const RtGridDev& G, const RtParams& P, double angular_window,
                double w_t, double w_r, float* xyz_out, float* trig_out, double* w_out,
                RtPlan* plan, RtJobDev* jd) {
  // rotated_point_cloud (:123-127): SearchParameters needs its max range.
  const float yaw = static_cast<float>(job.init[2]);
  const float ha0 = 0.5f * yaw;
  const float s0 = std::sin(ha0);
  const HV3 q0{s0 * 0.f, s0 * 0.f, s0 * 1.f};
  const float q0w = std::cos(ha0);
  float max_scan_range = 3.f * G.resolution;  // correlative_scan_matcher_2d.cc:34
  for (int i = 0; i < job.n; ++i) {
    const HV3 r = HRotate(q0w, q0, HV3{job.xyz[3 * i], job.xyz[3 * i + 1], job.xyz[3 * i + 2]});
    xyz_out[3 * i] = r.x;
    xyz_out[3 * i + 1] = r.y;
    xyz_out[3 * i + 2] = r.z;
    const float range = std::sqrt(r.x * r.x + r.y * r.y);
    max_scan_range = std::max(range, max_scan_range);
  }
  const double kSafetyMargin = 1. - 1e-3;
  const double step = kSafetyMargin * std::acos(1. - (G.resolution * G.resolution) /
                                                         (2. * (max_scan_range * max_scan_range)));
  const int num_angular = plan->num_angular;  // computed by the caller (needed for sizes)
  plan->step = step;
  double delta_theta = -num_angular * step;
  for (int k = 0; k < plan->num_scans; ++k, delta_theta += step) {
    const float ha = 0.5f * static_cast<float>(delta_theta);
    trig_out[2 * k] = std::cos(ha);
    trig_out[2 * k + 1] = std::sin(ha);
  }
  // weight classes: |orientation| = a * step (Candidate2D ctor), hypot over {|xo|, |yo|}
  for (int a = 0; a <= num_angular; ++a) {
    const double orientation = a * step;
    for (int jj = 0; jj <= P.lin; ++jj)
      for (int i = 0; i <= jj; ++i) {
        const double cx = -(jj)*G.resolution, cy = -(i)*G.resolution;
        const double e = std::hypot(cx, cy) * w_t + std::abs(orientation) * w_r;
        w_out[a * P.npair + jj * (jj + 1) / 2 + i] = std::exp(-(e * e));
      }
  }
  jd->n = job.n;
  jd->num_scans = plan->num_scans;
  jd->num_angular = num_angular;
  jd->tx = static_cast<float>(job.init[0]);  // Translation2f(double, double) (:135-137)
  jd->ty = static_cast<float>(job.init[1]);
  // Box the scan can reach: cell of the initial translation +- (max range + window)
  const double fx = (G.max_y - jd->ty) / G.resolution - 0.5, fy = (G.max_x - jd->tx) / G.resolution - 0.5;
  const double R = std::ceil(max_scan_range / G.resolution) + P.lin + 3;
  const long long rx0 = std::max<long long>(0, static_cast<long long>(std::floor(fx - R)));
  const long long rx1 = std::min<long long>(G.nx - 1, static_cast<long long>(std::ceil(fx + R)));
  const long long ry0 = std::max<long long>(0, static_cast<long long>(std::floor(fy - R)));
  const long long ry1 = std::min<long long>(G.ny - 1, static_cast<long long>(std::ceil(fy + R)));
  plan->smem = false;
  jd->x0 = jd->y0 = 0;
  if (rx1 < rx0 || ry1 < ry0) {       // the scan cannot reach the grid: any box will do
    plan->smem = true;
  } else {
    // the box starts on a 16-byte boundary of its row (8 cells): TMA global addresses
    const long long ax0 = rx0 & ~7LL;
    if (rx1 - ax0 + 1 <= G.bw && ry1 - ry0 + 1 <= G.bh) {
      plan->smem = true;
      jd->x0 = static_cast<int>(ax0);
      jd->y0 = static_cast<int>(ry0);
    }
  }
}

int NumAngular(const RtHostJob& job, double resolution, double angular_window) {
  // needs the max range of the rotated cloud: identical arithmetic to PrepareJob
  const float yaw = static_cast<float>(job.init[2]);
  const float ha0 = 0.5f * yaw;
  const float s0 = std::sin(ha0);
  const HV3 q0{s0 * 0.f, s0 * 0.f, s0 * 1.f};
  const float q0w = std::cos(ha0);
  float max_scan_range = 3.f * resolution;
  for (int i = 0; i < job.n; ++i) {
    const HV3 r = HRotate(q0w, q0, HV3{job.xyz[3 * i], job.xyz[3 * i + 1], job.xyz[3 * i + 2]});
    const float range = std::sqrt(r.x * r.x + r.y * r.y);
    max_scan_range = std::max(range, max_scan_range);
  }
  const double kSafetyMargin = 1. - 1e-3;
  const double step = kSafetyMargin * std::acos(1. - (resolution * resolution) /
                                                         (2. * (max_scan_range * max_scan_range)));
  return static_cast<int>(std::ceil(angular_window / step));
}

template <typename F>
void ParallelFor(int n, int max_threads, F f) {
  const int hw = static_cast<int>(std::thread::hardware_concurrency());
  const int t = std::max(1, std::min(std::min(max_threads, hw > 0 ? hw : 1), n / 8));
  if (t <= 1) {
    for (int i = 0; i < n; ++i) f(i);
    return;
  }
  std::vector<std::thread> th;
  std::atomic<int> next{0};
  for (int w = 0; w < t; ++w)
    th.emplace_back([&]() {
      for (;;) {
        const int i0 = next.fetch_add(8);
        if (i0 >= n) break;
        for (int i = i0; i < std::min(n, i0 + 8); ++i) f(i);
      }
    });
  for (auto& x : th) x.join();
}

// Runs jobs[0..num) against the grid on `ctx` (a lane).
csm_status RtRun(Ctx* ctx, const csm_rt_grid2d* grid, const RtHostJob* jobs, int num,
                 double linear_window, double angular_window, double w_t, double w_r,
                 csm_rt_result2d* results, csm_stats* stats) {
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const RtGridDev& G = grid->g;
  const int lin = static_cast<int>(std::ceil(linear_window / G.resolution));
  CSM_REQUIRE(lin >= 0 && lin < 2048, "linear search window");
  RtParams P;
  FillParams(&P, lin, grid->truncation, grid->max_weight);
  // sizes first (the staging layout needs them), then the parallel fill
  std::vector<RtPlan> plan(num);
  std::vector<RtJobDev> jd(num);
  std::vector<int> bad(1, 0);
  ParallelFor(num, 16, [&](int j) {
    plan[j].num_angular = NumAngular(jobs[j], G.resolution, angular_window);
    plan[j].num_scans = 2 * plan[j].num_angular + 1;
  });
  long long xyz_f = 0, trig_f = 0, w_d = 0, items = 0, cands = 0;
  for (int j = 0; j < num; ++j) {
    CSM_REQUIRE(plan[j].num_scans > 0 && plan[j].num_scans < (1 << 20), "angular window / step");
    jd[j].xyz_off = xyz_f;
    jd[j].trig_off = static_cast<int>(trig_f);
    jd[j].w_off = static_cast<int>(w_d);
    jd[j].item_base = static_cast<int>(items);
    xyz_f += 3LL * jobs[j].n;
    trig_f += plan[j].num_scans;
    w_d += static_cast<long long>(plan[j].num_angular + 1) * P.npair;
    items += plan[j].num_scans;
    cands += static_cast<long long>(plan[j].num_scans) * P.per_scan;
    CSM_REQUIRE(static_cast<long long>(plan[j].num_scans) * P.per_scan < (1LL << 31),
                "search window too large");
  }
  CSM_REQUIRE(items < (1LL << 30) && trig_f < (1LL << 30) && w_d < (1LL << 30), "batch too large");
  const size_t off_trig = (static_cast<size_t>(xyz_f) * 4 + 255) / 256 * 256;
  const size_t off_w = (off_trig + static_cast<size_t>(trig_f) * 8 + 255) / 256 * 256;
  const size_t off_jobs = (off_w + static_cast<size_t>(w_d) * 8 + 255) / 256 * 256;
  const size_t up_bytes = off_jobs + sizeof(RtJobDev) * num;
  PinnedBuf& up = ctx->P("rt_upload");
  DevBuf& d_up = ctx->D("rt_upload");
  DevBuf& d_best = ctx->D("rt_best");
  PinnedBuf& rb = ctx->P("rt_readback");
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(d_up.Reserve(up_bytes));
  CSM_TRY(d_best.Reserve(sizeof(unsigned long long) * num));
  CSM_TRY(rb.Reserve(sizeof(unsigned long long) * num));
  char* h = up.as<char>();
  ParallelFor(num, 16, [&](int j) {
    PrepareJob(jobs[j], G, P, angular_window, w_t, w_r, reinterpret_cast<float*>(h) + jd[j].xyz_off,
               reinterpret_cast<float*>(h + off_trig) + 2 * static_cast<size_t>(jd[j].trig_off),
               reinterpret_cast<double*>(h + off_w) + jd[j].w_off, &plan[j], &jd[j]);
  });
  bool all_smem = grid->has_tmap;
  for (int j = 0; j < num; ++j) all_smem = all_smem && plan[j].smem;
  std::memcpy(h + off_jobs, jd.data(), sizeof(RtJobDev) * num);

  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_CUDA(cudaMemcpyAsync(d_up.p, h, up_bytes, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemsetAsync(d_best.p, 0, sizeof(unsigned long long) * num, s));
  const char* d = d_up.as<char>();
  const int total_items = static_cast<int>(items);
  const int form = grid->d_wcells ? 2 : (all_smem ? 0 : 1);
  const size_t smem = form == 0 ? static_cast<size_t>(G.bw) * G.bh * 2 : 0;
  int per_sm = 1;
#define CSM_RT_LAUNCH(F, A)                                                                     \
  do {                                                                                          \
    if (smem > 48 * 1024)                                                                       \
      CSM_CUDA(cudaFuncSetAttribute(k_rt_match<F, A>,                                           \
                                    cudaFuncAttributeMaxDynamicSharedMemorySize,                \
                                    static_cast<int>(smem)));                                   \
    CSM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rt_match<F, A>,           \
                                                           kRtThreads, smem));                  \
    const int grid_dim = std::max(1, std::min((total_items + kRtWarps - 1) / kRtWarps,          \
                                              ctx->sm_count * std::max(1, per_sm)));            \
    k_rt_match<F, A><<<grid_dim, kRtThreads, smem, s>>>(                                        \
        grid->tmap, G, P, reinterpret_cast<const RtJobDev*>(d + off_jobs), num, total_items,    \
        reinterpret_cast<const float*>(d), reinterpret_cast<const float2*>(d + off_trig),       \
        reinterpret_cast<const double*>(d + off_w), d_best.as<unsigned long long>());           \
  } while (0)
  ProfBegin(ctx);
  const bool one_acc = P.per_scan <= 32;
  if (form == 0) { if (one_acc) CSM_RT_LAUNCH(0, 1); else CSM_RT_LAUNCH(0, 4); }
  else if (form == 1) { if (one_acc) CSM_RT_LAUNCH(1, 1); else CSM_RT_LAUNCH(1, 4); }
  else { if (one_acc) CSM_RT_LAUNCH(2, 1); else CSM_RT_LAUNCH(2, 4); }
#undef CSM_RT_LAUNCH
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, form == 0 ? "k_rt_match_tma" : (form == 1 ? "k_rt_match_gather" : "k_rt_match_tsdf"),
          static_cast<double>(cands));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(rb.p, d_best.p, sizeof(unsigned long long) * num,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  const unsigned long long* keys = rb.as<unsigned long long>();
  for (int j = 0; j < num; ++j) {
    const unsigned bits = static_cast<unsigned>(keys[j] >> 32);
    const unsigned best = 0xffffffffu - static_cast<unsigned>(keys[j] & 0xffffffffu);
    float best_score;
    std::memcpy(&best_score, &bits, 4);
    const int scan = static_cast<int>(best / P.per_scan);
    const int r = static_cast<int>(best % P.per_scan);
    const int xo = -lin + r / P.width, yo = -lin + r % P.width;
    csm_rt_result2d& o = results[j];
    o.score = best_score;
    o.pose_estimate[0] = jobs[j].init[0] + (-yo * G.resolution);
    o.pose_estimate[1] = jobs[j].init[1] + (-xo * G.resolution);
    o.pose_estimate[2] = jobs[j].init[2] + (scan - plan[j].num_angular) * plan[j].step;
    o.best_scan_index = scan;
    o.best_x_offset = xo;
    o.best_y_offset = yo;
    o.num_scans = plan[j].num_scans;
    o.candidates_scored = static_cast<int64_t>(plan[j].num_scans) * P.per_scan;
  }
  if (stats) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    stats->candidates_scored += cands;
    stats->lowest_resolution_candidates += cands;
    stats->device_ms += ms;
    stats->host_syncs += 1;
    if (num == 1) {
      stats->num_scans = results[0].num_scans;
      stats->best_scan_index = results[0].best_scan_index;
      stats->best_x_offset = results[0].best_x_offset;
      stats->best_y_offset = results[0].best_y_offset;
      stats->leaves_tied = 1;
    }
  }
  return CSM_OK;
}

// Single-call form: the grid is passed per call (the reference signature).  Every lane
// keeps one device copy (+ TMA descriptor) that is re-used while the dimensions stay the
// same — the active submap's grid keeps its limits between most scans — so a call costs
// one H2D of the cells, not a cudaMalloc / cudaFree pair.
std::mutex g_rt_cache_mu;
std::map<Ctx*, std::unique_ptr<csm_rt_grid2d>> g_rt_cache;

csm_status RtMatchHostGrid(const uint16_t* cells, const uint16_t* weight_cells, float truncation,
                           float max_weight, int32_t nx, int32_t ny, double resolution,
                           double max_x, double max_y, const float* xyz, int32_t n,
                           const double initial_pose[3], double linear_window,
                           double angular_window, double w_t, double w_r, int32_t device,
                           double* score, double pose_estimate[3], csm_stats* stats) {
  CSM_REQUIRE(cells && xyz && initial_pose && score && pose_estimate, "null pointer");  // :121
  CSM_REQUIRE(nx >= 1 && ny >= 1 && n >= 1 && resolution > 0., "sizes");
  LaneGuard guard;
  CSM_TRY(AcquireLane(device, &guard));
  Ctx* lane = guard.lane;
  csm_rt_grid2d* grid = nullptr;
  {
    std::lock_guard<std::mutex> lock(g_rt_cache_mu);
    std::unique_ptr<csm_rt_grid2d>& slot = g_rt_cache[lane];
    const bool reuse = slot && slot->g.nx == nx && slot->g.ny == ny &&
                       (slot->d_wcells != nullptr) == (weight_cells != nullptr);
    if (reuse) {
      slot->g.resolution = resolution;
      slot->g.max_x = max_x;
      slot->g.max_y = max_y;
      slot->truncation = truncation;
      slot->max_weight = max_weight;
      CSM_CUDA(cudaSetDevice(device));
      CSM_TRY(UploadCells(slot.get(), cells, weight_cells, lane->stream));
    } else {
      if (slot) {
        std::lock_guard<std::mutex> dl(slot->ctx->mu);
        cudaSetDevice(device);
        cudaStreamSynchronize(lane->stream);
        slot.reset();
      }
      csm_rt_grid2d* fresh = nullptr;
      CSM_TRY(GridCreate(cells, weight_cells, truncation, max_weight, nx, ny, resolution, max_x,
                         max_y, device, &fresh));
      slot.reset(fresh);
    }
    grid = slot.get();  // only this lane (locked by `guard`) ever uses its slot
  }
  RtHostJob job{xyz, n, {initial_pose[0], initial_pose[1], initial_pose[2]}};
  csm_rt_result2d r;
  std::memset(&r, 0, sizeof(r));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  CSM_TRY(RtRun(lane, grid, &job, 1, linear_window, angular_window, w_t, w_r, &r, stats));
  *score = r.score;
  std::memcpy(pose_estimate, r.pose_estimate, sizeof(double) * 3);
  return CSM_OK;
}

}  // namespace

namespace csm {

csm_status RtGridEncodeTmap(csm_rt_grid2d* g) {
  RtGridDev& d = g->g;
  // TMA box: as wide as the (padded) grid up to 256 cells, as many rows as fit the tile
  d.bw = std::min(d.pitch, 256);
  d.bh = std::max(1, std::min(std::min(d.ny, 256), kRtTileBytes / (d.bw * 2)));
  g->has_tmap = false;
  if (g->d_wcells) {
    std::memset(&g->tmap, 0, sizeof(g->tmap));
    return CSM_OK;
  }
  EncodeTiledFn encode = GetEncodeTiled();
  if (encode) {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.nx), static_cast<cuuint64_t>(d.ny)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.pitch) * 2};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(d.bw), static_cast<cuuint32_t>(d.bh)};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode(&g->tmap, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, g->d_cells, dims,
                              strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    g->has_tmap = r == CUDA_SUCCESS;
  }
  if (!g->has_tmap) {
    SetError("cuTensorMapEncodeTiled is unavailable or failed");
    return CSM_E_CUDA;
  }
  return CSM_OK;
}

}  // namespace csm

extern "C" {

csm_status csm_rt_grid2d_create(const uint16_t* cells, int32_t nx, int32_t ny, double resolution,
                                double max_x, double max_y, int32_t device, csm_rt_grid2d** out) {
  return GridCreate(cells, nullptr, 0.f, 0.f, nx, ny, resolution, max_x, max_y, device, out);
}

csm_status csm_rt_grid2d_update(csm_rt_grid2d* grid, const uint16_t* cells) {
  CSM_REQUIRE(grid && cells, "null pointer");
  // the weight cells would go stale
  CSM_REQUIRE(grid->d_wcells == nullptr, "a TSDF2D handle is updated by csm_rt_grid2d_update_tsdf");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  CSM_TRY(UploadCells(grid, cells, nullptr, grid->ctx->stream));
  grid->known_stale = true;
  CSM_CUDA(cudaStreamSynchronize(grid->ctx->stream));
  return CSM_OK;
}

csm_status csm_rt_grid2d_create_tsdf(const uint16_t* tsd_cells, const uint16_t* weight_cells,
                                     int32_t nx, int32_t ny, double resolution, double max_x,
                                     double max_y, float truncation_distance, float max_weight,
                                     int32_t device, csm_rt_grid2d** out) {
  CSM_REQUIRE(weight_cells != nullptr, "null weight cells");
  CSM_REQUIRE(truncation_distance > 0.f && max_weight > 0.f, "TSDF parameters");
  return GridCreate(tsd_cells, weight_cells, truncation_distance, max_weight, nx, ny, resolution,
                    max_x, max_y, device, out);
}

csm_status csm_rt_grid2d_update_tsdf(csm_rt_grid2d* grid, const uint16_t* tsd_cells,
                                     const uint16_t* weight_cells) {
  CSM_REQUIRE(grid && tsd_cells && weight_cells, "null pointer");
  CSM_REQUIRE(grid->d_wcells != nullptr, "the grid is not a TSDF2D");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  CSM_TRY(UploadCells(grid, tsd_cells, weight_cells, grid->ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(grid->ctx->stream));
  return CSM_OK;
}

csm_status csm_rt_grid2d_destroy(csm_rt_grid2d* grid) {
  if (!grid) return CSM_OK;
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  cudaSetDevice(grid->ctx->device);
  cudaStreamSynchronize(grid->ctx->stream);
  delete grid;
  return CSM_OK;
}

csm_status csm_rt_match2d_batch(const csm_rt_grid2d* grid, const csm_rt_job2d* jobs,
                                int32_t num_jobs, double linear_window, double angular_window,
                                double w_t, double w_r, csm_rt_result2d* results,
                                csm_stats* stats) {
  CSM_REQUIRE(grid && jobs && results, "null pointer");
  CSM_REQUIRE(num_jobs >= 1, "empty batch");
  for (int j = 0; j < num_jobs; ++j)
    CSM_REQUIRE(jobs[j].xyz != nullptr && jobs[j].num_points >= 1, "empty point cloud");
  LaneGuard guard;
  CSM_TRY(AcquireLane(grid->ctx->device, &guard));
  if (stats) std::memset(stats, 0, sizeof(*stats));
  const int kMaxJobs = 4096;  // per launch: bounds the staging buffers
  std::vector<RtHostJob> hj;
  for (int j0 = 0; j0 < num_jobs; j0 += kMaxJobs) {
    const int cnt = std::min(kMaxJobs, num_jobs - j0);
    hj.resize(cnt);
    for (int j = 0; j < cnt; ++j)
      hj[j] = RtHostJob{jobs[j0 + j].xyz, jobs[j0 + j].num_points,
                        {jobs[j0 + j].initial_pose[0], jobs[j0 + j].initial_pose[1],
                         jobs[j0 + j].initial_pose[2]}};
    CSM_TRY(RtRun(guard.lane, grid, hj.data(), cnt, linear_window, angular_window, w_t, w_r,
                  results + j0, stats));
  }
  return CSM_OK;
}

csm_status csm_rt_match2d(const uint16_t* cells, int32_t nx, int32_t ny, double resolution,
                          double max_x, double max_y, const float* xyz, int32_t n,
                          const double initial_pose[3], double linear_window,
                          double angular_window, double w_t, double w_r, int32_t device,
                          double* score, double pose_estimate[3], csm_stats* stats) {
  return RtMatchHostGrid(cells, nullptr, 0.f, 0.f, nx, ny, resolution, max_x, max_y, xyz, n,
                         initial_pose, linear_window, angular_window, w_t, w_r, device, score,
                         pose_estimate, stats);
}

csm_status csm_rt_match2d_tsdf(const uint16_t* tsd_cells, const uint16_t* weight_cells,
                               int32_t nx, int32_t ny, double resolution, double max_x,
                               double max_y, float truncation_distance, float max_weight,
                               const float* xyz, int32_t n, const double initial_pose[3],
                               double linear_window, double angular_window, double w_t,
                               double w_r, int32_t device, double* score,
                               double pose_estimate[3], csm_stats* stats) {
  CSM_REQUIRE(weight_cells != nullptr, "null weight cells");
  CSM_REQUIRE(truncation_distance > 0.f && max_weight > 0.f, "TSDF parameters");
  return RtMatchHostGrid(tsd_cells, weight_cells, truncation_distance, max_weight, nx, ny,
                         resolution, max_x, max_y, xyz, n, initial_pose, linear_window,
                         angular_window, w_t, w_r, device, score, pose_estimate, stats);
}

csm_status csm_rt_score_candidates2d(const uint16_t* cells, int32_t nx, int32_t ny,
                                     double resolution, double max_x, double max_y,
                                     const int32_t* discrete_scans, int32_t num_scans, int32_t n,
                                     int32_t num_angular_perturbations,
                                     double angular_perturbation_step_size,
                                     const int32_t* candidates, int32_t num_candidates, double w_t,
                                     double w_r, int32_t device, float* scores) {
  CSM_REQUIRE(cells && discrete_scans && candidates && scores, "null pointer");
  CSM_REQUIRE(num_scans >= 1 && n >= 1 && num_candidates >= 0, "sizes");
  if (num_candidates == 0) return CSM_OK;
  csm_rt_grid2d* grid = nullptr;
  CSM_TRY(GridCreate(cells, nullptr, 0.f, 0.f, nx, ny, resolution, max_x, max_y, device, &grid));
  std::unique_ptr<csm_rt_grid2d> owner(grid);
  LaneGuard guard;
  CSM_TRY(AcquireLane(device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(device));
  cudaStream_t s = ctx->stream;
  RtParams P;
  FillParams(&P, 0, 0.f, 0.f);
  std::vector<int4> lc(num_candidates);
  std::vector<double> w(num_candidates);
  for (int c = 0; c < num_candidates; ++c) {
    const int scan = candidates[3 * c], xo = candidates[3 * c + 1], yo = candidates[3 * c + 2];
    CSM_REQUIRE(scan >= 0 && scan < num_scans, "scan_index");
    lc[c] = make_int4(scan, xo, yo, 0);
    // Candidate2D ctor (corr...2d.h:77-86) + the weight of :170-174
    const double cx = -yo * resolution, cy = -xo * resolution;
    const double orientation = (scan - num_angular_perturbations) * angular_perturbation_step_size;
    const double e = std::hypot(cx, cy) * w_t + std::abs(orientation) * w_r;
    w[c] = std::exp(-(e * e));
  }
  DevBuf& d_ds = ctx->D("rt_hook_dscan");
  DevBuf& d_lc = ctx->D("rt_hook_cands");
  DevBuf& d_w = ctx->D("rt_hook_w");
  DevBuf& d_sc = ctx->D("rt_hook_scores");
  const size_t npts = static_cast<size_t>(num_scans) * n;
  CSM_TRY(d_ds.Reserve(npts * 8));
  CSM_TRY(d_lc.Reserve(sizeof(int4) * num_candidates));
  CSM_TRY(d_w.Reserve(8 * static_cast<size_t>(num_candidates)));
  CSM_TRY(d_sc.Reserve(4 * static_cast<size_t>(num_candidates)));
  CSM_CUDA(cudaMemcpyAsync(d_ds.p, discrete_scans, npts * 8, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(d_lc.p, lc.data(), sizeof(int4) * num_candidates, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(d_w.p, w.data(), 8 * static_cast<size_t>(num_candidates),
                           cudaMemcpyHostToDevice, s));
  k_rt_score_list<<<(num_candidates + 127) / 128, 128, 0, s>>>(
      grid->g, P, d_ds.as<int2>(), n, d_lc.as<int4>(), d_w.as<double>(), num_candidates,
      d_sc.as<float>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(scores, d_sc.p, 4 * static_cast<size_t>(num_candidates),
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  {
    std::lock_guard<std::mutex> lock(grid->ctx->mu);
    owner.reset();
  }
  return CSM_OK;
}

}  // extern "C"
