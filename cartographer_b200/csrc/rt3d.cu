// RealTimeCorrelativeScanMatcher3D::Match on the device
// (cartographer/mapping/internal/3d/scan_matching/real_time_correlative_scan_matcher_3d.cc:34-117).
//
// The exhaustive window is (2L+1)^3 translations x (2A+1)^3 rotations; a candidate's score
// is an ORDERED float sum of one HybridGrid probability per point of the cloud transformed
// by candidate = initial_pose.cast<float>() * transform (:40-44, :104-108).  Work split:
//   * one CTA per ROTATION: the rotated cloud q_c * p is the same for every translation
//     of that rotation, so the CTA rotates 256 points at a time into shared memory once;
//   * one thread per TRANSLATION: adds its candidate translation, rounds to the voxel
//     (HybridGrid::GetCellIndex, hybrid_grid.h:428-433), gathers the probability from the
//     dense device copy of the grid and accumulates in point order;
//   * the candidate poses (quaternion products, AngleAxisVectorToRotationQuaternion) and
//     the exp() of the delta-cost weight (:109-114) are evaluated on the host with libm
//     in the reference's operation order, like every transcendental of the path;
//   * "if (score > best_score)" over the generation order (:45-48) = first maximum:
//     64-bit atomicMax of (score bits << 32 | ~generation index).
#include <algorithm>
#include <climits>
#include <cmath>
#include <map>

#include "common.cuh"
#include "grid3d.cuh"

namespace csm {

struct Rt3Params {
  int n;          // points
  int T, R;       // translations, rotations
};

__global__ void k_rt3_scatter(const int* __restrict__ idx, const uint16_t* __restrict__ values,
                              long long n, Grid3Dev g, uint16_t* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int x = idx[3 * i] - g.lo[0], y = idx[3 * i + 1] - g.lo[1], z = idx[3 * i + 2] - g.lo[2];
  out[(static_cast<size_t>(z) * g.n[1] + y) * g.n[0] + x] = values[i];
}

constexpr int kRt3Chunk = 256;

__global__ void __launch_bounds__(128)
k_rt3_match(const Grid3Dev G, const Rt3Params P, const float* __restrict__ xyz,
            const float4* __restrict__ rot /* candidate rotation per r: w, x, y, z */,
            const float4* __restrict__ trans /* candidate translation per t: x, y, z, weight class */,
            const double* __restrict__ weights /* [class][r] */,
            unsigned long long* __restrict__ best) {
  __shared__ float s_x[kRt3Chunk], s_y[kRt3Chunk], s_z[kRt3Chunk];
  __shared__ unsigned long long s_best;
  const int r = blockIdx.x;
  const float4 q = rot[r];
  if (threadIdx.x == 0) s_best = 0ull;
  __syncthreads();
  for (int t0 = 0; t0 < P.T; t0 += blockDim.x) {
    const int t = t0 + threadIdx.x;
    const bool on = t < P.T;
    const float4 tc = trans[on ? t : 0];
    float sum = 0.f;
    for (int p0 = 0; p0 < P.n; p0 += kRt3Chunk) {
      __syncthreads();
      // Rigid3f * point, rotation part: Eigen quaternion * vector
      // (transform/rigid_transform.h:192-196)
      for (int i = threadIdx.x; i < kRt3Chunk && p0 + i < P.n; i += blockDim.x) {
        const float vx = xyz[3 * (p0 + i)], vy = xyz[3 * (p0 + i) + 1], vz = xyz[3 * (p0 + i) + 2];
        float ux = __fsub_rn(__fmul_rn(q.z, vz), __fmul_rn(q.w, vy));  // qv = (q.y, q.z, q.w)
        float uy = __fsub_rn(__fmul_rn(q.w, vx), __fmul_rn(q.y, vz));
        float uz = __fsub_rn(__fmul_rn(q.y, vy), __fmul_rn(q.z, vx));
        ux = __fadd_rn(ux, ux);
        uy = __fadd_rn(uy, uy);
        uz = __fadd_rn(uz, uz);
        const float cx = __fsub_rn(__fmul_rn(q.z, uz), __fmul_rn(q.w, uy));
        const float cy = __fsub_rn(__fmul_rn(q.w, ux), __fmul_rn(q.y, uz));
        const float cz = __fsub_rn(__fmul_rn(q.y, uy), __fmul_rn(q.z, ux));
        s_x[i] = __fadd_rn(__fadd_rn(vx, __fmul_rn(q.x, ux)), cx);   // q.x holds w
        s_y[i] = __fadd_rn(__fadd_rn(vy, __fmul_rn(q.x, uy)), cy);
        s_z[i] = __fadd_rn(__fadd_rn(vz, __fmul_rn(q.x, uz)), cz);
      }
      __syncthreads();
      if (on) {
        const int cnt = min(kRt3Chunk, P.n - p0);
#pragma unroll 4
        for (int i = 0; i < cnt; ++i) {
          // + translation, HybridGrid::GetCellIndex = lround(p / resolution) per axis
          const int x = static_cast<int>(lroundf(__fdiv_rn(__fadd_rn(s_x[i], tc.x), G.resolution))) - G.lo[0];
          const int y = static_cast<int>(lroundf(__fdiv_rn(__fadd_rn(s_y[i], tc.y), G.resolution))) - G.lo[1];
          const int z = static_cast<int>(lroundf(__fdiv_rn(__fadd_rn(s_z[i], tc.z), G.resolution))) - G.lo[2];
          int value = 0;
          if (static_cast<unsigned>(x) < static_cast<unsigned>(G.n[0]) &&
              static_cast<unsigned>(y) < static_cast<unsigned>(G.n[1]) &&
              static_cast<unsigned>(z) < static_cast<unsigned>(G.n[2]))
            value = __ldg(G.p + (static_cast<size_t>(z) * G.n[1] + y) * G.n[0] + x) & 0x7fff;
          // HybridGrid::GetProbability = ValueToProbability (probability_values.cc:29-37,56-60)
          const float prob = value == 0 ? G.min_probability
                                        : __fadd_rn(__fmul_rn(__int2float_rn(value), G.k_scale), G.bias);
          sum = __fadd_rn(sum, prob);
        }
      }
    }
    if (on) {
      float score = __fdiv_rn(sum, __int2float_rn(P.n));
      const double w = weights[static_cast<size_t>(__float_as_int(tc.w)) * P.R + r];
      score = __double2float_rn(__dmul_rn(static_cast<double>(score), w));  // float *= double (:109)
      const unsigned c = static_cast<unsigned>(t) * static_cast<unsigned>(P.R) + static_cast<unsigned>(r);
      const unsigned long long key =
          (static_cast<unsigned long long>(__float_as_uint(fmaxf(score, 0.f))) << 32) |
          (0xffffffffu - c);
      atomicMax(&s_best, key);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) atomicMax(best, s_best);
}

}  // namespace csm

using namespace csm;

namespace {

// ---- Eigen semantics on the host (same restatement as engine3d.cu / oracle_3d.cc) ----
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
Qf HNormalized(const Qf& q) {
  const float z = (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w);
  if (z > 0.f) {
    const float n = std::sqrt(z);
    return Qf{q.w / n, q.x / n, q.y / n, q.z / n};
  }
  return q;
}
Qf HAngleAxis(const Vf& aa) {  // transform/transform.h:85-99
  float scale = 0.5f, w = 1.f;
  const float sq = aa.x * aa.x + aa.y * aa.y + aa.z * aa.z;
  if (sq > 1e-8) {
    const float norm = std::sqrt(sq);
    scale = static_cast<float>(std::sin(norm / 2.) / norm);
    w = static_cast<float>(std::cos(norm / 2.));
  }
  return Qf{w, scale * aa.x, scale * aa.y, scale * aa.z};
}

}  // namespace

extern "C" {

csm_status csm_grid3d_create(const int32_t* idx, const uint16_t* values, int64_t n,
                             float resolution, int32_t device, csm_grid3d** out) {
  CSM_REQUIRE(out != nullptr, "null pointer");
  CSM_REQUIRE(n >= 0 && (n == 0 || (idx && values)), "voxel list");
  CSM_REQUIRE(resolution > 0.f, "resolution");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  cudaStream_t s = ctx->stream;
  std::unique_ptr<csm_grid3d> g(new csm_grid3d);
  g->ctx = ctx;
  Grid3Dev& d = g->g;
  std::memset(&d, 0, sizeof(d));
  int lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  for (int64_t i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) {
      const int v = idx[3 * i + a];
      if (i == 0 || v < lo[a]) lo[a] = v;
      if (i == 0 || v > hi[a]) hi[a] = v;
    }
  for (int a = 0; a < 3; ++a) {
    CSM_REQUIRE(lo[a] >= -8192 && hi[a] < 8192, "voxel index outside the 2^14 cube");  // hybrid_grid.h:387
    d.lo[a] = lo[a];
    d.n[a] = hi[a] - lo[a] + 1;
    g->tight.lo[a] = lo[a];
    g->tight.hi[a] = hi[a];
  }
  g->tight.empty = n == 0;
  const size_t vox = static_cast<size_t>(d.n[0]) * d.n[1] * d.n[2];
  CSM_REQUIRE(vox < (size_t(8) << 30), "dense volume too large");
  // whole 32-bit words: the inserter clears update markers with 32-bit atomics (insert3d.cu)
  const size_t bytes = std::max<size_t>((vox * 2 + 3) / 4 * 4, 256);
  CSM_CUDA(cudaMalloc(&g->d_vol, bytes));
  CSM_CUDA(cudaMemsetAsync(g->d_vol, 0, bytes, s));
  d.p = g->d_vol;
  d.resolution = resolution;
  {
    const float kMin = 0.1f, kMax = 1.f - kMin;
    d.k_scale = (kMax - kMin) / 32766.f;
    d.bias = kMin - d.k_scale;
    d.min_probability = kMin;
  }
  if (n > 0) {
    DevBuf& d_idx = ctx->D("g3_idx");
    DevBuf& d_val = ctx->D("g3_val");
    CSM_TRY(d_idx.Reserve(sizeof(int) * 3 * n));
    CSM_TRY(d_val.Reserve(sizeof(uint16_t) * n));
    CSM_CUDA(cudaMemcpyAsync(d_idx.p, idx, sizeof(int) * 3 * n, cudaMemcpyHostToDevice, s));
    CSM_CUDA(cudaMemcpyAsync(d_val.p, values, sizeof(uint16_t) * n, cudaMemcpyHostToDevice, s));
    k_rt3_scatter<<<DivUp(n, 256), 256, 0, s>>>(d_idx.as<int>(), d_val.as<uint16_t>(), n, d,
                                                 g->d_vol);
    CSM_LAUNCH_CHECK();
  }
  CSM_CUDA(cudaStreamSynchronize(s));
  *out = g.release();
  return CSM_OK;
}

csm_status csm_grid3d_destroy(csm_grid3d* grid) {
  if (!grid) return CSM_OK;
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  cudaSetDevice(grid->ctx->device);
  cudaStreamSynchronize(grid->ctx->stream);
  delete grid;
  return CSM_OK;
}

csm_status csm_rt_match3d(const csm_grid3d* grid, const float* xyz, int32_t n,
                          const double initial_pose[7], double linear_window,
                          double angular_window, double w_t, double w_r, float* score,
                          double pose_estimate[7], csm_stats* stats) {
  CSM_REQUIRE(grid && xyz && initial_pose && score && pose_estimate, "null pointer");  // :38
  CSM_REQUIRE(n >= 1, "empty point cloud");
  LaneGuard guard;
  CSM_TRY(AcquireLane(grid->ctx->device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const float resolution = grid->g.resolution;
  // GenerateExhaustiveSearchTransforms (:55-98)
  const int L = static_cast<int>(std::lround(linear_window / resolution));
  float max_scan_range = 3.f * resolution;
  for (int i = 0; i < n; ++i) {
    const float* p = xyz + 3 * i;
    const float range = std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    max_scan_range = std::max(range, max_scan_range);
  }
  const float kSafetyMargin = 1.f - 1e-3f;
  const float angular_step_size =
      kSafetyMargin * std::acos(1.f - (resolution * resolution) /
                                          (2.f * (max_scan_range * max_scan_range)));
  const int A = static_cast<int>(std::lround(angular_window / angular_step_size));
  CSM_REQUIRE(L >= 0 && L <= 64 && A >= 0 && A <= 64, "search window");
  const int W = 2 * L + 1, Rw = 2 * A + 1;
  const long long T = static_cast<long long>(W) * W * W, R = static_cast<long long>(Rw) * Rw * Rw;
  CSM_REQUIRE(T * R < (1LL << 31), "search window too large");
  // initial_pose_estimate.cast<float>()
  const Vf t_init{static_cast<float>(initial_pose[0]), static_cast<float>(initial_pose[1]),
                  static_cast<float>(initial_pose[2])};
  const Qf q_init{static_cast<float>(initial_pose[3]), static_cast<float>(initial_pose[4]),
                  static_cast<float>(initial_pose[5]), static_cast<float>(initial_pose[6])};
  // per rotation: transform rotation, candidate rotation = (q_init * q_r).normalized()
  // (rigid_transform.h:181-189) and GetAngle(transform) (transform.h:34-37)
  std::vector<Qf> q_r(R), q_c(R);
  std::vector<float> angle(R);
  {
    long long r = 0;
    for (int rz = -A; rz <= A; ++rz)
      for (int ry = -A; ry <= A; ++ry)
        for (int rx = -A; rx <= A; ++rx, ++r) {
          const Qf q = HAngleAxis(Vf{rx * angular_step_size, ry * angular_step_size,
                                     rz * angular_step_size});
          q_r[r] = q;
          q_c[r] = HNormalized(HMul(q_init, q));
          const float vec_norm = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
          angle[r] = 2.f * std::atan2(vec_norm, std::abs(q.w));
        }
  }
  // per translation: candidate translation = q_init * t + t_init, and its norm class
  std::vector<float4> trans(T);
  std::map<unsigned, int> klass;   // norm bits -> class
  std::vector<float> class_norm;
  {
    long long t = 0;
    for (int z = -L; z <= L; ++z)
      for (int y = -L; y <= L; ++y)
        for (int x = -L; x <= L; ++x, ++t) {
          const Vf tv{x * resolution, y * resolution, z * resolution};
          const Vf rt = HRot(q_init, tv);
          const float norm = std::sqrt(tv.x * tv.x + tv.y * tv.y + tv.z * tv.z);
          unsigned bits;
          std::memcpy(&bits, &norm, 4);
          auto it = klass.find(bits);
          if (it == klass.end()) {
            it = klass.emplace(bits, static_cast<int>(class_norm.size())).first;
            class_norm.push_back(norm);
          }
          float cls;
          std::memcpy(&cls, &it->second, 4);
          trans[t] = make_float4(rt.x + t_init.x, rt.y + t_init.y, rt.z + t_init.z, cls);
        }
  }
  // weights per (norm class, rotation): exp(-(norm * w_t + angle * w_r)^2) in double (:109-114)
  const size_t K = class_norm.size();
  std::vector<double> weights(K * R);
  for (size_t k = 0; k < K; ++k)
    for (long long r = 0; r < R; ++r) {
      const double e = class_norm[k] * w_t + angle[r] * w_r;
      weights[k * R + r] = std::exp(-(e * e));
    }
  // upload: cloud | rotations | translations | weights
  const size_t o_rot = (static_cast<size_t>(n) * 12 + 255) / 256 * 256;
  const size_t o_tr = (o_rot + static_cast<size_t>(R) * 16 + 255) / 256 * 256;
  const size_t o_w = (o_tr + static_cast<size_t>(T) * 16 + 255) / 256 * 256;
  const size_t bytes = o_w + weights.size() * 8;
  PinnedBuf& up = ctx->P("rt3_upload");
  DevBuf& d_up = ctx->D("rt3_upload");
  DevBuf& d_best = ctx->D("rt3_best");
  PinnedBuf& rb = ctx->P("rt3_readback");
  CSM_TRY(up.Reserve(bytes));
  CSM_TRY(d_up.Reserve(bytes));
  CSM_TRY(d_best.Reserve(8));
  CSM_TRY(rb.Reserve(8));
  char* h = up.as<char>();
  std::memcpy(h, xyz, static_cast<size_t>(n) * 12);
  for (long long r = 0; r < R; ++r)
    reinterpret_cast<float4*>(h + o_rot)[r] = make_float4(q_c[r].w, q_c[r].x, q_c[r].y, q_c[r].z);
  std::memcpy(h + o_tr, trans.data(), static_cast<size_t>(T) * 16);
  std::memcpy(h + o_w, weights.data(), weights.size() * 8);
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_CUDA(cudaMemcpyAsync(d_up.p, h, bytes, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemsetAsync(d_best.p, 0, 8, s));
  Rt3Params P;
  P.n = n;
  P.T = static_cast<int>(T);
  P.R = static_cast<int>(R);
  const char* d = d_up.as<char>();
  ProfBegin(ctx);
  k_rt3_match<<<static_cast<int>(R), 128, 0, s>>>(
      grid->g, P, reinterpret_cast<const float*>(d), reinterpret_cast<const float4*>(d + o_rot),
      reinterpret_cast<const float4*>(d + o_tr), reinterpret_cast<const double*>(d + o_w),
      d_best.as<unsigned long long>());
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, "k_rt3_match", static_cast<double>(T * R));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(rb.p, d_best.p, 8, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  const unsigned long long key = *rb.as<unsigned long long>();
  const unsigned bits = static_cast<unsigned>(key >> 32);
  const unsigned c = 0xffffffffu - static_cast<unsigned>(key & 0xffffffffu);
  float best_score;
  std::memcpy(&best_score, &bits, 4);
  const long long t = c / R, r = c % R;
  *score = best_score;
  // candidate.cast<double>()
  pose_estimate[0] = trans[t].x;
  pose_estimate[1] = trans[t].y;
  pose_estimate[2] = trans[t].z;
  pose_estimate[3] = q_c[r].w;
  pose_estimate[4] = q_c[r].x;
  pose_estimate[5] = q_c[r].y;
  pose_estimate[6] = q_c[r].z;
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->candidates_scored = T * R;
    stats->lowest_resolution_candidates = T * R;
    stats->num_scans = static_cast<int32_t>(R);
    stats->best_scan_index = static_cast<int32_t>(r);
    stats->best_x_offset = static_cast<int32_t>(t);
    stats->leaves_tied = 1;
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

}  // extern "C"
