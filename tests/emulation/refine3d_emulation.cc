// TEST INFRASTRUCTURE ONLY — see refine2d_emulation.cc.  Runs the DEVICE code of
// cartographer_b200/csrc/refine3d.cu (k_ceres_match3d and helpers, included verbatim) on the
// CPU, one std::thread per CUDA thread of one CTA, to check the kernel's control flow against
// the oracle where no GPU is present.  Not a fallback; never linked into the library.
#include <pthread.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#define CSM_REFINE_DEVICE_ONLY 1
#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__
#define __shared__ static
#define __launch_bounds__(...)

namespace {
struct Dim3 { unsigned x = 0, y = 0, z = 0; };
thread_local Dim3 threadIdx, blockIdx, blockDim;

constexpr int kEmuThreads = 256;
pthread_barrier_t g_block_barrier;
pthread_barrier_t g_warp_barrier[kEmuThreads / 32];
double g_shfl[kEmuThreads / 32][32];

inline void __syncthreads() { pthread_barrier_wait(&g_block_barrier); }
inline double __shfl_down_sync(unsigned, double v, int o) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  g_shfl[warp][lane] = v;
  pthread_barrier_wait(&g_warp_barrier[warp]);
  const double r = lane + o < 32 ? g_shfl[warp][lane + o] : v;
  pthread_barrier_wait(&g_warp_barrier[warp]);
  return r;
}
template <typename T> inline T __ldg(const T* p) { return *p; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __int2float_rn(int v) { return static_cast<float>(v); }
using std::isfinite;
}  // namespace

#include "../../cartographer_b200/csrc/refine3d.cu"
#include "../../cartographer_b200/csrc/value_conversion.h"

namespace {
void FillEmuJob(int num_clouds, const uint16_t* const* vol, const int32_t* lo, const int32_t* n,
                const float* resolution, const float* const* xyz, const int32_t* npts,
                const double* target_t, const double* init_pose, csm::Ref3JobDev* job,
                std::vector<float>* cloud) {
  std::memset(job, 0, sizeof(*job));
  job->num_clouds = num_clouds;
  for (int b = 0; b < num_clouds; ++b) {
    csm::Ref3Cloud& c = job->c[b];
    c.vol = vol[b];
    for (int a = 0; a < 3; ++a) {
      c.lo[a] = lo[3 * b + a];
      c.n[a] = n[3 * b + a];
    }
    c.resolution = resolution[b];
    // as MakeGrid3Dev (grid3d.cu) fills them
    const csm::ValueConversion probability =
        csm::MakeValueConversion(csm::kMinProbability, csm::kMaxProbability);
    c.k_scale = probability.scale;
    c.bias = probability.bias;
    c.min_probability = csm::kMinProbability;
    c.npts = npts[b];
    c.xyz_off = static_cast<long long>(cloud->size());
    cloud->insert(cloud->end(), xyz[b], xyz[b] + 3 * static_cast<size_t>(npts[b]));
  }
  for (int k = 0; k < 3; ++k) job->target_t[k] = target_t[k];
  for (int k = 0; k < 7; ++k) job->init[k] = init_pose[k];
}
}  // namespace

extern "C" {

// k_ceres_evaluate3d, one emulated thread after the other (the kernel has no barriers).
// opts = {translation_weight, rotation_weight, occupied_space_weight_0, _1}
void emu_ceres_evaluate3d(int num_clouds, const uint16_t* const* vol, const int32_t* lo,
                          const int32_t* n, const float* resolution, const float* const* xyz,
                          const int32_t* npts, const double* opts, const double* target_t,
                          const double* target_q, const double* pose, int with_jacobian,
                          double* residuals, double* jacobian) {
  csm::Ref3JobDev job;
  std::vector<float> cloud;
  const double init[7] = {0., 0., 0., target_q[0], target_q[1], target_q[2], target_q[3]};
  FillEmuJob(num_clouds, vol, lo, n, resolution, xyz, npts, target_t, init, &job, &cloud);
  csm::Ref3Opts P;
  std::memset(&P, 0, sizeof(P));
  P.translation_weight = opts[0];
  P.rotation_weight = opts[1];
  P.occupied_space_weight[0] = opts[2];
  P.occupied_space_weight[1] = opts[3];
  int rows = 6;
  for (int b = 0; b < num_clouds; ++b) rows += npts[b];
  blockDim.x = 256;
  for (int blk = 0; blk < (rows + 255) / 256; ++blk)
    for (int t = 0; t < 256; ++t) {
      blockIdx.x = blk;
      threadIdx.x = t;
      csm::k_ceres_evaluate3d(&job, P, cloud.data(), pose, with_jacobian, residuals, jacobian);
    }
}

// Dense boxes as csm_grid3d_create builds them: vol[b] has n[b][0..2] cells from lo[b][0..2].
// opts = {translation_weight, rotation_weight, use_nonmonotonic_steps, max_num_iterations,
//         occupied_space_weight_0, occupied_space_weight_1}
// out = {pose[7], initial_cost, final_cost, iterations, num_successful_steps, termination}
void emu_ceres_match3d(int num_clouds, const uint16_t* const* vol, const int32_t* lo,
                       const int32_t* n, const float* resolution, const float* const* xyz,
                       const int32_t* npts, const double* opts, const double* target_t,
                       const double* init_pose, double* out) {
  csm::Ref3JobDev job;
  std::vector<float> cloud;
  FillEmuJob(num_clouds, vol, lo, n, resolution, xyz, npts, target_t, init_pose, &job, &cloud);
  csm::Ref3Opts P;
  P.translation_weight = opts[0];
  P.rotation_weight = opts[1];
  P.use_nonmonotonic_steps = opts[2] != 0.;
  P.max_num_iterations = static_cast<int>(opts[3]);
  P.occupied_space_weight[0] = opts[4];
  P.occupied_space_weight[1] = opts[5];
  csm::Ref3ResultDev result;
  std::memset(&result, 0, sizeof(result));
  pthread_barrier_init(&g_block_barrier, nullptr, kEmuThreads);
  for (auto& b : g_warp_barrier) pthread_barrier_init(&b, nullptr, 32);
  std::vector<std::thread> threads;
  for (int t = 0; t < kEmuThreads; ++t)
    threads.emplace_back([&, t] {
      threadIdx.x = t;
      blockIdx.x = 0;
      csm::k_ceres_match3d(&job, P, cloud.data(), &result);
    });
  for (auto& t : threads) t.join();
  pthread_barrier_destroy(&g_block_barrier);
  for (auto& b : g_warp_barrier) pthread_barrier_destroy(&b);
  for (int k = 0; k < 7; ++k) out[k] = result.pose[k];
  out[7] = result.initial_cost;
  out[8] = result.final_cost;
  out[9] = result.iterations;
  out[10] = result.num_successful_steps;
  out[11] = result.termination;
}

}  // extern "C"
