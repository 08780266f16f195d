// TEST INFRASTRUCTURE ONLY — never linked into libcsm_b200.so and never used by the product.
//
// Runs the DEVICE code of cartographer_b200/csrc/refine2d.cu (k_ceres_match2d and its helper
// functions, included verbatim) on the CPU: one std::thread per CUDA thread of a CTA,
// pthread barriers for __syncthreads and for the warp shuffles.  The container that develops
// this repository has no GPU; this harness lets `-m "not gpu"` tests check the kernel's
// control flow (uniform branches around barriers, shared-memory hand-offs, the minimiser's
// state machine) against the oracle before a GPU run.  It proves nothing about performance
// and is not a fallback: the library has no CPU path.
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
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __int2float_rn(int v) { return static_cast<float>(v); }
using std::isfinite;
}  // namespace

#include "../../cartographer_b200/csrc/refine2d.cu"
#include "../../cartographer_b200/csrc/value_conversion.h"

namespace {

// One CTA of k_ceres_match2d for one job whose rows are `pitch` cells apart.
void RunMatch2D(const uint16_t* cells, int nx, int ny, int pitch, double resolution, double max_x,
                double max_y, const float* xyz, int n, const double* opts,
                const double* target_xy, const double* init_pose, double* out) {
  csm::RefJobDev job;
  std::memset(&job, 0, sizeof(job));
  job.cells = cells;
  job.nx = nx;
  job.ny = ny;
  job.pitch = pitch;
  job.n = n;
  job.xyz_off = 0;
  job.resolution = resolution;
  job.max_x = max_x;
  job.max_y = max_y;
  job.target[0] = target_xy[0];
  job.target[1] = target_xy[1];
  for (int k = 0; k < 3; ++k) job.init[k] = init_pose[k];
  csm::RefOpts P;
  P.occupied_space_weight = opts[0];
  P.translation_weight = opts[1];
  P.rotation_weight = opts[2];
  P.use_nonmonotonic_steps = opts[3] != 0.;
  P.max_num_iterations = static_cast<int>(opts[4]);
  const csm::ValueConversion cost =
      csm::MakeValueConversion(csm::kMinCorrespondenceCost, csm::kMaxCorrespondenceCost);
  P.k_scale = cost.scale;
  P.cost_bias = cost.bias;
  P.max_cost = csm::kMaxCorrespondenceCost;
  csm::RefResultDev result;
  std::memset(&result, 0, sizeof(result));
  pthread_barrier_init(&g_block_barrier, nullptr, kEmuThreads);
  for (auto& b : g_warp_barrier) pthread_barrier_init(&b, nullptr, 32);
  std::vector<std::thread> threads;
  for (int t = 0; t < kEmuThreads; ++t)
    threads.emplace_back([&, t] {
      threadIdx.x = t;
      blockIdx.x = 0;
      csm::k_ceres_match2d(&job, P, xyz, &result);
    });
  for (auto& t : threads) t.join();
  pthread_barrier_destroy(&g_block_barrier);
  for (auto& b : g_warp_barrier) pthread_barrier_destroy(&b);
  out[0] = result.pose[0];
  out[1] = result.pose[1];
  out[2] = result.pose[2];
  out[3] = result.initial_cost;
  out[4] = result.final_cost;
  out[5] = result.iterations;
  out[6] = result.num_successful_steps;
  out[7] = result.termination;
}

}  // namespace

extern "C" {

// opts = {occupied, translation, rotation, use_nonmonotonic_steps, max_num_iterations};
// out = {pose[3], initial_cost, final_cost, iterations, num_successful_steps, termination}.
void emu_ceres_match2d(const uint16_t* cells, int nx, int ny, double resolution, double max_x,
                       double max_y, const float* xyz, int n, const double* opts,
                       const double* target_xy, const double* init_pose, double* out) {
  RunMatch2D(cells, nx, ny, nx, resolution, max_x, max_y, xyz, n, opts, target_xy, init_pose, out);
}

// As emu_ceres_match2d with the cells in rows of `pitch` >= nx, as a device handle keeps them.
void emu_ceres_match2d_pitched(const uint16_t* cells, int nx, int ny, int pitch,
                               double resolution, double max_x, double max_y, const float* xyz,
                               int n, const double* opts, const double* target_xy,
                               const double* init_pose, double* out) {
  RunMatch2D(cells, nx, ny, pitch, resolution, max_x, max_y, xyz, n, opts, target_xy, init_pose,
             out);
}

}  // extern "C"
