// TEST INFRASTRUCTURE ONLY — never linked into libcsm_b200.so and never used by the product.
//
// The TSDF2D instantiation of k_ceres_match2d (cartographer_b200/csrc/refine2d.cu, included
// verbatim) run on the CPU as refine2d_emulation.cc runs the ProbabilityGrid one: one
// std::thread per CUDA thread of a CTA, pthread barriers for __syncthreads and the warp
// shuffles.  It checks the two-pass evaluation's barriers and hand-offs and the failure
// paths of the minimiser against the CPU restatement (tests/tsdf2d_oracle.py).
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
#include "../../cartographer_b200/csrc/tsdf_conversion.h"

namespace {

// One CTA of k_ceres_match2d for one TSDF2D job whose rows are `pitch` cells apart.
void RunMatchTsdf(const uint16_t* tsd_cells, const uint16_t* weight_cells, int nx, int ny,
                  int pitch, const double* grid, const float* xyz, int n, const double* opts,
                  const double* target_xy, const double* init_pose, double* out) {
  csm::RefJobDev job;
  std::memset(&job, 0, sizeof(job));
  job.cells = tsd_cells;
  job.nx = nx;
  job.ny = ny;
  job.pitch = pitch;
  job.n = n;
  job.resolution = grid[0];
  job.max_x = grid[1];
  job.max_y = grid[2];
  job.target[0] = target_xy[0];
  job.target[1] = target_xy[1];
  for (int k = 0; k < 3; ++k) job.init[k] = init_pose[k];
  const float truncation = static_cast<float>(grid[3]);
  const csm::TsdfConversion c = csm::MakeTsdfConversion(truncation, static_cast<float>(grid[4]));
  job.wcells = weight_cells;
  job.tsd_scale = c.tsd_scale;
  job.tsd_bias = c.tsd_bias;
  job.w_scale = c.w_scale;
  job.w_bias = c.w_bias;
  job.truncation = truncation;
  csm::RefOpts P;
  std::memset(&P, 0, sizeof(P));
  P.occupied_space_weight = opts[0];
  P.translation_weight = opts[1];
  P.rotation_weight = opts[2];
  P.use_nonmonotonic_steps = opts[3] != 0.;
  P.max_num_iterations = static_cast<int>(opts[4]);
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

// grid = {resolution, max_x, max_y, truncation, max_weight}; opts = {occupied, translation,
// rotation, use_nonmonotonic_steps, max_num_iterations}; out = {pose[3], initial_cost,
// final_cost, iterations, num_successful_steps, termination}.
void emu_ceres_match2d_tsdf(const uint16_t* tsd_cells, const uint16_t* weight_cells, int nx,
                            int ny, const double* grid, const float* xyz, int n,
                            const double* opts, const double* target_xy,
                            const double* init_pose, double* out) {
  RunMatchTsdf(tsd_cells, weight_cells, nx, ny, nx, grid, xyz, n, opts, target_xy, init_pose, out);
}

// As emu_ceres_match2d_tsdf with both cell arrays in rows of `pitch` >= nx.
void emu_ceres_match2d_tsdf_pitched(const uint16_t* tsd_cells, const uint16_t* weight_cells,
                                    int nx, int ny, int pitch, const double* grid,
                                    const float* xyz, int n, const double* opts,
                                    const double* target_xy, const double* init_pose,
                                    double* out) {
  RunMatchTsdf(tsd_cells, weight_cells, nx, ny, pitch, grid, xyz, n, opts, target_xy, init_pose,
               out);
}

}  // extern "C"
