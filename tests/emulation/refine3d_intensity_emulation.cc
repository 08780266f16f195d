// TEST INFRASTRUCTURE ONLY — see refine3d_emulation.cc, which this harness includes (and so
// the DEVICE code of cartographer_b200/csrc/refine3d.cu with it).  Adds entry points whose
// jobs carry IntensityCostFunction3D blocks, to check the kernel's intensity path and its
// Huber correction against the oracle where no GPU is present.  Never linked into the library.
#include "refine3d_emulation.cc"

namespace {
// Cloud b's intensity block: ivol[b] == NULL leaves it out.  The dense boxes hold
// GetIntensity as csm_intensity_grid3d_create builds them; iopts = {weight, huber_scale,
// intensity_threshold} per cloud.
void FillEmuIntensity(int num_clouds, const float* const* ivol, const int32_t* ilo,
                      const int32_t* in, const float* iresolution,
                      const float* const* intensities, const int32_t* npts, const double* iopts,
                      csm::Ref3IntensityJobDev* job, std::vector<float>* cloud) {
  std::memset(job, 0, sizeof(*job));
  for (int b = 0; b < num_clouds; ++b) {
    if (ivol[b] == nullptr) continue;
    csm::Ref3IntensityCloud& c = job->c[b];
    c.ivol = ivol[b];
    for (int a = 0; a < 3; ++a) {
      c.ilo[a] = ilo[3 * b + a];
      c.in[a] = in[3 * b + a];
    }
    c.iresolution = iresolution[b];
    c.intensity_off = static_cast<long long>(cloud->size());
    cloud->insert(cloud->end(), intensities[b], intensities[b] + npts[b]);
    c.intensity_weight = iopts[3 * b];
    c.huber_scale = iopts[3 * b + 1];
    c.intensity_threshold = static_cast<float>(iopts[3 * b + 2]);
  }
}
}  // namespace

extern "C" {

// emu_ceres_evaluate3d with intensity blocks (k_ceres_evaluate3d_intensity; rows in the
// problem's residual-block order)
void emu_ceres_evaluate3d_intensity(int num_clouds, const uint16_t* const* vol, const int32_t* lo,
                                    const int32_t* n, const float* resolution,
                                    const float* const* xyz, const int32_t* npts,
                                    const double* opts, const float* const* ivol,
                                    const int32_t* ilo, const int32_t* in,
                                    const float* iresolution, const float* const* intensities,
                                    const double* iopts, const double* target_t,
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
  csm::Ref3IntensityJobDev ijob;
  FillEmuIntensity(num_clouds, ivol, ilo, in, iresolution, intensities, npts, iopts, &ijob,
                   &cloud);
  int rows = 6;
  for (int b = 0; b < num_clouds; ++b) rows += npts[b] * (ivol[b] != nullptr ? 2 : 1);
  blockDim.x = 256;
  for (int blk = 0; blk < (rows + 255) / 256; ++blk)
    for (int t = 0; t < 256; ++t) {
      blockIdx.x = blk;
      threadIdx.x = t;
      csm::k_ceres_evaluate3d_intensity(&job, &ijob, P, cloud.data(), pose, with_jacobian,
                                        residuals, jacobian);
    }
}

// emu_ceres_match3d with intensity blocks (k_ceres_match3d_intensity); opts and out as there.
void emu_ceres_match3d_intensity(int num_clouds, const uint16_t* const* vol, const int32_t* lo,
                                 const int32_t* n, const float* resolution,
                                 const float* const* xyz, const int32_t* npts, const double* opts,
                                 const float* const* ivol, const int32_t* ilo, const int32_t* in,
                                 const float* iresolution, const float* const* intensities,
                                 const double* iopts, const double* target_t,
                                 const double* init_pose, double* out) {
  csm::Ref3JobDev job;
  std::vector<float> cloud;
  FillEmuJob(num_clouds, vol, lo, n, resolution, xyz, npts, target_t, init_pose, &job, &cloud);
  csm::Ref3Opts P;
  std::memset(&P, 0, sizeof(P));
  P.translation_weight = opts[0];
  P.rotation_weight = opts[1];
  P.use_nonmonotonic_steps = opts[2] != 0.;
  P.max_num_iterations = static_cast<int>(opts[3]);
  P.occupied_space_weight[0] = opts[4];
  P.occupied_space_weight[1] = opts[5];
  csm::Ref3IntensityJobDev ijob;
  FillEmuIntensity(num_clouds, ivol, ilo, in, iresolution, intensities, npts, iopts, &ijob,
                   &cloud);
  csm::Ref3ResultDev result;
  std::memset(&result, 0, sizeof(result));
  pthread_barrier_init(&g_block_barrier, nullptr, kEmuThreads);
  for (auto& b : g_warp_barrier) pthread_barrier_init(&b, nullptr, 32);
  std::vector<std::thread> threads;
  for (int t = 0; t < kEmuThreads; ++t)
    threads.emplace_back([&, t] {
      threadIdx.x = t;
      blockIdx.x = 0;
      csm::k_ceres_match3d_intensity(&job, &ijob, P, cloud.data(), &result);
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
