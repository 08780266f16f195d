// The dense device copy of a HybridGrid (csm_grid3d) shared by the real-time 3D matcher
// (rt3d.cu), the 3D post-match refinement (refine3d.cu) and the range-data inserter
// (insert3d.cu).
#ifndef CSM_GRID3D_CUH_
#define CSM_GRID3D_CUH_

#include "common.cuh"

namespace csm {

struct Grid3Dev {
  const uint16_t* p;   // dense box of HybridGrid values (0 outside / unallocated)
  int lo[3];
  int n[3];
  float resolution, k_scale, bias, min_probability;
};

// The smallest box holding every voxel a handle was made from and every origin / hit cell
// inserted since; empty until the first of them.  The dense box always contains it, and
// insert3d.cu sizes a grown box from it.
struct TightBox3 {
  bool empty = true;
  int lo[3] = {0, 0, 0};
  int hi[3] = {0, 0, 0};
};

}  // namespace csm

struct csm_grid3d {
  csm::Ctx* ctx = nullptr;
  csm::Grid3Dev g;
  uint16_t* d_vol = nullptr;
  csm::TightBox3 tight;
  ~csm_grid3d() { cudaFree(d_vol); }
};

// The dense device copy of an IntensityHybridGrid (refine3d.cu): GetIntensity per voxel of
// the bounding box of the voxels it was made from, 0 elsewhere.  The first insert
// (insert3d.cu) adds the AverageIntensityData volumes d_sum / d_count, filled from the voxel
// list the handle was made from (kept on the host until then).
struct csm_intensity_grid3d {
  csm::Ctx* ctx = nullptr;
  float* d_vol = nullptr;
  int lo[3] = {0, 0, 0};
  int n[3] = {0, 0, 0};
  float resolution = 0.f;
  csm::TightBox3 tight;
  float* d_sum = nullptr;
  int32_t* d_count = nullptr;
  std::vector<int32_t> made_idx, made_count;
  std::vector<float> made_sum;
  ~csm_intensity_grid3d() {
    cudaFree(d_vol);
    cudaFree(d_sum);
    cudaFree(d_count);
  }
};

namespace csm {

// The number *n of non-zero voxels of `g` and, when it is at most list_capacity, the voxels in
// HybridGrid's iteration order in device workspaces: *d_idx ({x, y, z} each) and *d_val, ready on
// the context's stream (engine3d.cu, what csm_grid3d_voxels returns).  Caller holds ctx->mu.
csm_status NonZeroVoxels3D(const csm_grid3d* g, long long list_capacity, long long* n,
                           const int** d_idx, const uint16_t** d_val);

}  // namespace csm

#endif  // CSM_GRID3D_CUH_
