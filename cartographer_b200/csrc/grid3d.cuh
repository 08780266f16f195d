// The dense device copy of a HybridGrid (csm_grid3d) shared by the real-time 3D matcher
// (rt3d.cu) and the 3D post-match refinement (refine3d.cu).
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

}  // namespace csm

struct csm_grid3d {
  csm::Ctx* ctx = nullptr;
  csm::Grid3Dev g;
  uint16_t* d_vol = nullptr;
  ~csm_grid3d() { cudaFree(d_vol); }
};

// The dense device copy of an IntensityHybridGrid (refine3d.cu): GetIntensity per voxel of
// the bounding box of the voxels it was made from, 0 elsewhere.
struct csm_intensity_grid3d {
  csm::Ctx* ctx = nullptr;
  float* d_vol = nullptr;
  int lo[3] = {0, 0, 0};
  int n[3] = {0, 0, 0};
  float resolution = 0.f;
  ~csm_intensity_grid3d() { cudaFree(d_vol); }
};

#endif  // CSM_GRID3D_CUH_
