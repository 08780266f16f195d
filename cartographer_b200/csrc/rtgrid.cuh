// The grid-resident ProbabilityGrid / TSDF2D handle shared by the real-time matcher
// (rt2d.cu) and the post-match refinement (refine2d.cu).
#ifndef CSM_RTGRID_CUH_
#define CSM_RTGRID_CUH_

#include <cuda.h>

#include "common.cuh"
#include "tsdf_conversion.h"

namespace csm {

struct RtGridDev {
  const uint16_t* cells;    // device copy, row pitch `pitch` cells
  const uint16_t* wcells;   // TSDF weight cells (nullptr for a ProbabilityGrid)
  int nx, ny, pitch;
  int bw, bh;               // TMA box (cells)
  double resolution, max_x, max_y;
};

}  // namespace csm

struct csm_rt_grid2d {
  csm::Ctx* ctx = nullptr;
  csm::RtGridDev g;
  uint16_t* d_cells = nullptr;
  uint16_t* d_wcells = nullptr;
  CUtensorMap tmap;
  bool has_tmap = false;
  float truncation = 0.f, max_weight = 0.f;
  ~csm_rt_grid2d() {
    cudaFree(d_cells);
    cudaFree(d_wcells);
  }
};

#endif  // CSM_RTGRID_CUH_
