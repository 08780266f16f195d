// The grid-resident ProbabilityGrid / TSDF2D handle shared by the real-time matcher
// (rt2d.cu), the post-match refinement (refine2d.cu) and the 2D range data inserters
// (insert2d.cu, insert_tsdf2d.cu).
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

// Grid2D::known_cells_box_ (2d/grid_2d.h): inclusive cell bounds, empty when lo > hi.
struct KnownBox2 {
  int lo[2] = {1, 1};
  int hi[2] = {0, 0};
  bool empty() const { return lo[0] > hi[0]; }
  void Extend(int x, int y) {
    if (empty()) {
      lo[0] = hi[0] = x;
      lo[1] = hi[1] = y;
      return;
    }
    lo[0] = x < lo[0] ? x : lo[0];
    lo[1] = y < lo[1] ? y : lo[1];
    hi[0] = x > hi[0] ? x : hi[0];
    hi[1] = y > hi[1] ? y : hi[1];
  }
  void Extend(const KnownBox2& o) {
    if (o.empty()) return;
    Extend(o.lo[0], o.lo[1]);
    Extend(o.hi[0], o.hi[1]);
  }
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
  // The known-cells box.  A handle made from cells (or refreshed by an update) takes the
  // bounding box of its non-zero cells, computed on the device when an insert, crop or read
  // first needs it (known_stale until then).
  csm::KnownBox2 known;
  bool known_stale = true;
  ~csm_rt_grid2d() {
    cudaFree(d_cells);
    cudaFree(d_wcells);
  }
};

namespace csm {

// (Re-)encodes the handle's TMA box and descriptor for its current cell array and
// dimensions (rt2d.cu).  Caller holds ctx->mu.
csm_status RtGridEncodeTmap(csm_rt_grid2d* g);

// Brings grid->known up to date (one stream synchronisation when it is stale; insert2d.cu).
// Caller holds ctx->mu.
csm_status RtGridKnownBox(csm_rt_grid2d* grid);

}  // namespace csm

#endif  // CSM_RTGRID_CUH_
