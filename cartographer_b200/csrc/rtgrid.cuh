// The grid-resident ProbabilityGrid / TSDF2D handle (grid2d.cu) shared by the real-time matcher
// (rt2d.cu), the post-match refinement (refine2d.cu), the precomputation stack (engine2d.cu) and
// the 2D range data inserters (insert2d.cu, insert_tsdf2d.cu).
#ifndef CSM_RTGRID_CUH_
#define CSM_RTGRID_CUH_

#include <cuda.h>

#include <cmath>

#include "common.cuh"
#include "value_conversion.h"

namespace csm {

constexpr int kMaxCells = 30000;            // per axis: the handle's size guard
constexpr int kRtTileBytes = 100 * 1024;    // the real-time matcher's staged TMA box (2 CTAs
                                            // in an H100 SM's 228 KB)

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

// The box of a device reduction {min x, min y, max x, max y} (empty: min > max).
inline KnownBox2 BoxFrom(const int* b) {
  KnownBox2 k;
  if (b[0] <= b[2]) {
    k.lo[0] = b[0];
    k.lo[1] = b[1];
    k.hi[0] = b[2];
    k.hi[1] = b[3];
  }
  return k;
}

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

// A handle made from host cells (row pitch nx; wcells and truncation > 0 for a TSDF2D), as
// csm_rt_grid2d_create does it.
csm_status RtGridCreate(const uint16_t* cells, const uint16_t* wcells, float truncation,
                        float max_weight, int32_t nx, int32_t ny, double resolution, double max_x,
                        double max_y, int32_t device, csm_rt_grid2d** out);

// Brings grid->known up to date (one stream synchronisation when it is stale).  Caller holds
// ctx->mu.
csm_status RefreshKnownBox(csm_rt_grid2d* grid);

// Uploads `cells` (and `wcells` if not null; host row pitch nx) into the handle's arrays on
// stream s.  The caller marks the known-cells box stale when the cells change.
csm_status UploadCells(csm_rt_grid2d* g, const uint16_t* cells, const uint16_t* wcells,
                       cudaStream_t s);

struct Limits2 {   // MapLimits (2d/map_limits.h)
  double resolution, max_x, max_y;
  int nx, ny;
  // GetCellIndex (map_limits.h:69-76): the float point enters double arithmetic.  One
  // definition for host and device: both llround round half away from zero.
  __host__ __device__ void CellIndex(float px, float py, long long* ix, long long* iy) const {
    *ix = llround((max_y - static_cast<double>(py)) / resolution - 0.5);
    *iy = llround((max_x - static_cast<double>(px)) / resolution - 0.5);
  }
  __host__ __device__ bool Contains(long long ix, long long iy) const {
    return ix >= 0 && iy >= 0 && ix < nx && iy < ny;
  }
};

// A handle's cell arrays: tsd / probability cells and, for a TSDF2D, weight cells.
struct CellArrays2 {
  uint16_t* cells = nullptr;
  uint16_t* wcells = nullptr;
  int pitch = 0;
};

// Reserves the context's staging of `n` known-cells boxes, so that the transactions of one
// insert (box_slot 0 .. n - 1) can start their box reductions without moving the buffers under
// one another's pending copies.  Caller holds ctx->mu.
csm_status ReserveKnownBoxSlots(Ctx* ctx, int n);

// The part of one 2D insert that changes the handle (caller holds ctx->mu):
//   1. Grow: Grid2D::GrowAsNeeded on the limits, from the bounding box of the insert's points;
//   2. Begin: starts the known-box reduction of a handle made from cells (before its cells
//      move) into staging slot `box_slot`, and allocates the grown arrays, on the handle's
//      stream;
//   3. the caller's kernels write `arrays` at limits L; the caller records ctx->ev1 (ctx->ev0
//      before its first device work) and synchronises the stream;
//   4. Commit: installs grown arrays, moves the old known box by the growth and extends it by
//      what the insert touched, and fills stats (may be NULL).
// Grown arrays not committed are freed when the transaction ends: the handle keeps its size
// and its cells.  Several transactions make one when the caller grows all of them before it
// begins any, gives each its own box slot (ReserveKnownBoxSlots first), and commits all of
// them or none.
class GridInsert2 {
 public:
  explicit GridInsert2(csm_rt_grid2d* grid, int box_slot = 0);
  ~GridInsert2();
  GridInsert2(const GridInsert2&) = delete;
  GridInsert2& operator=(const GridInsert2&) = delete;
  // false if the grid would grow past kMaxCells.
  bool Grow(float lo_x, float lo_y, float hi_x, float hi_y);
  csm_status Begin();
  csm_status Commit(const KnownBox2& touched, csm_stats* stats);

  Limits2 L;            // the grown limits
  CellArrays2 arrays;   // what the insert writes: the handle's own arrays, or grown copies

 private:
  csm_rt_grid2d* grid_;
  int box_slot_;
  int grow_x_ = 0, grow_y_ = 0;   // cell offset of the old cells in the grown arrays
  bool grown_ = false;            // `arrays` were allocated by Begin
  bool box_stale_ = false;
};

}  // namespace csm

#endif  // CSM_RTGRID_CUH_
