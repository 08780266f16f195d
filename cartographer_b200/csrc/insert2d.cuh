// What the two 2D inserters share (insert2d.cu for ProbabilityGrid handles, insert_tsdf2d.cu
// for TSDF2D handles): MapLimits and Grid2D::GrowLimits on the host, the handle's re-allocation
// for grown limits, the known-cells box reduction, and RayToPixelMask as one device walk.
#ifndef CSM_INSERT2D_CUH_
#define CSM_INSERT2D_CUH_

#include <algorithm>
#include <climits>
#include <cmath>
#include <memory>

#include "rtgrid.cuh"

namespace csm {

constexpr int kSubpixelScale = 1000;   // probability_grid_range_data_inserter_2d.cc:33,
                                       // tsdf_range_data_inserter_2d.cc:27
constexpr int kMaxCells = 30000;       // the handle's size guard (rt2d.cu GridCreate)

struct Limits2 {   // MapLimits (2d/map_limits.h)
  double resolution, max_x, max_y;
  int nx, ny;
  // GetCellIndex (map_limits.h:69-76): the float point enters double arithmetic
  void CellIndex(float px, float py, long long* ix, long long* iy) const {
    *ix = std::llround((max_y - static_cast<double>(py)) / resolution - 0.5);
    *iy = std::llround((max_x - static_cast<double>(px)) / resolution - 0.5);
  }
  bool Contains(long long ix, long long iy) const {
    return ix >= 0 && iy >= 0 && ix < nx && iy < ny;
  }
};

// Grid2D::GrowLimits(point) on the limits alone; the cell offset of the old cells in the new
// array accumulates into (ox, oy).  false if the grid would pass the size guard.
inline bool GrowLimits(float px, float py, Limits2* L, int* ox, int* oy) {
  for (;;) {
    long long ix, iy;
    L->CellIndex(px, py, &ix, &iy);
    if (L->Contains(ix, iy)) return true;
    if (2LL * L->nx >= kMaxCells || 2LL * L->ny >= kMaxCells) return false;
    const int x_offset = L->nx / 2, y_offset = L->ny / 2;
    L->max_x = L->max_x + L->resolution * static_cast<double>(y_offset);
    L->max_y = L->max_y + L->resolution * static_cast<double>(x_offset);
    L->nx *= 2;
    L->ny *= 2;
    *ox += x_offset;
    *oy += y_offset;
  }
}

// A zero-filled handle of the given limits (caller holds ctx->mu): a ProbabilityGrid or, with
// truncation > 0, a TSDF2D (tsd and weight 0) with that converter.  Its known-cells box is empty.
csm_status NewGrid(Ctx* ctx, int nx, int ny, double resolution, double max_x, double max_y,
                   std::unique_ptr<csm_rt_grid2d>* out, float truncation = 0.f,
                   float max_weight = 0.f);

// A handle's cell arrays for grown limits: the old block at cell offset (ox, oy), unknown (0)
// around it, in both arrays of a TSDF2D.
struct CellArrays2 {
  uint16_t* cells = nullptr;
  uint16_t* wcells = nullptr;
  int pitch = 0;
};

// Allocates and fills the grown arrays of `grid` for limits L on stream s (caller holds
// ctx->mu).  The handle itself is not changed.
csm_status GrowCellArrays2(const csm_rt_grid2d* grid, const Limits2& L, int ox, int oy,
                           cudaStream_t s, CellArrays2* out);

// Installs `arrays` and the limits L into the handle and re-encodes its TMA descriptor;
// `arrays` gets the old arrays back, to be freed once the stream is done with them.
csm_status InstallCellArrays2(csm_rt_grid2d* grid, const Limits2& L, CellArrays2* arrays);

// Launches the known-box reduction of the handle's (tsd) cells into box4 (device, 4 ints:
// min x, min y, max x, max y) on its stream.
csm_status LaunchKnownBox(csm_rt_grid2d* grid, int* box4);
KnownBox2 BoxFrom(const int* box4);

// RayToPixelMask(begin, end, kSubpixelScale) (internal/2d/ray_to_pixel_mask.cc:34-156): calls
// emit(x, y) for every pixel of the mask, in the reference's order, each once.  Same integer
// walk as the reference, int64 where it is int64.
template <typename Emit>
__device__ __forceinline__ void RayToPixelMask2(int2 b, int2 e, Emit&& emit) {
  const int s = kSubpixelScale;
  int last_x = INT_MIN, last_y = INT_MIN;
  auto push = [&](int x, int y) {
    if (x == last_x && y == last_y) return;
    last_x = x;
    last_y = y;
    emit(x, y);
  };
  if (b.x > e.x) {   // ordered by x (:39-41)
    const int2 t = b;
    b = e;
    e = t;
  }
  if (b.x / s == e.x / s) {   // vertical line in full pixels (:49-60)
    const int x = b.x / s;
    const int end_y = max(b.y, e.y) / s;
    for (int y = min(b.y, e.y) / s; y <= end_y; ++y) push(x, y);
    return;
  }
  const long long dx = e.x - b.x;
  const long long dy = e.y - b.y;
  const long long denominator = 2LL * s * dx;
  int cx = b.x / s, cy = b.y / s;
  push(cx, cy);
  long long sub_y = (2LL * (b.y % s) + 1) * dx;
  const int first_pixel = 2 * s - 2 * (b.x % s) - 1;
  const int last_pixel = 2 * (e.x % s) + 1;
  const int end_x = max(b.x, e.x) / s;
  sub_y += dy * first_pixel;
  if (dy > 0) {
    while (true) {
      push(cx, cy);
      while (sub_y > denominator) {
        sub_y -= denominator;
        ++cy;
        push(cx, cy);
      }
      ++cx;
      if (sub_y == denominator) {   // exact corner: diagonal step
        sub_y -= denominator;
        ++cy;
      }
      if (cx == end_x) break;
      sub_y += dy * 2 * s;
    }
    sub_y += dy * last_pixel;
    push(cx, cy);
    while (sub_y > denominator) {
      sub_y -= denominator;
      ++cy;
      push(cx, cy);
    }
  } else {
    while (true) {
      push(cx, cy);
      while (sub_y < 0) {
        sub_y += denominator;
        --cy;
        push(cx, cy);
      }
      ++cx;
      if (sub_y == 0) {
        sub_y += denominator;
        --cy;
      }
      if (cx == end_x) break;
      sub_y += dy * 2 * s;
    }
    sub_y += dy * last_pixel;
    push(cx, cy);
    while (sub_y < 0) {
      sub_y += denominator;
      --cy;
      push(cx, cy);
    }
  }
}

// Blocks of 256 threads for `work` items, at least one and at most `cap`.
inline unsigned Blocks(long long work, long long cap = 1 << 16) {
  return static_cast<unsigned>(std::max(1LL, std::min(cap, (work + 255) / 256)));
}

}  // namespace csm

#endif  // CSM_INSERT2D_CUH_
