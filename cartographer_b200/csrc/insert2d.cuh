// What the two 2D inserters share (insert2d.cu for ProbabilityGrid handles, insert_tsdf2d.cu
// for TSDF2D handles) beyond the handle itself (rtgrid.cuh): the subpixel scale, RayToPixelMask
// as one device walk, and launch sizes.
#ifndef CSM_INSERT2D_CUH_
#define CSM_INSERT2D_CUH_

#include <algorithm>
#include <climits>

#include "rtgrid.cuh"

namespace csm {

constexpr int kSubpixelScale = 1000;   // probability_grid_range_data_inserter_2d.cc:33,
                                       // tsdf_range_data_inserter_2d.cc:27

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

}  // namespace csm

#endif  // CSM_INSERT2D_CUH_
