// The 2D stages' device cores for data that already lives on the device (local_slam2d.cu): the
// refinement of refine2d.cu and the submap insert of insert2d.cu, without the host copies and
// checks of their public entry points.
#ifndef CSM_RESIDENT2D_CUH_
#define CSM_RESIDENT2D_CUH_

#include "rtgrid.cuh"

namespace csm {

// CeresScanMatcher2D::Match of the cloud d_xyz (n x {x, y, z}, on ctx's device, complete before
// the call) on ctx's stream; the caller holds ctx->mu and has checked the pose and the target.
// One stream synchronisation; stats (may be NULL) gets host_syncs and device_ms.
csm_status CeresMatch2DResident(Ctx* ctx, const csm_rt_grid2d* grid, const float* d_xyz, int n,
                                const double target[2], const double init[3],
                                const csm_ceres_options2d* options, csm_ceres_result2d* result,
                                csm_stats* stats);

// The points of an insert_submaps call already on the device: d_pts holds the returns, then the
// misses, as {x, y} (complete before the call); lo / hi are their bounding box with the origin,
// l1 the sum of the rays' L1 lengths, and every point is finite.
struct InsertPoints2 {
  const float2* d_pts;
  float lo_x, lo_y, hi_x, hi_y;
  double l1;
};

// csm_range_inserter2d_insert_submaps on resident points; locks the inserter's context itself.
csm_status InsertSubmapsResident(const csm_range_inserter2d* inserter, const float origin[3],
                                 const InsertPoints2& points, int32_t num_returns,
                                 int32_t num_misses, csm_rt_grid2d* const* grids,
                                 int32_t num_grids, csm_stats* stats);

}  // namespace csm

#endif  // CSM_RESIDENT2D_CUH_
