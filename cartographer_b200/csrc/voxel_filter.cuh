// The device core of VoxelFilter and AdaptiveVoxelFilter (voxel_filter.cu), for callers whose
// clouds already live on the device: it enqueues the whole batch on a context's stream and
// leaves its outputs there, with no stream synchronisation.
#ifndef CSM_VOXEL_FILTER_CUH_
#define CSM_VOXEL_FILTER_CUH_

#include <vector>

#include "common.cuh"

namespace csm {

struct VoxelFilterDeviceOut {
  const int* kept_indices;    // the clouds' kept indices one after another, each into its cloud
  const int* num_kept;        // per cloud
  const unsigned char* kept;  // per input point: kept (over the whole batch)
  const void* states;         // per cloud, VoxelFilterStateBytes() each: VoxelFilterCheckStates
};

// Enqueues the batch of clouds off (offsets, off.back() points) on ctx's stream in workspace
// `workspace` (distinct names for batches enqueued back to back).  The points come from the
// host clouds xyz, or from d_xyz on the device when it is not null.  options == nullptr runs
// VoxelFilter at resolution[c]; otherwise AdaptiveVoxelFilter, restricted to the points that
// d_pre_active flags when it is not null.  `start` (may be null) is recorded before the first
// device operation.  Arguments are checked by the caller.
csm_status VoxelFilterEnqueue(Ctx* ctx, const char* workspace, const float* const* xyz,
                              const float* d_xyz, const std::vector<int>& off,
                              const float* resolution,
                              const csm_adaptive_voxel_filter_options* options,
                              const unsigned char* d_pre_active, cudaEvent_t start,
                              VoxelFilterDeviceOut* result);
size_t VoxelFilterStateBytes();
// CSM_E_INTERNAL if a cloud's adaptive search did not settle (host copies of the states).
csm_status VoxelFilterCheckStates(const void* states, int num_clouds);

}  // namespace csm

#endif  // CSM_VOXEL_FILTER_CUH_
