// LocalTrajectoryBuilder2D (mapping/internal/2d/local_trajectory_builder_2d.cc:65-300) on the
// device, from synchronized range data to the submap insert, with the range data kept in device
// memory between the stages.  The host keeps what needs double precision and libm: the
// extrapolator's poses, the gravity alignment, Embed3D of the 2D pose and the motion filter.
//
//   accumulate  AddRangeData's per-point loop (:163-186): every hit and its origin through its
//               Rigid3f pose, the range test, and the returns and misses appended to the
//               accumulation buffers in input order (one inclusive scan of {return, miss} flags
//               and a scatter).  No stream synchronisation.
//   match       TransformToGravityAlignedFrameAndFilter (:51-63) and AddAccumulatedRangeData up
//               to the pose (:211-244): TransformRangeData and CropRangeData (the same scan and
//               scatter), then VoxelFilter of the returns and the misses and AdaptiveVoxelFilter
//               of the filtered returns (voxel_filter.cu's core on the device clouds: the
//               adaptive filter runs over the cropped returns restricted to those the voxel
//               filter kept, which is the filtered cloud in order), then ScanMatch (:65-102):
//               the real-time matcher (rt2d.cu) and CeresScanMatcher2D (refine2d.cu's core on
//               the device cloud).
//   insert      TransformRangeData of the kept range data into the local frame (:237-240), its
//               bounding box and ray lengths, and ActiveSubmaps2D's inserts (insert2d.cu's core
//               on the device points).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "point_batch.cuh"
#include "resident2d.cuh"
#include "rigid3f.h"
#include "voxel_filter.cuh"

namespace csm {
namespace {

constexpr int kThreads = 256;

struct Int2Sum {
  __device__ int2 operator()(const int2& a, const int2& b) const {
    return make_int2(a.x + b.x, a.y + b.y);
  }
};

__device__ inline Rigid3f LoadRigid(const float* p) {
  return Rigid3f{Vec3f{p[0], p[1], p[2]}, Quatf{p[3], p[4], p[5], p[6]}};
}

// AddRangeData's loop body (:165-185) for hit i: its point in the local frame and whether it is
// a return (x) or a miss (y).
__global__ void k_ls_classify(const float* __restrict__ hits, int n,
                              const float* __restrict__ origins,
                              const int* __restrict__ origin_index,
                              const float* __restrict__ poses, const int* __restrict__ pose_index,
                              float min_range, float max_range, float missing_data_ray_length,
                              float3* __restrict__ pts, int2* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Rigid3f pose = LoadRigid(poses + 7 * pose_index[i]);
  const float* o = origins + 3 * origin_index[i];
  const Vec3f origin = Rigid3Apply(pose, Vec3f{o[0], o[1], o[2]});
  const Vec3f hit = Rigid3Apply(pose, Vec3f{hits[3 * i], hits[3 * i + 1], hits[3 * i + 2]});
  const float dx = FSub(hit.x, origin.x), dy = FSub(hit.y, origin.y), dz = FSub(hit.z, origin.z);
  const float range = FSqrt(FAdd(FAdd(FMul(dx, dx), FMul(dy, dy)), FMul(dz, dz)));
  int2 f = make_int2(0, 0);
  float3 p = make_float3(hit.x, hit.y, hit.z);
  if (range >= min_range) {
    if (range <= max_range) {
      f.x = 1;
    } else {
      const float s = FDiv(missing_data_ray_length, range);
      p = make_float3(FAdd(origin.x, FMul(s, dx)), FAdd(origin.y, FMul(s, dy)),
                      FAdd(origin.z, FMul(s, dz)));
      f.y = 1;
    }
  }
  pts[i] = p;
  flags[i] = f;
}

// TransformRangeData + CropRangeData (range_data.cc:25-39) of the accumulated range data: entry
// i < bound is return i (acc[i]), entry bound + k miss k (acc[cap + k]); entries past the
// accumulated counts are not kept.
__global__ void k_ls_gravity_crop(const float3* __restrict__ acc, long long cap, long long bound,
                                  const int* __restrict__ counts, Rigid3f T, float min_z,
                                  float max_z, float3* __restrict__ pts, int2* __restrict__ flags) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= 2 * bound) return;
  const bool is_return = i < bound;
  const long long k = is_return ? i : i - bound;
  int2 f = make_int2(0, 0);
  if (k < counts[is_return ? 0 : 1]) {
    const float3 a = acc[is_return ? k : cap + k];
    const Vec3f p = Rigid3Apply(T, Vec3f{a.x, a.y, a.z});
    pts[i] = make_float3(p.x, p.y, p.z);
    const int keep = min_z <= p.z && p.z <= max_z;
    if (is_return) f.x = keep; else f.y = keep;
  }
  flags[i] = f;
}

// The stable compaction: entry i goes to returns[base.x + rank] or misses[base.y + rank] by its
// flag, `incl` the inclusive sums of the flags.
__global__ void k_ls_scatter(const float3* __restrict__ pts, const int2* __restrict__ flags,
                             const int2* __restrict__ incl, long long n,
                             const int* __restrict__ base, float3* __restrict__ returns,
                             float3* __restrict__ misses) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int2 f = flags[i];
  if (f.x) returns[base[0] + incl[i].x - 1] = pts[i];
  if (f.y) misses[base[1] + incl[i].y - 1] = pts[i];
}

__global__ void k_ls_bump(int* counts, const int2* __restrict__ incl, long long n) {
  if (threadIdx.x == 0 && n > 0) {
    counts[0] += incl[n - 1].x;
    counts[1] += incl[n - 1].y;
  }
}

// The voxel-filtered range data (clouds 0 and 1 of the first batch, cloud 1 at n_r) and the
// adaptively filtered returns, gathered from the cropped points.
__global__ void k_ls_gather(const float3* __restrict__ cropped, int n_r, int n,
                            const int* __restrict__ vf_idx, const int* __restrict__ vf_num,
                            const int* __restrict__ avf_idx, const int* __restrict__ avf_num,
                            float3* __restrict__ vf, float3* __restrict__ filtered) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  if (j < vf_num[0] + vf_num[1]) vf[j] = cropped[vf_idx[j] + (j < vf_num[0] ? 0 : n_r)];
  if (j < avf_num[0]) filtered[j] = cropped[avf_idx[j]];
}

// Ordered-int keys of floats, so that integer min / max order them as floats.
__device__ inline int FloatKey(float f) {
  const int b = __float_as_int(f);
  return b >= 0 ? b : b ^ 0x7fffffff;
}
inline float KeyFloat(int k) {
  const int b = k >= 0 ? k : k ^ 0x7fffffff;
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}

// range_data_in_local (:237-240): the kept range data through Embed3D(pose_estimate_2d), its
// {x, y} for the inserter, every point's ray L1 length (in double, as the inserter's host pass
// sums them) and the bounding box (box: min x, min y, max x, max y as FloatKey, then a
// non-finite flag).
__global__ void k_ls_to_local(const float3* __restrict__ vf, int n, Rigid3f T, float ox, float oy,
                              float3* __restrict__ local, float2* __restrict__ local2,
                              double* __restrict__ l1, int* box) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool in = false;
  float x = 0.f, y = 0.f;
  if (i < n) {
    const float3 a = vf[i];
    const Vec3f p = Rigid3Apply(T, Vec3f{a.x, a.y, a.z});
    local[i] = make_float3(p.x, p.y, p.z);
    local2[i] = make_float2(p.x, p.y);
    l1[i] = fabs(static_cast<double>(p.x) - ox) + fabs(static_cast<double>(p.y) - oy);
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) atomicOr(box + 4, 1);
    in = true;
    x = p.x;
    y = p.y;
  }
  const int lo_x = __reduce_min_sync(0xffffffffu, in ? FloatKey(x) : INT_MAX);
  const int lo_y = __reduce_min_sync(0xffffffffu, in ? FloatKey(y) : INT_MAX);
  const int hi_x = __reduce_max_sync(0xffffffffu, in ? FloatKey(x) : INT_MIN);
  const int hi_y = __reduce_max_sync(0xffffffffu, in ? FloatKey(y) : INT_MIN);
  if ((threadIdx.x & 31) == 0 && lo_x <= hi_x) {
    atomicMin(box + 0, lo_x);
    atomicMin(box + 1, lo_y);
    atomicMax(box + 2, hi_x);
    atomicMax(box + 3, hi_y);
  }
}

Rigid3f HostRigid(const float* p) {
  return Rigid3f{Vec3f{p[0], p[1], p[2]}, Quatf{p[3], p[4], p[5], p[6]}};
}

// Whether `bytes` more device memory can be had.
csm_status CheckFits(size_t bytes) {
  size_t free_b = 0, total_b = 0;
  CSM_CUDA(cudaMemGetInfo(&free_b, &total_b));
  if (bytes > free_b) {
    SetError("local SLAM buffers: %zu bytes do not fit the device (%zu free)", bytes, free_b);
    return CSM_E_CAPACITY;
  }
  return CSM_OK;
}

}  // namespace
}  // namespace csm

using namespace csm;

struct csm_local_slam2d {
  Ctx* ctx = nullptr;
  csm_local_slam_options2d o;
  csm_range_inserter2d* inserter = nullptr;
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;
  // accumulation: returns at [0, acc_cap), misses at [acc_cap, 2 acc_cap); counts[0..1] on the
  // device; acc_bound bounds both counts (the hits accumulated since the last match)
  float3* acc = nullptr;
  size_t acc_bytes = 0;
  long long acc_cap = 0, acc_bound = 0;
  int num_accumulated = 0;
  int* d_counts = nullptr;   // accumulated returns, misses; cropped returns, misses
  // the current scan (valid after a match that was not dropped)
  DevBuf work, scan, vf, filtered, local, local2, l1, scratch;
  int n_crop_r = 0, n_crop_m = 0, n_vf_r = 0, n_vf_m = 0, n_filtered = 0;
  float ga_origin[3] = {0, 0, 0}, local_origin[3] = {0, 0, 0};
  bool cropped_ready = false, scan_ready = false, local_ready = false;
  PinnedBuf down;
  std::vector<float> h_filtered;
  // accumulate's upload staging: two pinned slots, each reused once its copy has run
  PinnedBuf stage[2];
  cudaEvent_t stage_ev[2] = {nullptr, nullptr};
  int stage_next = 0;
  ~csm_local_slam2d() {
    if (ctx) {
      cudaSetDevice(ctx->device);
      cudaStreamSynchronize(ctx->stream);
    }
    cudaFree(acc);
    cudaFree(d_counts);
    for (PinnedBuf* b : {&down, &stage[0], &stage[1]})
      if (b->p) cudaFreeHost(b->p);
    for (DevBuf* b : {&work, &scan, &vf, &filtered, &local, &local2, &l1, &scratch})
      if (b->p) cudaFree(b->p);
    for (cudaEvent_t e : {ev_a, ev_b, stage_ev[0], stage_ev[1]})
      if (e) cudaEventDestroy(e);
    if (inserter) csm_range_inserter2d_destroy(inserter);
  }
};

namespace {

csm_status CheckOptions(const csm_local_slam_options2d* o) {
  CSM_REQUIRE(std::isfinite(o->min_range) && std::isfinite(o->max_range) &&
                  std::isfinite(o->min_z) && std::isfinite(o->max_z) &&
                  std::isfinite(o->missing_data_ray_length),
              "non-finite range or z option");
  CSM_REQUIRE(std::isfinite(o->voxel_filter_size) && o->voxel_filter_size > 0.f,
              "voxel_filter_size");
  CSM_REQUIRE(o->num_accumulated_range_data >= 1, "num_accumulated_range_data");
  const csm_adaptive_voxel_filter_options& a = o->adaptive_voxel_filter;
  CSM_REQUIRE(std::isfinite(a.max_length) && a.max_length > 0.f, "max_length");
  CSM_REQUIRE(!std::isnan(a.min_num_points) && !std::isnan(a.max_range),
              "min_num_points / max_range");
  CSM_REQUIRE(std::isfinite(o->linear_search_window) && o->linear_search_window >= 0. &&
                  std::isfinite(o->angular_search_window) && o->angular_search_window >= 0. &&
                  std::isfinite(o->translation_delta_cost_weight) &&
                  std::isfinite(o->rotation_delta_cost_weight),
              "real-time matcher options");
  const csm_ceres_options2d& c = o->ceres;
  CSM_REQUIRE(c.occupied_space_weight > 0. && c.translation_weight > 0. &&
                  c.rotation_weight > 0. && std::isfinite(c.occupied_space_weight) &&
                  std::isfinite(c.translation_weight) && std::isfinite(c.rotation_weight),
              "Ceres weights");
  CSM_REQUIRE(c.max_num_iterations > 0, "max_num_iterations");
  return CSM_OK;
}

// Enqueues the inclusive scan of flags[0 .. n) and the scatter of pts into returns / misses at
// the device counts base[0..1], then adds the totals to them.
csm_status Compact(csm_local_slam2d* h, const float3* pts, const int2* flags, int2* incl,
                   long long n, int* base, float3* returns, float3* misses) {
  if (n == 0) return CSM_OK;
  cudaStream_t s = h->ctx->stream;
  size_t bytes = 0;
  CSM_CUDA(cub::DeviceScan::InclusiveScan(nullptr, bytes, flags, incl, Int2Sum(), n, s));
  CSM_TRY(h->scratch.Reserve(bytes));
  CSM_CUDA(cub::DeviceScan::InclusiveScan(h->scratch.p, bytes, flags, incl, Int2Sum(), n, s));
  k_ls_scatter<<<DivUp(n, kThreads), kThreads, 0, s>>>(pts, flags, incl, n, base, returns, misses);
  CSM_LAUNCH_CHECK();
  k_ls_bump<<<1, 32, 0, s>>>(base, incl, n);
  CSM_LAUNCH_CHECK();
  return CSM_OK;
}

}  // namespace

extern "C" {

csm_status csm_local_slam2d_create(const csm_local_slam_options2d* options, int32_t device,
                                   csm_local_slam2d** out) {
  CSM_REQUIRE(options && out, "null pointer");
  CSM_TRY(CheckOptions(options));
  std::unique_ptr<csm_local_slam2d> h(new csm_local_slam2d);
  CSM_TRY(csm_range_inserter2d_create(&options->inserter, device, &h->inserter));
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  h->ctx = ctx;
  h->o = *options;
  for (DevBuf* b : {&h->work, &h->scan, &h->vf, &h->filtered, &h->local, &h->local2, &h->l1,
                    &h->scratch})
    b->stream = ctx->stream;
  CSM_CUDA(cudaMalloc(&h->d_counts, 4 * sizeof(int)));
  CSM_CUDA(cudaMemsetAsync(h->d_counts, 0, 4 * sizeof(int), ctx->stream));
  for (cudaEvent_t* e : {&h->ev_a, &h->ev_b}) CSM_CUDA(cudaEventCreate(e));
  for (cudaEvent_t& e : h->stage_ev) CSM_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  *out = h.release();
  return CSM_OK;
}

csm_status csm_local_slam2d_destroy(csm_local_slam2d* handle) {
  if (!handle) return CSM_OK;
  std::unique_lock<std::mutex> lock(handle->ctx->mu);
  cudaSetDevice(handle->ctx->device);
  cudaStreamSynchronize(handle->ctx->stream);
  csm_range_inserter2d* ins = handle->inserter;
  handle->inserter = nullptr;
  delete handle;
  lock.unlock();
  return csm_range_inserter2d_destroy(ins);
}

csm_status csm_local_slam2d_accumulate(csm_local_slam2d* h, const float* hits, int32_t num_hits,
                                       const float* origins, int32_t num_origins,
                                       const int32_t* origin_index, const float* poses,
                                       int32_t num_poses, const int32_t* pose_index,
                                       csm_stats* stats) {
  CSM_REQUIRE(h, "null handle");
  CSM_REQUIRE(num_hits >= 1 && num_origins >= 1 && num_poses >= 1, "empty input");
  CSM_REQUIRE(hits && origins && origin_index && poses && pose_index, "null pointer");
  CSM_REQUIRE(Finite(hits, 3 * static_cast<size_t>(num_hits)) &&
                  Finite(origins, 3 * static_cast<size_t>(num_origins)),
              "non-finite point");
  CSM_REQUIRE(Finite(poses, 7 * static_cast<size_t>(num_poses)), "non-finite pose");
  for (int i = 0; i < num_hits; ++i) {
    CSM_REQUIRE(origin_index[i] >= 0 && origin_index[i] < num_origins, "origin_index");
    CSM_REQUIRE(pose_index[i] >= 0 && pose_index[i] < num_poses, "pose_index");
  }
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const bool fresh = h->num_accumulated == 0;
  const long long bound = (fresh ? 0 : h->acc_bound) + num_hits;
  CSM_REQUIRE(bound < (1LL << 30), "more than 2^30 accumulated points");
  const int n = num_hits;
  const size_t o_org = Align(sizeof(float) * 3 * n);
  const size_t o_oi = o_org + Align(sizeof(float) * 3 * num_origins);
  const size_t o_pose = o_oi + Align(sizeof(int) * n);
  const size_t o_pi = o_pose + Align(sizeof(float) * 7 * num_poses);
  const size_t up_bytes = o_pi + Align(sizeof(int) * n);
  const size_t o_pts = up_bytes;
  const size_t o_flags = o_pts + Align(sizeof(float3) * n);
  const size_t o_incl = o_flags + Align(sizeof(int2) * n);
  const size_t work_bytes = o_incl + Align(sizeof(int2) * n);
  // every allocation is checked and made before anything is enqueued
  const bool grow = bound > h->acc_cap;
  const long long new_cap = grow ? std::max(bound, 2 * h->acc_cap) : h->acc_cap;
  const size_t need = (grow ? sizeof(float3) * 2 * new_cap : 0) +
                      (work_bytes > h->work.cap ? work_bytes + work_bytes / 2 + 256 : 0);
  if (need > 0) CSM_TRY(CheckFits(need));
  CSM_TRY(h->work.Reserve(work_bytes));
  // the staging slot, once its previous copy (two calls ago) has run
  const int slot = h->stage_next;
  h->stage_next ^= 1;
  CSM_CUDA(cudaEventSynchronize(h->stage_ev[slot]));
  CSM_TRY(h->stage[slot].Reserve(up_bytes));
  char* hp = h->stage[slot].as<char>();
  std::memcpy(hp, hits, sizeof(float) * 3 * n);
  std::memcpy(hp + o_org, origins, sizeof(float) * 3 * num_origins);
  std::memcpy(hp + o_oi, origin_index, sizeof(int) * n);
  std::memcpy(hp + o_pose, poses, sizeof(float) * 7 * num_poses);
  std::memcpy(hp + o_pi, pose_index, sizeof(int) * n);

  if (fresh) CSM_CUDA(cudaMemsetAsync(h->d_counts, 0, 2 * sizeof(int), s));
  if (grow) {
    // the returns keep their place; the misses move to the new capacity
    float3* q = nullptr;
    CSM_CUDA(cudaMallocAsync(&q, sizeof(float3) * 2 * new_cap, s));
    if (h->acc && !fresh) {
      CSM_CUDA(cudaMemcpyAsync(q, h->acc, sizeof(float3) * h->acc_cap, cudaMemcpyDeviceToDevice, s));
      CSM_CUDA(cudaMemcpyAsync(q + new_cap, h->acc + h->acc_cap, sizeof(float3) * h->acc_cap,
                               cudaMemcpyDeviceToDevice, s));
    }
    if (h->acc) CSM_CUDA(cudaFreeAsync(h->acc, s));
    h->acc = q;
    h->acc_cap = new_cap;
  }
  char* d = h->work.as<char>();
  CSM_CUDA(cudaMemcpyAsync(d, hp, up_bytes, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaEventRecord(h->stage_ev[slot], s));
  float3* pts = reinterpret_cast<float3*>(d + o_pts);
  int2* flags = reinterpret_cast<int2*>(d + o_flags);
  k_ls_classify<<<DivUp(n, kThreads), kThreads, 0, s>>>(
      reinterpret_cast<const float*>(d), n, reinterpret_cast<const float*>(d + o_org),
      reinterpret_cast<const int*>(d + o_oi), reinterpret_cast<const float*>(d + o_pose),
      reinterpret_cast<const int*>(d + o_pi), h->o.min_range, h->o.max_range,
      h->o.missing_data_ray_length, pts, flags);
  CSM_LAUNCH_CHECK();
  CSM_TRY(Compact(h, pts, flags, reinterpret_cast<int2*>(d + o_incl), n, h->d_counts, h->acc,
                  h->acc + h->acc_cap));
  h->acc_bound = bound;
  ++h->num_accumulated;
  h->scan_ready = h->local_ready = false;
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));   // no synchronisation: device_ms is not measured
  }
  return CSM_OK;
}

csm_status csm_local_slam2d_match(csm_local_slam2d* h, const float to_gravity[7],
                                  const float origin[3], const double pose_prediction[3],
                                  const csm_rt_grid2d* grid, csm_local_slam_match2d* result,
                                  csm_stats* stats) {
  CSM_REQUIRE(h && to_gravity && origin && pose_prediction && result, "null pointer");
  CSM_REQUIRE(Finite(to_gravity, 7), "non-finite pose");
  CSM_REQUIRE(Finite(origin, 3), "non-finite point");
  CSM_REQUIRE(Finite(pose_prediction, 3), "non-finite pose");
  CSM_REQUIRE(h->num_accumulated > 0, "no range data accumulated");
  if (grid) {
    CSM_REQUIRE(grid->d_wcells == nullptr, "local SLAM matches against ProbabilityGrid submaps");
    CSM_REQUIRE(grid->ctx == h->ctx, "grid on another device than the builder");
  }
  Ctx* ctx = h->ctx;
  std::unique_lock<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  csm_local_slam_match2d r;
  std::memset(&r, 0, sizeof(r));
  csm_stats st;
  std::memset(&st, 0, sizeof(st));
  const Rigid3f T = HostRigid(to_gravity);
  // the crop covers the points accumulated since the last match, whatever the capacity
  const long long cap = h->acc_cap, bound = h->acc_bound;
  const size_t o_flags = Align(sizeof(float3) * 2 * bound);
  const size_t o_incl = o_flags + Align(sizeof(int2) * 2 * bound);
  const size_t o_ga = o_incl + Align(sizeof(int2) * 2 * bound);
  const size_t work_bytes = o_ga + Align(sizeof(float3) * 2 * bound);
  CSM_TRY(h->work.Reserve(work_bytes));
  CSM_TRY(h->down.Reserve(Align(16 * sizeof(int)) + Align(3 * VoxelFilterStateBytes()) +
                          sizeof(float3) * std::max<long long>(bound, 1)));
  char* d = h->work.as<char>();
  float3* ga = reinterpret_cast<float3*>(d + o_ga);
  int* hc = h->down.as<int>();

  // ---- 1: TransformRangeData + CropRangeData; the cropped counts ----
  CSM_CUDA(cudaEventRecord(h->ev_a, s));
  CSM_CUDA(cudaMemsetAsync(h->d_counts + 2, 0, 2 * sizeof(int), s));
  if (bound > 0) {
    k_ls_gravity_crop<<<DivUp(2 * bound, kThreads), kThreads, 0, s>>>(
        h->acc, cap, bound, h->d_counts, T, h->o.min_z, h->o.max_z, reinterpret_cast<float3*>(d),
        reinterpret_cast<int2*>(d + o_flags));
    CSM_LAUNCH_CHECK();
    CSM_TRY(Compact(h, reinterpret_cast<float3*>(d), reinterpret_cast<int2*>(d + o_flags),
                    reinterpret_cast<int2*>(d + o_incl), 2 * bound, h->d_counts + 2, ga,
                    ga + bound));
  }
  CSM_CUDA(cudaMemcpyAsync(hc, h->d_counts + 2, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaEventRecord(h->ev_b, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, h->ev_a, h->ev_b);
  st.device_ms += ms;
  st.host_syncs = 1;
  // the call ends the accumulation (num_accumulated_ = 0, :191) whatever it finds
  h->num_accumulated = 0;
  h->cropped_ready = h->scan_ready = h->local_ready = false;
  const int n_r = hc[0], n_m = hc[1];
  h->n_crop_r = n_r;
  h->n_crop_m = n_m;
  h->n_vf_r = h->n_vf_m = h->n_filtered = 0;
  h->h_filtered.clear();
  const Vec3f go = Rigid3Apply(T, Vec3f{origin[0], origin[1], origin[2]});
  h->ga_origin[0] = go.x;
  h->ga_origin[1] = go.y;
  h->ga_origin[2] = go.z;
  auto finish = [&]() {
    *result = r;
    if (stats) *stats = st;
    return CSM_OK;
  };
  // ---- 2: VoxelFilter of both clouds, AdaptiveVoxelFilter of the filtered returns ----
  const int n = n_r + n_m;
  CSM_TRY(h->scan.Reserve(sizeof(float3) * n));
  CSM_TRY(h->vf.Reserve(sizeof(float3) * n));
  CSM_TRY(h->filtered.Reserve(sizeof(float3) * n_r));
  float3* cropped = h->scan.as<float3>();
  const size_t o_st = Align(16 * sizeof(int));
  const size_t o_pts = o_st + Align(3 * VoxelFilterStateBytes());
  CSM_CUDA(cudaEventRecord(h->ev_a, s));
  CSM_CUDA(cudaMemcpyAsync(cropped, ga, sizeof(float3) * n_r, cudaMemcpyDeviceToDevice, s));
  if (n_m > 0)
    CSM_CUDA(cudaMemcpyAsync(cropped + n_r, ga + bound, sizeof(float3) * n_m,
                             cudaMemcpyDeviceToDevice, s));
  h->cropped_ready = true;   // a dropped scan's cropped misses stay readable too
  if (n_r == 0) {   // :217-220
    r.status = CSM_LOCAL_SLAM_DROPPED_EMPTY_RETURNS;
    return finish();
  }
  const float vs[2] = {h->o.voxel_filter_size, h->o.voxel_filter_size};
  VoxelFilterDeviceOut vf_out, avf_out;
  CSM_TRY(VoxelFilterEnqueue(ctx, "local_slam_vf", nullptr, reinterpret_cast<const float*>(cropped),
                             {0, n_r, n}, vs, nullptr, nullptr, nullptr, &vf_out));
  CSM_TRY(VoxelFilterEnqueue(ctx, "local_slam_avf", nullptr,
                             reinterpret_cast<const float*>(cropped), {0, n_r}, nullptr,
                             &h->o.adaptive_voxel_filter, vf_out.kept, nullptr, &avf_out));
  k_ls_gather<<<DivUp(n, kThreads), kThreads, 0, s>>>(
      cropped, n_r, n, vf_out.kept_indices, vf_out.num_kept, avf_out.kept_indices,
      avf_out.num_kept, h->vf.as<float3>(), h->filtered.as<float3>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(hc + 2, vf_out.num_kept, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(hc + 4, avf_out.num_kept, sizeof(int), cudaMemcpyDeviceToHost, s));
  char* hd = h->down.as<char>();
  CSM_CUDA(cudaMemcpyAsync(hd + o_st, avf_out.states, VoxelFilterStateBytes(),
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(hd + o_pts, h->filtered.p, sizeof(float3) * n_r,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaEventRecord(h->ev_b, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  cudaEventElapsedTime(&ms, h->ev_a, h->ev_b);
  st.device_ms += ms;
  st.host_syncs += 1;
  CSM_TRY(VoxelFilterCheckStates(hd + o_st, 1));
  h->n_vf_r = hc[2];
  h->n_vf_m = hc[3];
  h->n_filtered = hc[4];
  r.num_filtered = h->n_filtered;
  r.num_returns = h->n_vf_r;
  r.num_misses = h->n_vf_m;
  h->h_filtered.assign(reinterpret_cast<const float*>(hd + o_pts),
                       reinterpret_cast<const float*>(hd + o_pts) + 3 * h->n_filtered);
  if (h->n_filtered == 0) {   // :231-233
    r.status = CSM_LOCAL_SLAM_DROPPED_EMPTY_FILTERED;
    return finish();
  }

  // ---- 3: ScanMatch (:65-102) ----
  r.status = CSM_LOCAL_SLAM_MATCHED;
  double initial[3] = {pose_prediction[0], pose_prediction[1], pose_prediction[2]};
  if (grid == nullptr) {
    std::memcpy(r.pose_estimate, pose_prediction, sizeof(double) * 3);
    h->scan_ready = true;
    return finish();
  }
  r.matched_submap = 1;
  lock.unlock();   // the real-time matcher takes a lane of its own
  if (h->o.use_online_correlative_scan_matching) {
    csm_rt_job2d job;
    std::memset(&job, 0, sizeof(job));
    job.xyz = h->h_filtered.data();
    job.num_points = h->n_filtered;
    std::memcpy(job.initial_pose, pose_prediction, sizeof(double) * 3);
    csm_rt_result2d rt;
    csm_stats rs;
    std::memset(&rs, 0, sizeof(rs));
    CSM_TRY(csm_rt_match2d_batch(grid, &job, 1, h->o.linear_search_window,
                                 h->o.angular_search_window, h->o.translation_delta_cost_weight,
                                 h->o.rotation_delta_cost_weight, &rt, &rs));
    st.device_ms += rs.device_ms;
    st.host_syncs += rs.host_syncs;
    r.rt_score = rt.score;
    std::memcpy(initial, rt.pose_estimate, sizeof(double) * 3);
  }
  lock.lock();
  CSM_CUDA(cudaSetDevice(ctx->device));
  csm_stats cs;
  std::memset(&cs, 0, sizeof(cs));
  CSM_TRY(CeresMatch2DResident(ctx, grid, reinterpret_cast<const float*>(h->filtered.p),
                               h->n_filtered, pose_prediction, initial, &h->o.ceres, &r.ceres,
                               &cs));
  st.device_ms += cs.device_ms;
  st.host_syncs += cs.host_syncs;
  std::memcpy(r.pose_estimate, r.ceres.pose_estimate, sizeof(double) * 3);
  h->scan_ready = true;
  return finish();
}

csm_status csm_local_slam2d_insert(csm_local_slam2d* h, const float pose[7],
                                   csm_rt_grid2d* const* grids, int32_t num_grids,
                                   float local_origin[3], csm_stats* stats) {
  CSM_REQUIRE(h && pose && grids, "null pointer");
  CSM_REQUIRE(Finite(pose, 7), "non-finite pose");
  CSM_REQUIRE(h->scan_ready && !h->local_ready, "no matched scan to insert");
  CSM_REQUIRE(num_grids >= 1 && num_grids <= 65535, "num_grids");
  for (int g = 0; g < num_grids; ++g) {
    CSM_REQUIRE(grids[g] != nullptr, "null grid");
    CSM_REQUIRE(grids[g]->d_wcells == nullptr, "local SLAM inserts into ProbabilityGrid submaps");
    CSM_REQUIRE(grids[g]->ctx == h->ctx, "grid on another device than the builder");
  }
  Ctx* ctx = h->ctx;
  const Rigid3f T = HostRigid(pose);
  const Vec3f lo = Rigid3Apply(T, Vec3f{h->ga_origin[0], h->ga_origin[1], h->ga_origin[2]});
  const float org[3] = {lo.x, lo.y, lo.z};
  CSM_REQUIRE(Finite(org, 3), "non-finite point");
  const int n = h->n_vf_r + h->n_vf_m;
  csm_stats st;
  std::memset(&st, 0, sizeof(st));
  InsertPoints2 pts;
  {
    std::lock_guard<std::mutex> lock(ctx->mu);
    CSM_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    CSM_TRY(h->local.Reserve(sizeof(float3) * n));
    CSM_TRY(h->local2.Reserve(sizeof(float2) * n));
    size_t red_bytes = 0;
    CSM_CUDA(cub::DeviceReduce::Sum(nullptr, red_bytes, static_cast<const double*>(nullptr),
                                    static_cast<double*>(nullptr), n, s));
    const size_t o_sum = Align(sizeof(double) * n);
    const size_t o_box = o_sum + Align(sizeof(double));
    const size_t o_temp = o_box + Align(8 * sizeof(int));
    CSM_TRY(h->l1.Reserve(o_temp + red_bytes));
    CSM_TRY(h->down.Reserve(64));
    char* d = h->l1.as<char>();
    int* d_box = reinterpret_cast<int*>(d + o_box);
    const int init_box[5] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN, 0};
    char* hd = h->down.as<char>();
    std::memcpy(hd + 16, init_box, sizeof(init_box));
    CSM_CUDA(cudaEventRecord(h->ev_a, s));
    CSM_CUDA(cudaMemcpyAsync(d_box, hd + 16, sizeof(init_box), cudaMemcpyHostToDevice, s));
    k_ls_to_local<<<DivUp(n, kThreads), kThreads, 0, s>>>(
        h->vf.as<float3>(), n, T, org[0], org[1], h->local.as<float3>(), h->local2.as<float2>(),
        reinterpret_cast<double*>(d), d_box);
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cub::DeviceReduce::Sum(d + o_temp, red_bytes, reinterpret_cast<const double*>(d),
                                    reinterpret_cast<double*>(d + o_sum), n, s));
    CSM_CUDA(cudaMemcpyAsync(hd, d + o_sum, sizeof(double), cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaMemcpyAsync(hd + 16, d_box, sizeof(init_box), cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaEventRecord(h->ev_b, s));
    CSM_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->ev_a, h->ev_b);
    st.device_ms = ms;
    st.host_syncs = 1;
    const int* box = reinterpret_cast<const int*>(hd + 16);
    CSM_REQUIRE(box[4] == 0, "non-finite point");
    pts.d_pts = h->local2.as<float2>();
    pts.lo_x = std::min(org[0], KeyFloat(box[0]));
    pts.lo_y = std::min(org[1], KeyFloat(box[1]));
    pts.hi_x = std::max(org[0], KeyFloat(box[2]));
    pts.hi_y = std::max(org[1], KeyFloat(box[3]));
    std::memcpy(&pts.l1, hd, sizeof(double));
  }
  csm_stats is;
  std::memset(&is, 0, sizeof(is));
  CSM_TRY(InsertSubmapsResident(h->inserter, org, pts, h->n_vf_r, h->n_vf_m, grids, num_grids,
                                &is));
  st.device_ms += is.device_ms;
  st.host_syncs += is.host_syncs;
  std::memcpy(h->local_origin, org, sizeof(org));
  h->local_ready = true;
  if (local_origin) std::memcpy(local_origin, org, sizeof(org));
  if (stats) *stats = st;
  return CSM_OK;
}

csm_status csm_local_slam2d_read(const csm_local_slam2d* h, int32_t which, float* xyz,
                                 int64_t capacity, int32_t* count) {
  CSM_REQUIRE(h && count, "null pointer");
  CSM_REQUIRE(which >= 0 && which <= CSM_LOCAL_SLAM_LOCAL_MISSES, "which");
  Ctx* ctx = h->ctx;
  if (which == CSM_LOCAL_SLAM_FILTERED) {   // the host copy of the last match
    *count = h->n_filtered;
    CSM_REQUIRE(xyz || h->n_filtered == 0 || capacity == 0, "null xyz");
    if (xyz && capacity >= h->n_filtered) {
      std::memcpy(xyz, h->h_filtered.data(), sizeof(float) * 3 * h->n_filtered);
      return CSM_OK;
    }
    if (xyz) {
      SetError("capacity %lld below %d points", static_cast<long long>(capacity), *count);
      return CSM_E_CAPACITY;
    }
    return CSM_OK;
  }
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const float3* src = nullptr;
  int num = 0;
  switch (which) {
    case CSM_LOCAL_SLAM_ACCUMULATED_RETURNS:
    case CSM_LOCAL_SLAM_ACCUMULATED_MISSES: {
      int c[2] = {0, 0};
      if (h->num_accumulated > 0) {
        CSM_CUDA(cudaMemcpyAsync(c, h->d_counts, sizeof(c), cudaMemcpyDeviceToHost, s));
        CSM_CUDA(cudaStreamSynchronize(s));
      }
      const bool ret = which == CSM_LOCAL_SLAM_ACCUMULATED_RETURNS;
      num = ret ? c[0] : c[1];
      src = ret ? h->acc : h->acc + h->acc_cap;
      break;
    }
    case CSM_LOCAL_SLAM_CROPPED_RETURNS:
      num = h->cropped_ready ? h->n_crop_r : 0;
      src = h->scan.as<float3>();
      break;
    case CSM_LOCAL_SLAM_CROPPED_MISSES:
      num = h->cropped_ready ? h->n_crop_m : 0;
      src = h->scan.as<float3>() + h->n_crop_r;
      break;
    case CSM_LOCAL_SLAM_FILTERED_RETURNS:
      num = h->n_vf_r;
      src = h->vf.as<float3>();
      break;
    case CSM_LOCAL_SLAM_FILTERED_MISSES:
      num = h->n_vf_m;
      src = h->vf.as<float3>() + h->n_vf_r;
      break;
    case CSM_LOCAL_SLAM_LOCAL_RETURNS:
      num = h->local_ready ? h->n_vf_r : 0;
      src = h->local.as<float3>();
      break;
    case CSM_LOCAL_SLAM_LOCAL_MISSES:
      num = h->local_ready ? h->n_vf_m : 0;
      src = h->local.as<float3>() + h->n_vf_r;
      break;
  }
  *count = num;
  if (xyz == nullptr) return CSM_OK;
  if (capacity < num) {
    SetError("capacity %lld below %d points", static_cast<long long>(capacity), num);
    return CSM_E_CAPACITY;
  }
  if (num > 0) {
    CSM_CUDA(cudaMemcpyAsync(xyz, src, sizeof(float3) * num, cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaStreamSynchronize(s));
  }
  return CSM_OK;
}

}  // extern "C"
