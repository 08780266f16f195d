// Submap textures for display (proto::SubmapQuery::Response::SubmapTexture) straight from the
// device grid handles: ProbabilityGrid / TSDF2D::DrawToSubmapTexture (probability_grid.cc:109-147,
// internal/2d/tsdf_2d.cc:137-181) from a csm_rt_grid2d, and the X-ray view AddToTextureProto
// (mapping/3d/submap_3d.cc:51-176) from a csm_grid3d.  The per-cell and per-voxel work runs here;
// the gzip member, the slice pose and the message framing are host work (submap_texture.h).
// Built with -fmad=false: every float expression is the reference's, uncontracted.
#include <algorithm>
#include <climits>
#include <cmath>
#include <string>

#include <cub/device/device_radix_sort.cuh>

#include "grid3d.cuh"
#include "insert2d.cuh"
#include "rigid3f.h"
#include "rtgrid.cuh"
#include "submap_texture.h"

namespace csm {
namespace {

constexpr int kTexThreads = 256;
constexpr float kXrayObstructedCellProbabilityLimit = 0.501f;   // submap_3d.cc:89

// The step table into shared memory (every kernel here looks it up at divergent indices).
__device__ __forceinline__ void LoadSteps(const LogOddsSteps& steps, float* s) {
  for (int i = threadIdx.x; i < kLogOddsSteps; i += blockDim.x) s[i] = steps.t[i];
  __syncthreads();
}

// The (value, alpha) bytes of `delta` (probability_grid.cc:129-133, submap_3d.cc:136-139).
__device__ __forceinline__ void PutDelta(int delta, uint8_t* out) {
  const uint8_t alpha = static_cast<uint8_t>(delta > 0 ? 0 : -delta);
  const uint8_t value = static_cast<uint8_t>(delta > 0 ? delta : 0);
  out[0] = value;
  out[1] = (value || alpha) ? alpha : 1;
}

// ---- 2D: one thread per cell of the cropped limits (Grid2D::ComputeCroppedLimits) ----
struct Tex2Args {
  const uint16_t* cells;     // probability / tsd cells, row pitch `pitch`
  const uint16_t* wcells;    // TSDF2D weight cells (nullptr for a ProbabilityGrid)
  int pitch, ox, oy, w, h;   // the crop box: offset (ox, oy), w x h cells
  ValueConversion cost;      // ProbabilityGrid: value -> correspondence cost
  const float* tsd_pow;      // TSDF2D: value -> pow(|tsd| / max_tsd, 0.5f)
  const float* weight_norm;  // TSDF2D: value -> weight / max_weight
  uint8_t* out;              // 2 bytes per cell, x fastest
};

__global__ void __launch_bounds__(kTexThreads) k_tex2(Tex2Args a, LogOddsSteps steps) {
  __shared__ float s[kLogOddsSteps];
  LoadSteps(steps, s);
  const long long total = static_cast<long long>(a.w) * a.h;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % a.w), y = static_cast<int>(i / a.w);
    const size_t at = static_cast<size_t>(y + a.oy) * a.pitch + (x + a.ox);
    const uint16_t v = a.cells[at];
    uint8_t* o = a.out + 2 * i;
    if (v == 0) {   // !IsKnown
      o[0] = 0;
      o[1] = 0;
      continue;
    }
    int delta;
    if (a.wcells == nullptr) {
      // GetProbability = 1 - ValueToCorrespondenceCost(v)
      const float p = FSub(1.f, FAdd(FMul(static_cast<float>(v), a.cost.scale), a.cost.bias));
      delta = 128 - LogOddsIntegerFromSteps(p, s);
    } else {
      const double nt = a.tsd_pow[v];
      const double nw = a.weight_norm[a.wcells[at]];
      delta = static_cast<int>(round(__dmul_rn(nw, __dsub_rn(__dmul_rn(nt, 255.), 128.))));
    }
    PutDelta(delta, o);
  }
}

// ---- 3D ----
// ExtractVoxelData (submap_3d.cc:80-110) per voxel of the iteration-order list: the kept voxels'
// pixel (x, y), z index and value in pix[i] (value 0 for a voxel below the limit), and the pixel
// box and the kept count reduced into box = {min x, min y, max x, max y, kept}.
__global__ void __launch_bounds__(kTexThreads)
k_tex3_extract(const int* __restrict__ idx, const uint16_t* __restrict__ val, long long n,
               Rigid3f pose, float resolution, float resolution_inverse, ValueConversion prob,
               int4* __restrict__ pix, int* __restrict__ box) {
  int lo_x = INT_MAX, lo_y = INT_MAX, hi_x = INT_MIN, hi_y = INT_MIN, kept = 0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint16_t v = val[i];
    const float p = FAdd(FMul(static_cast<float>(v), prob.scale), prob.bias);
    if (p < kXrayObstructedCellProbabilityLimit) {
      pix[i] = make_int4(0, 0, 0, 0);
      continue;
    }
    const Vec3f c{FMul(static_cast<float>(idx[3 * i]), resolution),
                  FMul(static_cast<float>(idx[3 * i + 1]), resolution),
                  FMul(static_cast<float>(idx[3 * i + 2]), resolution)};
    const Vec3f g = Rigid3Apply(pose, c);
    const int px = static_cast<int>(lroundf(FMul(g.x, resolution_inverse)));
    const int py = static_cast<int>(lroundf(FMul(g.y, resolution_inverse)));
    const int pz = static_cast<int>(lroundf(FMul(g.z, resolution_inverse)));
    pix[i] = make_int4(px, py, pz, v);
    lo_x = min(lo_x, px);
    lo_y = min(lo_y, py);
    hi_x = max(hi_x, px);
    hi_y = max(hi_y, py);
    ++kept;
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo_x = min(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, o));
    lo_y = min(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, o));
    hi_x = max(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, o));
    hi_y = max(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, o));
    kept += __shfl_xor_sync(0xffffffffu, kept, o);
  }
  if ((threadIdx.x & 31) == 0 && kept > 0) {
    atomicMin(box, lo_x);
    atomicMin(box + 1, lo_y);
    atomicMax(box + 2, hi_x);
    atomicMax(box + 3, hi_y);
    atomicAdd(box + 4, kept);
  }
}

// The sort keys: pixel (max_x - x) * width + (max_y - y) (AccumulatePixelData, :63-65) for a
// kept voxel, `pixels` (past every pixel) for the others; the values are list positions.
__global__ void __launch_bounds__(kTexThreads)
k_tex3_keys(const int4* __restrict__ pix, long long n, int max_x, int max_y, int width,
            unsigned pixels, unsigned* __restrict__ keys, unsigned* __restrict__ pos) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int4 p = pix[i];
    keys[i] = p.w == 0 ? pixels
                       : static_cast<unsigned>(max_x - p.x) * static_cast<unsigned>(width) +
                             static_cast<unsigned>(max_y - p.y);
    pos[i] = static_cast<unsigned>(i);
  }
}

// AccumulatePixelData and ComputePixelValues (:52-77, :114-144), one thread per run of equal
// keys in the stably sorted list: the thread at a run's head walks the run, which holds that
// pixel's voxels in iteration order, so the float probability sum adds them in the reference's
// order.  Pixels without a voxel keep the (0, 0) the output was cleared to.
__global__ void __launch_bounds__(kTexThreads)
k_tex3_runs(const unsigned* __restrict__ keys, const unsigned* __restrict__ pos, int kept,
            const int4* __restrict__ pix, ValueConversion prob, LogOddsSteps steps,
            uint8_t* __restrict__ out) {
  __shared__ float s[kLogOddsSteps];
  LoadSteps(steps, s);
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= kept) return;
  const unsigned key = keys[j];
  if (j > 0 && keys[j - 1] == key) return;
  int count = 0, min_z = INT_MAX, max_z = INT_MIN;
  float probability_sum = 0.f, max_probability = 0.5f;
  for (int k = j; k < kept && keys[k] == key; ++k) {
    const int4 p = pix[pos[k]];
    ++count;
    min_z = min(min_z, p.z);
    max_z = max(max_z, p.z);
    const float probability = FAdd(FMul(static_cast<float>(p.w), prob.scale), prob.bias);
    probability_sum = FAdd(probability_sum, probability);
    max_probability = max_probability < probability ? probability : max_probability;
  }
  constexpr float kMinZDifference = 3.f;
  constexpr float kFreeSpaceWeight = 0.15f;
  const float z_difference = static_cast<float>(max_z - min_z);
  if (z_difference < kMinZDifference) return;
  const float d = FSub(z_difference, static_cast<float>(count));
  const float free_space = d < 0.f ? 0.f : d;
  const float free_space_weight = FMul(kFreeSpaceWeight, free_space);
  const float total_weight = FAdd(static_cast<float>(count), free_space_weight);
  const float free_space_probability = FSub(1.f, max_probability);
  float average = FDiv(FAdd(probability_sum, FMul(free_space_probability, free_space_weight)),
                       total_weight);
  average = average > kMaxProbability ? kMaxProbability
                                      : (average < kMinProbability ? kMinProbability : average);
  PutDelta(128 - LogOddsIntegerFromSteps(average, s), out + 2 * static_cast<size_t>(key));
}

const LogOddsSteps& Steps() {
  static const LogOddsSteps steps = MakeLogOddsSteps();
  return steps;
}

// Gzips `raw` and writes the message (or only its size) as the *_to_proto entry points do.
csm_status FinishTexture(const uint8_t* raw, size_t raw_len, int32_t width, int32_t height,
                         double resolution, const Pose3d& slice, uint8_t* buf, int64_t capacity,
                         int64_t* size) {
  std::string cells;
  if (!GzipMember(raw, raw_len, &cells)) {
    SetError("zlib failed to compress the texture cells");
    return CSM_E_INTERNAL;
  }
  const TextureMessage m = SizeTexture(cells.size(), width, height, resolution, slice);
  *size = m.total;
  if (m.total >= (int64_t(1) << 31)) {
    SetError("a serialized SubmapTexture of %lld bytes exceeds protobuf's 2 GiB limit",
             static_cast<long long>(m.total));
    return CSM_E_CAPACITY;
  }
  if (!buf) return CSM_OK;
  if (capacity < m.total) {
    SetError("capacity %lld is below the %lld bytes of the message",
             static_cast<long long>(capacity), static_cast<long long>(m.total));
    return CSM_E_CAPACITY;
  }
  WriteTexture(buf, m, cells, width, height, resolution, slice);
  return CSM_OK;
}

Pose3d PoseFrom(const double p[7]) {
  return Pose3d{Vec3d{p[0], p[1], p[2]}, Quat4d{p[3], p[4], p[5], p[6]}};
}

}  // namespace
}  // namespace csm

using namespace csm;

extern "C" {

csm_status csm_rt_grid2d_to_texture(const csm_rt_grid2d* grid, const double local_pose[7],
                                    uint8_t* buf, int64_t capacity, int64_t* size) {
  CSM_REQUIRE(grid != nullptr && local_pose != nullptr && size != nullptr, "null pointer");
  CSM_REQUIRE(Finite(local_pose, 7), "non-finite pose");
  csm_rt_grid2d* g = const_cast<csm_rt_grid2d*>(grid);   // the known-cells box is a cache
  Ctx* ctx = g->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_TRY(RefreshKnownBox(g));
  const RtGridDev& d = g->g;
  const bool tsdf = g->d_wcells != nullptr;
  // ComputeCroppedLimits (grid_2d.cc:110-120)
  int ox = 0, oy = 0, w = 1, h = 1;
  if (!g->known.empty()) {
    ox = g->known.lo[0];
    oy = g->known.lo[1];
    w = g->known.hi[0] - ox + 1;
    h = g->known.hi[1] - oy + 1;
  }
  const size_t cells = static_cast<size_t>(w) * h;
  cudaStream_t s = ctx->stream;
  Tex2Args a;
  a.cells = g->d_cells;
  a.wcells = g->d_wcells;
  a.pitch = d.pitch;
  a.ox = ox;
  a.oy = oy;
  a.w = w;
  a.h = h;
  a.cost = MakeValueConversion(kMinCorrespondenceCost, kMaxCorrespondenceCost);
  a.tsd_pow = a.weight_norm = nullptr;
  if (tsdf) {
    // TSDValueConverter's tables (tsd_value_converter.cc:24-34): value 0 gives min_tsd and
    // weight 0; the powers and quotients are taken here, on the host's libm
    PinnedBuf& up = ctx->P("tex2_tables");
    CSM_TRY(up.Reserve(sizeof(float) * 2 * kValueCount));
    float* t = up.as<float>();
    const TsdfConversion c = MakeTsdfConversion(g->truncation, g->max_weight);
    for (int v = 0; v < kValueCount; ++v) {
      const float tsd = v == 0 ? c.min_tsd : v * c.tsd_scale + c.tsd_bias;
      const float weight = v == 0 ? 0.f : v * c.w_scale + c.w_bias;
      t[v] = std::pow(std::abs(tsd) / g->truncation, 0.5f);
      t[kValueCount + v] = weight / g->max_weight;
    }
    DevBuf* d_t;
    CSM_TRY(ctx->Reserve("tex2_tables", sizeof(float) * 2 * kValueCount, &d_t));
    CSM_CUDA(cudaMemcpyAsync(d_t->p, t, sizeof(float) * 2 * kValueCount, cudaMemcpyHostToDevice,
                             s));
    a.tsd_pow = d_t->as<float>();
    a.weight_norm = d_t->as<float>() + kValueCount;
  }
  DevBuf* d_out;
  CSM_TRY(ctx->Reserve("tex2_out", 2 * cells, &d_out));
  a.out = d_out->as<uint8_t>();
  k_tex2<<<Blocks(static_cast<long long>(cells), ctx->sm_count * 8), kTexThreads, 0, s>>>(
      a, Steps());
  CSM_LAUNCH_CHECK();
  PinnedBuf& h_out = ctx->P("tex2_out");
  CSM_TRY(h_out.Reserve(2 * cells));
  CSM_CUDA(cudaMemcpyAsync(h_out.p, d_out->p, 2 * cells, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  // slice_pose = local_pose.inverse() * Translation(max_x, max_y, 0) with the cropped limits'
  // max (probability_grid.cc:141-145)
  const double max_x = d.max_x - d.resolution * oy;
  const double max_y = d.max_y - d.resolution * ox;
  const Pose3d slice = InverseTimesTranslation(PoseFrom(local_pose), Vec3d{max_x, max_y, 0.});
  return FinishTexture(h_out.as<uint8_t>(), 2 * cells, w, h, d.resolution, slice, buf, capacity,
                       size);
}

csm_status csm_grid3d_to_texture(const csm_grid3d* grid, const double global_submap_pose[7],
                                 uint8_t* buf, int64_t capacity, int64_t* size) {
  CSM_REQUIRE(grid != nullptr && global_submap_pose != nullptr && size != nullptr,
              "null pointer");
  CSM_REQUIRE(Finite(global_submap_pose, 7), "non-finite pose");
  Ctx* ctx = grid->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const float resolution = grid->g.resolution;
  long long n = 0;
  const int* d_idx = nullptr;
  const uint16_t* d_val = nullptr;
  CSM_TRY(NonZeroVoxels3D(grid, LLONG_MAX, &n, &d_idx, &d_val));
  if (n >= INT_MAX) {   // the sort's item count
    SetError("%lld non-zero voxels are too many to draw", n);
    return CSM_E_CAPACITY;
  }
  // Eigen::Array2i min_index(INT_MAX, INT_MAX), max_index(INT_MIN, INT_MIN) (:154-155)
  int box[5] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN, 0};
  const ValueConversion prob = MakeValueConversion(kMinProbability, kMaxProbability);
  DevBuf* d_pix = nullptr;
  if (n > 0) {
    DevBuf* d_box;
    CSM_TRY(ctx->Reserve("tex3_box", sizeof(box), &d_box));
    CSM_TRY(ctx->Reserve("tex3_pix", sizeof(int4) * n, &d_pix));
    CSM_CUDA(cudaMemcpyAsync(d_box->p, box, sizeof(box), cudaMemcpyHostToDevice, s));
    const double* p = global_submap_pose;
    const Rigid3f pose{Vec3f{static_cast<float>(p[0]), static_cast<float>(p[1]),
                             static_cast<float>(p[2])},
                       Quatf{static_cast<float>(p[3]), static_cast<float>(p[4]),
                             static_cast<float>(p[5]), static_cast<float>(p[6])}};
    k_tex3_extract<<<Blocks(n, ctx->sm_count * 8), kTexThreads, 0, s>>>(
        d_idx, d_val, n, pose, resolution, 1.f / resolution, prob, d_pix->as<int4>(),
        d_box->as<int>());
    CSM_LAUNCH_CHECK();
    PinnedBuf& h_box = ctx->P("tex3_box");
    CSM_TRY(h_box.Reserve(sizeof(box)));
    CSM_CUDA(cudaMemcpyAsync(h_box.p, d_box->p, sizeof(box), cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaStreamSynchronize(s));
    std::memcpy(box, h_box.p, sizeof(box));
  }
  // width = max_y - min_y + 1 and height = max_x - min_x + 1 in int (:157-158).  Without a kept
  // voxel the box stays (INT_MAX, INT_MIN), and x86-64's wrap-around makes both 2.
  const int32_t width = static_cast<int32_t>(static_cast<uint32_t>(box[3]) -
                                             static_cast<uint32_t>(box[1]) + 1u);
  const int32_t height = static_cast<int32_t>(static_cast<uint32_t>(box[2]) -
                                              static_cast<uint32_t>(box[0]) + 1u);
  const long long pixels = static_cast<long long>(width) * height;
  if (pixels >= (1ll << 30)) {
    SetError("a texture of %d x %d pixels is too large", height, width);
    return CSM_E_CAPACITY;
  }
  const int kept = box[4];
  PinnedBuf& h_out = ctx->P("tex3_out");
  CSM_TRY(h_out.Reserve(2 * static_cast<size_t>(pixels)));
  if (kept == 0) {
    std::memset(h_out.p, 0, 2 * static_cast<size_t>(pixels));
  } else {
    int end_bit = 1;
    while ((1ll << end_bit) <= pixels) ++end_bit;   // keys and the sentinel `pixels`
    size_t sort_bytes = 0;
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, static_cast<unsigned*>(nullptr),
                                             static_cast<unsigned*>(nullptr),
                                             static_cast<unsigned*>(nullptr),
                                             static_cast<unsigned*>(nullptr), static_cast<int>(n),
                                             0, end_bit, s));
    const size_t lane = (sizeof(unsigned) * n + 255) / 256 * 256;
    DevBuf* d_work;
    CSM_TRY(ctx->Reserve("tex3_sort", 4 * lane + sort_bytes, &d_work));
    unsigned* keys_in = d_work->as<unsigned>();
    unsigned* pos_in = reinterpret_cast<unsigned*>(d_work->as<char>() + lane);
    unsigned* keys = reinterpret_cast<unsigned*>(d_work->as<char>() + 2 * lane);
    unsigned* pos = reinterpret_cast<unsigned*>(d_work->as<char>() + 3 * lane);
    DevBuf* d_out;
    CSM_TRY(ctx->Reserve("tex3_out", 2 * static_cast<size_t>(pixels), &d_out));
    CSM_CUDA(cudaMemsetAsync(d_out->p, 0, 2 * static_cast<size_t>(pixels), s));
    k_tex3_keys<<<Blocks(n, ctx->sm_count * 8), kTexThreads, 0, s>>>(
        d_pix->as<int4>(), n, box[2], box[3], width, static_cast<unsigned>(pixels), keys_in,
        pos_in);
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(d_work->as<char>() + 4 * lane, sort_bytes, keys_in,
                                             keys, pos_in, pos, static_cast<int>(n), 0, end_bit,
                                             s));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    k_tex3_runs<<<DivUp(kept, kTexThreads), kTexThreads, 0, s>>>(
        keys, pos, kept, d_pix->as<int4>(), prob, Steps(), d_out->as<uint8_t>());
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cudaMemcpyAsync(h_out.p, d_out->p, 2 * static_cast<size_t>(pixels),
                             cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaStreamSynchronize(s));
  }
  // slice_pose = global_submap_pose.inverse() * Translation(max_x * resolution,
  // max_y * resolution, global z), the products in float (:172-175)
  const Pose3d pose = PoseFrom(global_submap_pose);
  const Pose3d slice = InverseTimesTranslation(
      pose, Vec3d{static_cast<double>(static_cast<float>(box[2]) * resolution),
                  static_cast<double>(static_cast<float>(box[3]) * resolution), pose.t.z});
  return FinishTexture(h_out.as<uint8_t>(), 2 * static_cast<size_t>(pixels), width, height,
                       static_cast<double>(resolution), slice, buf, capacity, size);
}

}  // extern "C"
