// TSDFRangeDataInserter2D::Insert + FinishUpdate on the device
// (cartographer/mapping/internal/2d/tsdf_range_data_inserter_2d.cc:131-239) into a TSDF2D
// csm_rt_grid2d, with NormalEstimation2D (normal_estimation_2d.cc) and Grid2D::GrowLimits.
//
// TSDF2D::SetCell sets the update marker and InsertHit skips marked cells, so each cell is
// written at most once per insert, from its value before the insert, by the first ray (in the
// sorted order) whose pair with it has a non-zero weight (UpdateCell returns early on 0 without
// a marker).  That is a per-cell "lowest ray index wins" selection, independent of thread order:
//   * the host grows the limits, sorts the returns and estimates the normals (std::sort and libm,
//     O(returns)), and computes one record per ray in the reference's float / double mix: the
//     range, the superscaled begin and end, cos / sin of the normal and the ray's weight factors;
//     each ray gets a slot range of |dx| + |dy| + 1 pixels by prefix sum, as in insert2d.cu;
//   * k_tsdf2_rays replays RayToPixelMask into the slots (one thread per ray) and flags a mask
//     pixel outside the grid; k_tsdf2_pairs computes every (ray, cell) pair's update and flags a
//     marked tsd cell; a stable radix sort of the claiming pairs by cell keeps ray order within a
//     cell, so k_tsdf2_apply writes each cell once from its first pair, with no marker;
//   * the known-cells box grows by a min / max reduction over the written cells and comes back
//     with the error flags in the insert's one synchronisation.  A flagged insert writes nothing:
//     the apply kernel reads the flags first, and grown arrays are installed only afterwards.
// Built with -fmad=false: every per-cell operation is the reference's float or double operation.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "insert2d.cuh"

struct csm_tsdf_inserter2d {
  csm::Ctx* ctx = nullptr;
  csm_tsdf_inserter_options2d options;
};

namespace csm {

constexpr int kErrMaskOutside = 1, kErrMarked = 2;

// One ray of the insert, in the sorted order.
struct TsdfRay2 {
  int2 begin, end;      // superscaled ray_begin / ray_end
  float hit_x, hit_y;
  float range;
  float cos_n, sin_n;   // of the estimated normal (projection only)
  float weight;         // weight_factor_range * weight_factor_angle_ray_normal
};

struct TsdfParams2 {
  double resolution, max_x, max_y;
  float origin_x, origin_y;
  float truncation;     // the inserter's (Clamp of update_tsd)
  float max_weight;     // the inserter's (UpdateCell's std::min)
  float sigma;          // update_weight_distance_cell_to_hit_kernel_bandwidth (0: off)
  float sqrt_two_pi;    // kSqrtTwoPi, a float
  int project;
  int nx, ny, pitch;
  unsigned no_claim;    // sort key of a slot that claims no cell (above every flat index)
  TsdfConversion conv;  // the handle's value -> tsd / weight
  float max_tsd, tsd_resolution, max_w, weight_resolution;   // the handle's tsd / weight -> value
};

// GaussianKernel (:49-51): float sigma, double kernel, float result.
__host__ __device__ inline float TsdfGaussian(float x, float sigma, float sqrt_two_pi) {
  const float s = sqrt_two_pi * sigma;
  const float s2 = sigma * sigma;
  return static_cast<float>(1.0 / static_cast<double>(s) *
                            exp(-0.5 * static_cast<double>(x) * static_cast<double>(x) /
                                static_cast<double>(s2)));
}

// RoundToInt(...) + 1 of TSDToValue / WeightToValue (tsd_value_converter.h:39-55).
__device__ inline uint16_t TsdfToValue(float v, float lo, float hi, float resolution) {
  const float c = v > hi ? hi : (v < lo ? lo : v);
  return static_cast<uint16_t>(static_cast<int>(lroundf((c - lo) * resolution)) + 1);
}

__global__ void k_tsdf2_rays(const TsdfRay2* __restrict__ rays, const int* __restrict__ off,
                             int num_rays, int nx, int ny, int pitch, int* __restrict__ slots,
                             int* __restrict__ slot_ray, int* err) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= num_rays) return;
  int* out = slots + off[r];
  const int cap = off[r + 1] - off[r];
  int count = 0;
  bool outside = false;
  RayToPixelMask2(rays[r].begin, rays[r].end, [&](int x, int y) {
    int flat = -1;
    if (x >= 0 && y >= 0 && x < nx && y < ny)
      flat = y * pitch + x;
    else
      outside = true;
    if (count < cap)
      out[count] = flat;
    else
      outside = true;   // cannot happen for a mask inside the grid
    ++count;
  });
  for (int k = count; k < cap; ++k) out[k] = -1;
  for (int k = 0; k < cap; ++k) slot_ray[off[r] + k] = r;
  if (outside) atomicOr(err, kErrMaskOutside);
}

// InsertHit's cell loop body (:204-223) for every slot.
__global__ void k_tsdf2_pairs(const TsdfRay2* __restrict__ rays, const int* __restrict__ slots,
                              const int* __restrict__ slot_ray, int num_slots, TsdfParams2 P,
                              const uint16_t* __restrict__ tsd_cells, unsigned* __restrict__ keys,
                              int* __restrict__ vals, float* __restrict__ update_tsd,
                              float* __restrict__ update_weight, int* err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= num_slots) return;
  const int flat = slots[i];
  unsigned key = P.no_claim;
  if (flat >= 0) {
    const TsdfRay2 R = rays[slot_ray[i]];
    const int x = flat % P.pitch, y = flat / P.pitch;
    // MapLimits::GetCellCenter: double, then float
    const float cx = static_cast<float>(P.max_x - P.resolution * (y + 0.5));
    const float cy = static_cast<float>(P.max_y - P.resolution * (x + 0.5));
    const float dx = cx - P.origin_x, dy = cy - P.origin_y;
    float t = R.range - __fsqrt_rn(dx * dx + dy * dy);
    if (P.project) t = (cx - R.hit_x) * R.cos_n + (cy - R.hit_y) * R.sin_n;
    t = t > P.truncation ? P.truncation : (t < -P.truncation ? -P.truncation : t);   // Clamp
    float w = R.weight;
    if (P.sigma != 0.f) w = w * TsdfGaussian(t, P.sigma, P.sqrt_two_pi);
    if (tsd_cells[flat] & kUpdateMarker) atomicOr(err, kErrMarked);
    if (w != 0.f) key = static_cast<unsigned>(flat);   // UpdateCell's early return claims nothing
    update_tsd[i] = t;
    update_weight[i] = w;
  }
  keys[i] = key;
  vals[i] = i;
}

// UpdateCell + SetCell (:227-239, tsdf_2d.cc:55-68) of each cell's first claiming pair.
__global__ void k_tsdf2_apply(const unsigned* __restrict__ keys, const int* __restrict__ vals,
                              int num_slots, const float* __restrict__ update_tsd,
                              const float* __restrict__ update_weight, TsdfParams2 P,
                              uint16_t* tsd_cells, uint16_t* weight_cells, int* flags) {
  if (*(volatile int*)flags != 0) return;   // a refused insert writes nothing
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= num_slots) return;
  const unsigned key = keys[i];
  if (key == P.no_claim || (i > 0 && keys[i - 1] == key)) return;
  const int slot = vals[i];
  const float ut = update_tsd[slot], uw = update_weight[slot];
  const int tv = tsd_cells[key] & 0x7fff, wv = weight_cells[key] & 0x7fff;
  // GetTSDAndWeight through the handle's conversion tables (value 0: min tsd, weight 0)
  const float tsd = tv ? tv * P.conv.tsd_scale + P.conv.tsd_bias : P.conv.min_tsd;
  const float w = wv ? wv * P.conv.w_scale + P.conv.w_bias : 0.f;
  float updated_weight = w + uw;
  const float updated_sdf = (tsd * w + ut * uw) / updated_weight;
  updated_weight = P.max_weight < updated_weight ? P.max_weight : updated_weight;   // std::min
  tsd_cells[key] = TsdfToValue(updated_sdf, P.conv.min_tsd, P.max_tsd, P.tsd_resolution);
  weight_cells[key] = TsdfToValue(updated_weight, 0.f, P.max_w, P.weight_resolution);
  const int x = static_cast<int>(key) % P.pitch, y = static_cast<int>(key) / P.pitch;
  atomicMin(flags + 1, x);
  atomicMin(flags + 2, y);
  atomicMax(flags + 3, x);
  atomicMax(flags + 4, y);
}

}  // namespace csm

using namespace csm;

namespace {

struct P3 { float x, y, z; };

// Eigen's norm() / normalized() of float vectors: the squares summed in index order, one sqrt,
// a division per component.
float Norm2(float x, float y) { return std::sqrt(x * x + y * y); }
float Norm3(float x, float y, float z) { return std::sqrt(x * x + y * y + z * z); }

// RangeDataSorter (:69-88)
struct RangeDataSorter {
  float ox, oy;
  bool operator()(const P3& lhs, const P3& rhs) const {
    float lx = lhs.x - ox, ly = lhs.y - oy, rx = rhs.x - ox, ry = rhs.y - oy;
    const float ln = lx * lx + ly * ly, rn = rx * rx + ry * ry;
    if (ln > 0.f) {
      const float s = std::sqrt(ln);
      lx /= s;
      ly /= s;
    }
    if (rn > 0.f) {
      const float s = std::sqrt(rn);
      rx /= s;
      ry /= s;
    }
    if ((ly < 0.f) != (ry < 0.f)) return ly < 0.f;
    if (ly < 0.f) return lx < rx;
    return lx > rx;
  }
};

// EstimateNormal (normal_estimation_2d.cc:30-61)
float EstimateNormal(const std::vector<P3>& r, size_t i, size_t begin, size_t end, const P3& o) {
  const P3& p = r[i];
  if (end - begin < 2) return std::atan2(o.y - p.y, o.x - p.x);
  float mx = 0.f, my = 0.f, mz = 0.f;
  const float tox = o.x - p.x, toy = o.y - p.y, toz = o.z - p.z;
  for (size_t k = begin; k < end; ++k) {
    if (k == i) continue;
    const float tx = p.x - r[k].x, ty = p.y - r[k].y;
    float nx = -ty, ny = tx, nz = 0.f;
    if (Norm3(nx, ny, nz) < 1e-6f) continue;
    if (nx * tox + ny * toy + nz * toz < 0) {
      nx = -nx;
      ny = -ny;
      nz = -nz;
    }
    const float z = nx * nx + ny * ny + nz * nz;
    if (z > 0.f) {
      const float s = std::sqrt(z);
      nx /= s;
      ny /= s;
      nz /= s;
    }
    mx += nx;
    my += ny;
    mz += nz;
  }
  return std::atan2(my, mx);
}

// EstimateNormals (normal_estimation_2d.cc:78-109) over returns sorted by angle.
std::vector<float> EstimateNormals(const std::vector<P3>& r, const P3& o, int num_samples,
                                   float radius) {
  std::vector<float> normals;
  normals.reserve(r.size());
  const size_t max_num_samples = static_cast<size_t>(num_samples);
  for (size_t cur = 0; cur < r.size(); ++cur) {
    const P3& hit = r[cur];
    size_t begin = cur;
    for (; begin > 0 && cur - begin < max_num_samples / 2 &&
           Norm3(hit.x - r[begin - 1].x, hit.y - r[begin - 1].y, hit.z - r[begin - 1].z) < radius;
         --begin) {
    }
    size_t end = cur;
    for (; end < r.size() && end - cur < std::ceil(max_num_samples / 2.0) + 1 &&
           Norm3(hit.x - r[end].x, hit.y - r[end].y, hit.z - r[end].z) < radius;
         ++end) {
    }
    normals.push_back(EstimateNormal(r, cur, begin, end, o));
  }
  return normals;
}

// common::NormalizeAngleDifference<float>
float NormalizeAngleDifference(float d) {
  const float kPi = static_cast<float>(M_PI);
  while (d > kPi) d -= 2. * kPi;
  while (d < -kPi) d += 2. * kPi;
  return d;
}

}  // namespace

extern "C" {

csm_status csm_tsdf_inserter2d_create(const csm_tsdf_inserter_options2d* options, int32_t device,
                                      csm_tsdf_inserter2d** out) {
  CSM_REQUIRE(options && out, "null pointer");
  // CreateNormalEstimationOptions2D's CHECK_GTs (normal_estimation_2d.cc:70-71)
  CSM_REQUIRE(options->num_normal_samples > 0, "num_normal_samples");
  CSM_REQUIRE(options->sample_radius > 0.0, "sample_radius");
  CSM_REQUIRE(options->truncation_distance > 0.0 && std::isfinite(options->truncation_distance),
              "truncation_distance");
  CSM_REQUIRE(options->maximum_weight > 0.0 && std::isfinite(options->maximum_weight),
              "maximum_weight");
  CSM_REQUIRE(std::isfinite(options->sample_radius) &&
                  std::isfinite(options->update_weight_angle_scan_normal_to_ray_kernel_bandwidth) &&
                  std::isfinite(options->update_weight_distance_cell_to_hit_kernel_bandwidth),
              "non-finite option");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::unique_ptr<csm_tsdf_inserter2d> ins(new csm_tsdf_inserter2d);
  ins->ctx = ctx;
  ins->options = *options;
  *out = ins.release();
  return CSM_OK;
}

csm_status csm_tsdf_inserter2d_destroy(csm_tsdf_inserter2d* inserter) {
  delete inserter;
  return CSM_OK;
}

csm_status csm_tsdf_inserter2d_insert(const csm_tsdf_inserter2d* inserter, const float origin[3],
                                      const float* returns, int32_t num_returns,
                                      csm_rt_grid2d* grid, csm_stats* stats) {
  CSM_REQUIRE(inserter && origin && grid, "null pointer");
  CSM_REQUIRE(num_returns >= 0 && (num_returns == 0 || returns), "returns");
  CSM_REQUIRE(grid->d_wcells != nullptr, "a ProbabilityGrid handle takes the ProbabilityGrid inserter");
  Ctx* ctx = inserter->ctx;
  CSM_REQUIRE(grid->ctx == ctx, "grid on another device than the inserter");
  const int n = num_returns;
  CSM_REQUIRE(Finite(origin, 3) && Finite(returns, 3 * static_cast<size_t>(n)), "non-finite point");
  const csm_tsdf_inserter_options2d& opt = inserter->options;
  const float truncation = static_cast<float>(opt.truncation_distance);
  std::lock_guard<std::mutex> lock(ctx->mu);
  const P3 o{origin[0], origin[1], origin[2]};
  std::vector<P3> pts(n);
  if (n > 0) std::memcpy(pts.data(), returns, sizeof(P3) * static_cast<size_t>(n));

  // ---- GrowAsNeeded (:33-47): each return extended by the truncation along its 3D ray ----
  float lo_x = o.x, lo_y = o.y, hi_x = o.x, hi_y = o.y;
  for (const P3& p : pts) {
    float dx = p.x - o.x, dy = p.y - o.y, dz = p.z - o.z;
    const float z = dx * dx + dy * dy + dz * dz;
    if (z > 0.f) {
      const float s = std::sqrt(z);
      dx /= s;
      dy /= s;
    }
    const float ex = p.x + truncation * dx, ey = p.y + truncation * dy;
    lo_x = std::min(lo_x, ex);
    lo_y = std::min(lo_y, ey);
    hi_x = std::max(hi_x, ex);
    hi_y = std::max(hi_y, ey);
  }
  GridInsert2 tx(grid);
  CSM_REQUIRE(tx.Grow(lo_x, lo_y, hi_x, hi_y), "the grid would grow past 30000 cells");
  const Limits2& L = tx.L;

  // ---- sort and normals (:139-152) ----
  const bool angle_weight = opt.update_weight_angle_scan_normal_to_ray_kernel_bandwidth != 0.f;
  const bool project = opt.project_sdf_distance_to_scan_normal != 0;
  std::vector<float> normals;
  if (project || angle_weight) {
    std::sort(pts.begin(), pts.end(), RangeDataSorter{o.x, o.y});
    normals = EstimateNormals(pts, o, opt.num_normal_samples, static_cast<float>(opt.sample_radius));
  }

  // ---- one record per ray (InsertHit :171-201) ----
  const float sqrt_two_pi = static_cast<float>(std::sqrt(2.0 * M_PI));
  const Limits2 S{L.resolution / kSubpixelScale, L.max_x, L.max_y, L.nx * kSubpixelScale,
                  L.ny * kSubpixelScale};
  // a superscaled index whose pixel (C division) lies outside the grid puts that pixel in the mask
  auto superscaled = [&](float px, float py, int2* out) -> bool {
    long long ix, iy;
    S.CellIndex(px, py, &ix, &iy);
    if (ix <= -kSubpixelScale || iy <= -kSubpixelScale || ix >= S.nx || iy >= S.ny) return false;
    *out = make_int2(static_cast<int>(ix), static_cast<int>(iy));
    return true;
  };
  std::vector<TsdfRay2> rays;
  rays.reserve(n);
  std::vector<int> off(1, 0);
  off.reserve(n + 1);
  long long total = 0;
  for (int k = 0; k < n; ++k) {
    const float hx = pts[k].x, hy = pts[k].y;
    const float rx = hx - o.x, ry = hy - o.y;
    const float range = Norm2(rx, ry);
    if (range < truncation) continue;
    const float ratio = truncation / range;
    const float bx = opt.update_free_space ? o.x : o.x + (1.0f - ratio) * rx;
    const float by = opt.update_free_space ? o.y : o.y + (1.0f - ratio) * ry;
    const float ex = o.x + (1.0f + ratio) * rx, ey = o.y + (1.0f + ratio) * ry;
    TsdfRay2 R;
    CSM_REQUIRE(superscaled(bx, by, &R.begin) && superscaled(ex, ey, &R.end),
                "a ray mask leaves the grown grid");
    const float normal = normals.empty() ? std::numeric_limits<float>::quiet_NaN() : normals[k];
    float w_angle = 1.f;
    if (angle_weight) {
      const float a = NormalizeAngleDifference(normal - std::atan2(-ry, -rx));
      w_angle = TsdfGaussian(
          a, static_cast<float>(opt.update_weight_angle_scan_normal_to_ray_kernel_bandwidth),
          sqrt_two_pi);
    }
    float w_range = 1.f;
    if (opt.update_weight_range_exponent != 0) {   // ComputeRangeWeightFactor (:90-96)
      w_range = 0.f;
      if (std::abs(range) > 1e-6f)
        w_range = static_cast<float>(
            1.f / std::pow(static_cast<double>(range),
                           static_cast<double>(opt.update_weight_range_exponent)));
    }
    R.hit_x = hx;
    R.hit_y = hy;
    R.range = range;
    R.cos_n = project ? std::cos(normal) : 0.f;
    R.sin_n = project ? std::sin(normal) : 0.f;
    R.weight = w_range * w_angle;
    rays.push_back(R);
    total += std::abs(R.end.x / kSubpixelScale - R.begin.x / kSubpixelScale) +
             std::abs(R.end.y / kSubpixelScale - R.begin.y / kSubpixelScale) + 1;
    CSM_REQUIRE(total < (1LL << 30), "too many ray pixels");
    off.push_back(static_cast<int>(total));
  }
  const int num_rays = static_cast<int>(rays.size());
  const int num_slots = static_cast<int>(total);

  TsdfParams2 P;
  std::memset(&P, 0, sizeof(P));
  P.resolution = L.resolution;
  P.max_x = L.max_x;
  P.max_y = L.max_y;
  P.origin_x = o.x;
  P.origin_y = o.y;
  P.truncation = truncation;
  P.max_weight = static_cast<float>(opt.maximum_weight);
  P.sigma = static_cast<float>(opt.update_weight_distance_cell_to_hit_kernel_bandwidth);
  P.sqrt_two_pi = sqrt_two_pi;
  P.project = project ? 1 : 0;
  P.nx = L.nx;
  P.ny = L.ny;
  P.pitch = tx.arrays.pitch;
  P.no_claim = static_cast<unsigned>(P.pitch) * static_cast<unsigned>(L.ny);
  P.conv = MakeTsdfConversion(grid->truncation, grid->max_weight);
  P.max_tsd = grid->truncation;   // TSDValueConverter(max_tsd, max_weight)
  P.tsd_resolution = ValueResolution(-grid->truncation, grid->truncation);
  P.max_w = grid->max_weight;
  P.weight_resolution = ValueResolution(0.f, grid->max_weight);

  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_TRY(tx.Begin());
  const CellArrays2& work = tx.arrays;

  // ---- upload: flags + box | ray records | slot offsets; workspace for slots and pairs ----
  auto align = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t o_rays = align(5 * sizeof(int));
  const size_t o_off = o_rays + align(sizeof(TsdfRay2) * num_rays);
  const size_t up_bytes = o_off + align(sizeof(int) * (num_rays + 1));
  const size_t ns = static_cast<size_t>(num_slots);
  const size_t o_slots = up_bytes;
  const size_t o_slot_ray = o_slots + align(sizeof(int) * ns);
  const size_t o_keys = o_slot_ray + align(sizeof(int) * ns);
  const size_t o_keys_out = o_keys + align(sizeof(unsigned) * ns);
  const size_t o_vals = o_keys_out + align(sizeof(unsigned) * ns);
  const size_t o_vals_out = o_vals + align(sizeof(int) * ns);
  const size_t o_utsd = o_vals_out + align(sizeof(int) * ns);
  const size_t o_uw = o_utsd + align(sizeof(float) * ns);
  const size_t o_temp = o_uw + align(sizeof(float) * ns);
  int end_bit = 1;
  while (end_bit < 32 && (P.no_claim >> end_bit) != 0) ++end_bit;
  size_t temp_bytes = 0;
  if (num_slots > 0) {
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(
        nullptr, temp_bytes, static_cast<unsigned*>(nullptr), static_cast<unsigned*>(nullptr),
        static_cast<int*>(nullptr), static_cast<int*>(nullptr), num_slots, 0, end_bit, s));
  }
  PinnedBuf& up = ctx->P("tsdf2_upload");
  PinnedBuf& h_back = ctx->P("tsdf2_back");
  DevBuf& d_work = ctx->D("tsdf2_work");
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(h_back.Reserve(5 * sizeof(int)));
  CSM_TRY(d_work.Reserve(o_temp + temp_bytes));
  char* h = up.as<char>();
  const int init[5] = {0, INT_MAX, INT_MAX, INT_MIN, INT_MIN};
  std::memcpy(h, init, sizeof(init));
  if (num_rays > 0) std::memcpy(h + o_rays, rays.data(), sizeof(TsdfRay2) * num_rays);
  std::memcpy(h + o_off, off.data(), sizeof(int) * (num_rays + 1));
  char* d = d_work.as<char>();
  int* d_flags = reinterpret_cast<int*>(d);
  CSM_CUDA(cudaMemcpyAsync(d, h, up_bytes, cudaMemcpyHostToDevice, s));
  if (num_rays > 0) {
    const TsdfRay2* d_rays = reinterpret_cast<const TsdfRay2*>(d + o_rays);
    int* d_slots = reinterpret_cast<int*>(d + o_slots);
    int* d_slot_ray = reinterpret_cast<int*>(d + o_slot_ray);
    unsigned* d_keys = reinterpret_cast<unsigned*>(d + o_keys);
    unsigned* d_keys_out = reinterpret_cast<unsigned*>(d + o_keys_out);
    int* d_vals = reinterpret_cast<int*>(d + o_vals);
    int* d_vals_out = reinterpret_cast<int*>(d + o_vals_out);
    float* d_utsd = reinterpret_cast<float*>(d + o_utsd);
    float* d_uw = reinterpret_cast<float*>(d + o_uw);
    k_tsdf2_rays<<<Blocks(num_rays, 1LL << 30), 256, 0, s>>>(
        d_rays, reinterpret_cast<const int*>(d + o_off), num_rays, L.nx, L.ny, P.pitch, d_slots,
        d_slot_ray, d_flags);
    CSM_LAUNCH_CHECK();
    k_tsdf2_pairs<<<Blocks(num_slots, 1LL << 30), 256, 0, s>>>(
        d_rays, d_slots, d_slot_ray, num_slots, P, work.cells, d_keys, d_vals, d_utsd, d_uw,
        d_flags);
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(d + o_temp, temp_bytes, d_keys, d_keys_out, d_vals,
                                             d_vals_out, num_slots, 0, end_bit, s));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    k_tsdf2_apply<<<Blocks(num_slots, 1LL << 30), 256, 0, s>>>(
        d_keys_out, d_vals_out, num_slots, d_utsd, d_uw, P, work.cells, work.wcells, d_flags);
    CSM_LAUNCH_CHECK();
  }
  CSM_CUDA(cudaMemcpyAsync(h_back.p, d_flags, 5 * sizeof(int), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  const int* hb = h_back.as<int>();
  if (hb[0] != 0) {
    SetError("%s:%d: invalid argument: %s", __FILE__, __LINE__,
             (hb[0] & kErrMarked) ? "a tsd cell on a ray carries the update marker"
                                  : "a ray mask leaves the grown grid");
    return CSM_E_INVALID;
  }
  return tx.Commit(BoxFrom(hb + 1), stats);
}

}  // extern "C"
