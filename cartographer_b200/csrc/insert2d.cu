// ProbabilityGridRangeDataInserter2D::Insert on the device
// (cartographer/mapping/2d/probability_grid_range_data_inserter_2d.cc:35-133) into a
// csm_rt_grid2d handle, with Grid2D::GrowLimits (2d/grid_2d.cc:125-164) and
// ProbabilityGrid::ComputeCroppedGrid (2d/probability_grid.cc:91-107) from device to device.
//
// The reference applies the hit table to every return's cell, then the miss table to every
// pixel of RayToPixelMask (internal/2d/ray_to_pixel_mask.cc) of each return's ray and each
// miss's ray.  A cell updated once carries kUpdateMarker and is skipped until FinishUpdate
// (grid_2d.cc:99-106), so each touched cell ends at hit_table[v] & 0x7fff if a return hits it,
// else miss_table[v] & 0x7fff, whatever the order inside each phase.  Here:
//   * the host decides growth (it holds the limits), computes every superscaled index, and
//     checks them all, so an invalid call changes nothing;
//   * each ray's mask has at most |dx| + |dy| + 1 pixels (it moves one pixel in x, in y or,
//     across an exact corner, in both per step), so the host gives every ray a slot range by
//     prefix sum: k_ins2_hits (one thread per return), k_ins2_rays (one thread per ray
//     replays the reference's integer walk into its slots), k_ins2_misses (one thread per
//     slot) and k_ins2_finish (clears the markers of the hit cells and mask pixels again);
//   * a 16-bit atomicCAS applies a table only while the marker is clear;
//   * the known-cells box follows on the host: a mask contains both its end pixels and stays
//     inside their bounding box, so the box grows by the hit pixels and, with free space on
//     and at least one ray, by the origin's and the misses' pixels.
#include <algorithm>
#include <climits>
#include <cmath>

#include "insert2d.cuh"

struct csm_range_inserter2d {
  csm::Ctx* ctx = nullptr;
  csm_range_inserter_options2d options;
  uint16_t* d_tables = nullptr;   // hit table | miss table, 32768 entries each
  ~csm_range_inserter2d() { cudaFree(d_tables); }
};

namespace csm {

constexpr int kValueCount2 = 32768;              // probability_values.cc:26
constexpr uint16_t kUpdateMarker2 = 1u << 15;    // probability_values.h:82

// ProbabilityGrid::ApplyLookupTable (probability_grid.cc:58-71) without the bookkeeping.
__device__ __forceinline__ void ApplyTable2(uint16_t* cell, const uint16_t* __restrict__ table) {
  unsigned short* c = reinterpret_cast<unsigned short*>(cell);
  unsigned short old = *c;
  while (!(old & kUpdateMarker2)) {
    const unsigned short prev = atomicCAS(c, old, table[old]);
    if (prev == old) return;
    old = prev;
  }
}

__global__ void k_ins2_hits(const int* __restrict__ hit_flat, int n, uint16_t* cells,
                            const uint16_t* __restrict__ hit_table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ApplyTable2(cells + hit_flat[i], hit_table);
}

// RayToPixelMask(begin, end, kSubpixelScale) of ray r into slots [off[r], off[r + 1]) as flat
// cell indices; the slots it does not fill stay -1.
__global__ void k_ins2_rays(int2 begin, const int2* __restrict__ ends, const int* __restrict__ off,
                            int num_rays, int pitch, int* __restrict__ slots) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= num_rays) return;
  int* out = slots + off[r];
  const int cap = off[r + 1] - off[r];
  int count = 0;
  RayToPixelMask2(begin, ends[r], [&](int x, int y) {
    if (count < cap) out[count] = y * pitch + x;
    ++count;
  });
  for (int k = count; k < cap; ++k) out[k] = -1;
}

__global__ void k_ins2_misses(const int* __restrict__ slots, int num_slots, uint16_t* cells,
                              const uint16_t* __restrict__ miss_table) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < num_slots; i += gridDim.x * blockDim.x) {
    const int flat = slots[i];
    if (flat >= 0) ApplyTable2(cells + flat, miss_table);
  }
}

// FinishUpdate: clears the marker of every hit cell and mask pixel (the same cell may be
// listed many times; neighbouring 16-bit cells share a word).
__global__ void k_ins2_finish(const int* __restrict__ hit_flat, int n,
                              const int* __restrict__ slots, int num_slots, uint16_t* cells) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n + num_slots;
       i += gridDim.x * blockDim.x) {
    const int flat = i < n ? hit_flat[i] : slots[i - n];
    if (flat < 0) continue;
    unsigned* word = reinterpret_cast<unsigned*>(cells + (flat & ~1));
    atomicAnd(word, ~(static_cast<unsigned>(kUpdateMarker2) << (16 * (flat & 1))));
  }
}

// Bounding box {min x, min y, max x, max y} of the non-zero cells (box pre-set to empty).
__global__ void k_ins2_known_box(const uint16_t* __restrict__ cells, int nx, int ny, int pitch,
                                 int* box) {
  int lo_x = INT_MAX, lo_y = INT_MAX, hi_x = INT_MIN, hi_y = INT_MIN;
  const long long total = static_cast<long long>(nx) * ny;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % nx), y = static_cast<int>(i / nx);
    if (cells[static_cast<size_t>(y) * pitch + x] == 0) continue;
    lo_x = min(lo_x, x);
    lo_y = min(lo_y, y);
    hi_x = max(hi_x, x);
    hi_y = max(hi_y, y);
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo_x = min(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, o));
    lo_y = min(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, o));
    hi_x = max(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, o));
    hi_y = max(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, o));
  }
  if ((threadIdx.x & 31) == 0 && hi_x != INT_MIN) {
    atomicMin(box, lo_x);
    atomicMin(box + 1, lo_y);
    atomicMax(box + 2, hi_x);
    atomicMax(box + 3, hi_y);
  }
}

// ComputeCroppedGrid's cell loop: cropped (x, y) = SetProbability(GetProbability(source
// (x + ox, y + oy))) for known cells, through the host-computed round-trip table.
__global__ void k_ins2_crop(const uint16_t* __restrict__ src, int src_pitch, int ox, int oy,
                            uint16_t* __restrict__ dst, int nx, int ny, int dst_pitch,
                            const uint16_t* __restrict__ table) {
  const long long total = static_cast<long long>(nx) * ny;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % nx), y = static_cast<int>(i / nx);
    const uint16_t v = src[static_cast<size_t>(y + oy) * src_pitch + (x + ox)];
    if (v != 0) dst[static_cast<size_t>(y) * dst_pitch + x] = table[v & 0x7fff];
  }
}

}  // namespace csm

using namespace csm;

namespace {

// ---- probability_values.{h,cc} in float, as the reference evaluates them ----
constexpr float kMinProbability = 0.1f;
constexpr float kMaxProbability = 1.f - kMinProbability;
constexpr float kMinCorrespondenceCost = 1.f - kMaxProbability;
constexpr float kMaxCorrespondenceCost = 1.f - kMinProbability;

float Odds(float p) { return p / (1.f - p); }
float ProbabilityFromOdds(float odds) { return odds / (odds + 1.f); }
uint16_t CorrespondenceCostToValue(float c) {   // BoundedFloatToValue (probability_values.h:32-44)
  const float v = c > kMaxCorrespondenceCost ? kMaxCorrespondenceCost
                                             : (c < kMinCorrespondenceCost ? kMinCorrespondenceCost : c);
  return static_cast<uint16_t>(
      std::lround((v - kMinCorrespondenceCost) *
                  (32766.f / (kMaxCorrespondenceCost - kMinCorrespondenceCost))) + 1);
}
// kValueToCorrespondenceCost (SlowValueToBoundedFloat, probability_values.cc:29-37, 62-66)
float ValueToCorrespondenceCost(int value) {
  if (value == 0) return kMaxCorrespondenceCost;
  const float kScale = (kMaxCorrespondenceCost - kMinCorrespondenceCost) / (kValueCount2 - 2.f);
  return value * kScale + (kMinCorrespondenceCost - kScale);
}
// ComputeLookupTableToApplyCorrespondenceCostOdds (probability_values.cc:89-105)
void CostOddsTable(float odds, uint16_t* table) {
  table[0] = CorrespondenceCostToValue(1.f - ProbabilityFromOdds(odds)) + kUpdateMarker2;
  for (int cell = 1; cell != kValueCount2; ++cell)
    table[cell] = CorrespondenceCostToValue(
                      1.f - ProbabilityFromOdds(odds * Odds(1.f - ValueToCorrespondenceCost(cell)))) +
                  kUpdateMarker2;
}
// SetProbability(GetProbability(v)) of a known cell (probability_grid.cc:41-49, 78-82): the
// value -> cost -> probability -> cost -> value round trip in float.
const std::vector<uint16_t>& CropTable() {
  static const std::vector<uint16_t> table = [] {
    std::vector<uint16_t> t(kValueCount2, 0);
    for (int v = 1; v < kValueCount2; ++v)
      t[v] = CorrespondenceCostToValue(1.f - (1.f - ValueToCorrespondenceCost(v)));
    return t;
  }();
  return table;
}

bool Finite(const float* p, size_t n) {
  for (size_t i = 0; i < n; ++i)
    if (!std::isfinite(p[i])) return false;
  return true;
}

}  // namespace

namespace csm {

csm_status LaunchKnownBox(csm_rt_grid2d* grid, int* box4) {
  Ctx* ctx = grid->ctx;
  const int init[4] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN};
  CSM_CUDA(cudaMemcpyAsync(box4, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
  const long long total = static_cast<long long>(grid->g.nx) * grid->g.ny;
  k_ins2_known_box<<<Blocks(total, ctx->sm_count * 8), 256, 0, ctx->stream>>>(
      grid->d_cells, grid->g.nx, grid->g.ny, grid->g.pitch, box4);
  CSM_LAUNCH_CHECK();
  return CSM_OK;
}

KnownBox2 BoxFrom(const int* b) {
  KnownBox2 k;
  if (b[0] <= b[2]) {
    k.lo[0] = b[0];
    k.lo[1] = b[1];
    k.hi[0] = b[2];
    k.hi[1] = b[3];
  }
  return k;
}

csm_status NewGrid(Ctx* ctx, int nx, int ny, double resolution, double max_x, double max_y,
                   std::unique_ptr<csm_rt_grid2d>* out, float truncation, float max_weight) {
  std::unique_ptr<csm_rt_grid2d> g(new csm_rt_grid2d);
  g->ctx = ctx;
  RtGridDev& d = g->g;
  std::memset(&d, 0, sizeof(d));
  d.nx = nx;
  d.ny = ny;
  d.pitch = (nx + 7) / 8 * 8;   // rows are multiples of 16 bytes (TMA global strides)
  d.resolution = resolution;
  d.max_x = max_x;
  d.max_y = max_y;
  const size_t bytes = static_cast<size_t>(d.pitch) * ny * 2;
  CSM_CUDA(cudaMalloc(&g->d_cells, bytes));
  CSM_CUDA(cudaMemsetAsync(g->d_cells, 0, bytes, ctx->stream));
  if (truncation > 0.f) {   // a TSDF2D: weight cells and the converter's parameters
    g->truncation = truncation;
    g->max_weight = max_weight;
    CSM_CUDA(cudaMalloc(&g->d_wcells, bytes));
    CSM_CUDA(cudaMemsetAsync(g->d_wcells, 0, bytes, ctx->stream));
  }
  d.cells = g->d_cells;
  d.wcells = g->d_wcells;
  CSM_TRY(RtGridEncodeTmap(g.get()));
  g->known_stale = false;   // empty
  *out = std::move(g);
  return CSM_OK;
}

csm_status GrowCellArrays2(const csm_rt_grid2d* grid, const Limits2& L, int ox, int oy,
                           cudaStream_t s, CellArrays2* out) {
  CellArrays2 a;
  a.pitch = (L.nx + 7) / 8 * 8;   // rows are multiples of 16 bytes (TMA global strides)
  const size_t bytes = static_cast<size_t>(a.pitch) * L.ny * 2;
  const uint16_t* olds[2] = {grid->d_cells, grid->d_wcells};
  uint16_t** news[2] = {&a.cells, &a.wcells};
  for (int k = 0; k < 2; ++k) {
    if (!olds[k]) continue;
    cudaError_t e = cudaMalloc(news[k], bytes);
    if (e == cudaSuccess) e = cudaMemsetAsync(*news[k], 0, bytes, s);
    if (e == cudaSuccess)
      e = cudaMemcpy2DAsync(*news[k] + static_cast<size_t>(oy) * a.pitch + ox,
                            static_cast<size_t>(a.pitch) * 2, olds[k],
                            static_cast<size_t>(grid->g.pitch) * 2,
                            static_cast<size_t>(grid->g.nx) * 2, grid->g.ny,
                            cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) {
      cudaStreamSynchronize(s);
      cudaFree(a.cells);
      cudaFree(a.wcells);
      SetError("%s:%d: growing the grid failed: %s", __FILE__, __LINE__, cudaGetErrorString(e));
      return CSM_E_CUDA;
    }
  }
  *out = a;
  return CSM_OK;
}

csm_status InstallCellArrays2(csm_rt_grid2d* grid, const Limits2& L, CellArrays2* arrays) {
  CellArrays2 old;
  old.cells = grid->d_cells;
  old.wcells = grid->d_wcells;
  old.pitch = grid->g.pitch;
  grid->d_cells = arrays->cells;
  grid->d_wcells = arrays->wcells;
  grid->g.cells = arrays->cells;
  grid->g.wcells = arrays->wcells;
  grid->g.nx = L.nx;
  grid->g.ny = L.ny;
  grid->g.pitch = arrays->pitch;
  grid->g.max_x = L.max_x;
  grid->g.max_y = L.max_y;
  *arrays = old;
  return RtGridEncodeTmap(grid);
}

csm_status RtGridKnownBox(csm_rt_grid2d* grid) {
  if (!grid->known_stale) return CSM_OK;
  Ctx* ctx = grid->ctx;
  CSM_CUDA(cudaSetDevice(ctx->device));
  DevBuf& d_box = ctx->D("ins2_box");
  PinnedBuf& h_box = ctx->P("ins2_box");
  CSM_TRY(d_box.Reserve(4 * sizeof(int)));
  CSM_TRY(h_box.Reserve(4 * sizeof(int)));
  CSM_TRY(LaunchKnownBox(grid, d_box.as<int>()));
  CSM_CUDA(cudaMemcpyAsync(h_box.p, d_box.p, 4 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  grid->known = BoxFrom(h_box.as<int>());
  grid->known_stale = false;
  return CSM_OK;
}

}  // namespace csm

extern "C" {

csm_status csm_rt_grid2d_create_empty(double resolution, double max_x, double max_y,
                                      int32_t num_x_cells, int32_t num_y_cells, int32_t device,
                                      csm_rt_grid2d** out) {
  CSM_REQUIRE(out != nullptr, "null pointer");
  CSM_REQUIRE(resolution > 0. && std::isfinite(resolution) && std::isfinite(max_x) &&
                  std::isfinite(max_y), "limits");
  CSM_REQUIRE(num_x_cells >= 1 && num_y_cells >= 1, "sizes");
  CSM_REQUIRE(num_x_cells < kMaxCells && num_y_cells < kMaxCells, "grid too large");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_rt_grid2d> g;
  CSM_TRY(NewGrid(ctx, num_x_cells, num_y_cells, resolution, max_x, max_y, &g));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = g.release();
  return CSM_OK;
}

csm_status csm_rt_grid2d_read(const csm_rt_grid2d* grid, csm_rt_grid2d_info* info,
                              uint16_t* cells, int64_t capacity) {
  CSM_REQUIRE(grid != nullptr && info != nullptr, "null pointer");
  csm_rt_grid2d* g = const_cast<csm_rt_grid2d*>(grid);   // the box is a cache
  std::lock_guard<std::mutex> lock(g->ctx->mu);
  const RtGridDev& d = g->g;
  CSM_REQUIRE(cells == nullptr || capacity >= static_cast<int64_t>(d.nx) * d.ny, "capacity");
  CSM_CUDA(cudaSetDevice(g->ctx->device));
  CSM_TRY(RtGridKnownBox(g));
  std::memset(info, 0, sizeof(*info));
  info->num_x_cells = d.nx;
  info->num_y_cells = d.ny;
  info->resolution = d.resolution;
  info->max_x = d.max_x;
  info->max_y = d.max_y;
  info->known_empty = g->known.empty() ? 1 : 0;
  info->known_min_x = g->known.lo[0];
  info->known_min_y = g->known.lo[1];
  info->known_max_x = g->known.hi[0];
  info->known_max_y = g->known.hi[1];
  info->is_tsdf = g->d_wcells != nullptr;
  if (cells) {
    CSM_CUDA(cudaMemcpy2DAsync(cells, static_cast<size_t>(d.nx) * 2, g->d_cells,
                               static_cast<size_t>(d.pitch) * 2, static_cast<size_t>(d.nx) * 2,
                               d.ny, cudaMemcpyDeviceToHost, g->ctx->stream));
    CSM_CUDA(cudaStreamSynchronize(g->ctx->stream));
  }
  return CSM_OK;
}

csm_status csm_rt_grid2d_crop(const csm_rt_grid2d* grid, csm_rt_grid2d** out) {
  CSM_REQUIRE(grid != nullptr && out != nullptr, "null pointer");
  CSM_REQUIRE(grid->d_wcells == nullptr, "a TSDF2D handle is not cropped here");
  csm_rt_grid2d* src = const_cast<csm_rt_grid2d*>(grid);   // the box is a cache
  Ctx* ctx = src->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_TRY(RtGridKnownBox(src));
  // ComputeCroppedLimits (grid_2d.cc:110-120)
  int ox = 0, oy = 0, nx = 1, ny = 1;
  if (!src->known.empty()) {
    ox = src->known.lo[0];
    oy = src->known.lo[1];
    nx = src->known.hi[0] - ox + 1;
    ny = src->known.hi[1] - oy + 1;
  }
  const double resolution = src->g.resolution;
  const double max_x = src->g.max_x - resolution * static_cast<double>(oy);
  const double max_y = src->g.max_y - resolution * static_cast<double>(ox);
  std::unique_ptr<csm_rt_grid2d> g;
  CSM_TRY(NewGrid(ctx, nx, ny, resolution, max_x, max_y, &g));
  const std::vector<uint16_t>& table = CropTable();
  DevBuf& d_table = ctx->D("ins2_crop_table");
  CSM_TRY(d_table.Reserve(table.size() * sizeof(uint16_t)));
  CSM_CUDA(cudaMemcpyAsync(d_table.p, table.data(), table.size() * sizeof(uint16_t),
                           cudaMemcpyHostToDevice, ctx->stream));
  if (!src->known.empty()) {
    k_ins2_crop<<<Blocks(static_cast<long long>(nx) * ny, ctx->sm_count * 8), 256, 0,
                  ctx->stream>>>(src->d_cells, src->g.pitch, ox, oy, g->d_cells, nx, ny,
                                 g->g.pitch, d_table.as<uint16_t>());
    CSM_LAUNCH_CHECK();
    // every row and column of the box holds a known cell, and so does the crop's edge
    g->known.lo[0] = g->known.lo[1] = 0;
    g->known.hi[0] = nx - 1;
    g->known.hi[1] = ny - 1;
  }
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = g.release();
  return CSM_OK;
}

csm_status csm_range_inserter2d_create(const csm_range_inserter_options2d* options,
                                       int32_t device, csm_range_inserter2d** out) {
  CSM_REQUIRE(options && out, "null pointer");
  // CreateProbabilityGridRangeDataInserterOptions2D's CHECK_GT / CHECK_LT (:111-112); beyond
  // them, a hit probability of 1 or a negative miss probability would make NaN / negative odds
  CSM_REQUIRE(options->hit_probability > 0.5 && options->hit_probability < 1.0, "hit_probability");
  CSM_REQUIRE(options->miss_probability < 0.5 && options->miss_probability >= 0.0,
              "miss_probability");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_range_inserter2d> ins(new csm_range_inserter2d);
  ins->ctx = ctx;
  ins->options = *options;
  // Odds(options.hit_probability()): the double option enters Odds(float) (:119-122)
  std::vector<uint16_t> tables(2 * kValueCount2);
  CostOddsTable(Odds(static_cast<float>(options->hit_probability)), tables.data());
  CostOddsTable(Odds(static_cast<float>(options->miss_probability)), tables.data() + kValueCount2);
  CSM_CUDA(cudaMalloc(&ins->d_tables, tables.size() * sizeof(uint16_t)));
  CSM_CUDA(cudaMemcpy(ins->d_tables, tables.data(), tables.size() * sizeof(uint16_t),
                      cudaMemcpyHostToDevice));
  *out = ins.release();
  return CSM_OK;
}

csm_status csm_range_inserter2d_destroy(csm_range_inserter2d* inserter) {
  if (!inserter) return CSM_OK;
  std::lock_guard<std::mutex> lock(inserter->ctx->mu);
  cudaSetDevice(inserter->ctx->device);
  cudaStreamSynchronize(inserter->ctx->stream);
  delete inserter;
  return CSM_OK;
}

csm_status csm_range_inserter2d_insert(const csm_range_inserter2d* inserter,
                                       const float origin[3], const float* returns,
                                       int32_t num_returns, const float* misses,
                                       int32_t num_misses, csm_rt_grid2d* grid,
                                       csm_stats* stats) {
  CSM_REQUIRE(inserter && origin && grid, "null pointer");
  CSM_REQUIRE(num_returns >= 0 && (num_returns == 0 || returns), "returns");
  CSM_REQUIRE(num_misses >= 0 && (num_misses == 0 || misses), "misses");
  CSM_REQUIRE(grid->d_wcells == nullptr, "a TSDF2D handle takes the TSDF inserter");
  Ctx* ctx = inserter->ctx;
  CSM_REQUIRE(grid->ctx == ctx, "grid on another device than the inserter");
  const int n = num_returns, m = num_misses;
  CSM_REQUIRE(Finite(origin, 3) && Finite(returns, 3 * static_cast<size_t>(n)) &&
                  Finite(misses, 3 * static_cast<size_t>(m)),
              "non-finite point");
  const bool free_space = inserter->options.insert_free_space != 0;
  std::lock_guard<std::mutex> lock(ctx->mu);
  // ---- GrowAsNeeded (:35-50) on the limits, before anything changes ----
  float lo_x = origin[0], lo_y = origin[1], hi_x = origin[0], hi_y = origin[1];
  auto extend = [&](const float* p, int k) {
    for (int i = 0; i < k; ++i) {
      const float x = p[3 * static_cast<size_t>(i)], y = p[3 * static_cast<size_t>(i) + 1];
      lo_x = std::min(lo_x, x);
      lo_y = std::min(lo_y, y);
      hi_x = std::max(hi_x, x);
      hi_y = std::max(hi_y, y);
    }
  };
  extend(returns, n);
  extend(misses, m);
  constexpr float kPadding = 1e-6f;
  Limits2 L{grid->g.resolution, grid->g.max_x, grid->g.max_y, grid->g.nx, grid->g.ny};
  int grow_x = 0, grow_y = 0;
  CSM_REQUIRE(GrowLimits(lo_x - kPadding, lo_y - kPadding, &L, &grow_x, &grow_y) &&
                  GrowLimits(hi_x + kPadding, hi_y + kPadding, &L, &grow_x, &grow_y),
              "the grid would grow past 30000 cells");
  const bool grow = L.nx != grid->g.nx;
  // ---- superscaled indices (:58-65) ----
  Limits2 S{L.resolution / kSubpixelScale, L.max_x, L.max_y, L.nx * kSubpixelScale,
            L.ny * kSubpixelScale};
  auto superscaled = [&](const float* p, int2* out) -> bool {
    long long ix, iy;
    S.CellIndex(p[0], p[1], &ix, &iy);
    if (!S.Contains(ix, iy)) return false;
    *out = make_int2(static_cast<int>(ix), static_cast<int>(iy));
    return true;
  };
  int2 begin;
  CSM_REQUIRE(superscaled(origin, &begin), "origin outside the grown limits");
  const int num_rays = free_space ? n + m : 0;
  std::vector<int2> ends(std::max(n, num_rays));
  std::vector<int> hit_flat(n), off(num_rays + 1, 0);
  const int pitch = grow ? (L.nx + 7) / 8 * 8 : grid->g.pitch;
  KnownBox2 touched;
  for (int i = 0; i < n; ++i) {
    CSM_REQUIRE(superscaled(returns + 3 * static_cast<size_t>(i), &ends[i]),
                "return outside the grown limits");
    const int x = ends[i].x / kSubpixelScale, y = ends[i].y / kSubpixelScale;
    hit_flat[i] = y * pitch + x;
    touched.Extend(x, y);
  }
  if (free_space) {
    for (int i = 0; i < m; ++i) {
      int2& e = ends[n + i];
      CSM_REQUIRE(superscaled(misses + 3 * static_cast<size_t>(i), &e),
                  "miss outside the grown limits");
      touched.Extend(e.x / kSubpixelScale, e.y / kSubpixelScale);
    }
    if (num_rays > 0) touched.Extend(begin.x / kSubpixelScale, begin.y / kSubpixelScale);
    const int bx = begin.x / kSubpixelScale, by = begin.y / kSubpixelScale;
    long long total = 0;
    for (int r = 0; r < num_rays; ++r) {
      off[r] = static_cast<int>(total);
      total += std::abs(ends[r].x / kSubpixelScale - bx) + std::abs(ends[r].y / kSubpixelScale - by) + 1;
      CSM_REQUIRE(total < (1LL << 31), "too many ray pixels");
    }
    off[num_rays] = static_cast<int>(total);
  }
  const int num_slots = off[num_rays];

  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  // ---- the known box of a handle made from cells, before its cells move ----
  const bool box_stale = grid->known_stale;
  DevBuf& d_box = ctx->D("ins2_box");
  PinnedBuf& h_box = ctx->P("ins2_box");
  if (box_stale) {
    CSM_TRY(d_box.Reserve(4 * sizeof(int)));
    CSM_TRY(h_box.Reserve(4 * sizeof(int)));
    CSM_TRY(LaunchKnownBox(grid, d_box.as<int>()));
    CSM_CUDA(cudaMemcpyAsync(h_box.p, d_box.p, 4 * sizeof(int), cudaMemcpyDeviceToHost, s));
  }
  // ---- growth: the old block at the doubling offset, unknown (0) around it ----
  uint16_t* retired = nullptr;
  if (grow) {
    CellArrays2 arrays;
    CSM_TRY(GrowCellArrays2(grid, L, grow_x, grow_y, s, &arrays));
    const csm_status st = InstallCellArrays2(grid, L, &arrays);
    retired = arrays.cells;
    if (st != CSM_OK) {
      cudaStreamSynchronize(s);
      cudaFree(retired);
      return st;
    }
  }
  // ---- upload: hit cells | ray ends | slot offsets ----
  if (n > 0 || num_rays > 0) {
    const size_t o_ends = (sizeof(int) * static_cast<size_t>(n) + 255) / 256 * 256;
    const size_t o_off = o_ends + (sizeof(int2) * static_cast<size_t>(num_rays) + 255) / 256 * 256;
    const size_t o_slots = o_off + (sizeof(int) * static_cast<size_t>(num_rays + 1) + 255) / 256 * 256;
    const size_t up_bytes = o_slots;
    PinnedBuf& up = ctx->P("ins2_upload");
    DevBuf& d_up = ctx->D("ins2_upload");
    CSM_TRY(up.Reserve(up_bytes));
    CSM_TRY(d_up.Reserve(up_bytes + sizeof(int) * static_cast<size_t>(num_slots)));
    char* h = up.as<char>();
    std::memcpy(h, hit_flat.data(), sizeof(int) * static_cast<size_t>(n));
    std::memcpy(h + o_ends, ends.data(), sizeof(int2) * static_cast<size_t>(num_rays));
    std::memcpy(h + o_off, off.data(), sizeof(int) * static_cast<size_t>(num_rays + 1));
    CSM_CUDA(cudaMemcpyAsync(d_up.p, h, up_bytes, cudaMemcpyHostToDevice, s));
    char* d = d_up.as<char>();
    const int* d_hits = reinterpret_cast<const int*>(d);
    int* d_slots = reinterpret_cast<int*>(d + o_slots);
    const uint16_t* hit_table = inserter->d_tables;
    const uint16_t* miss_table = inserter->d_tables + kValueCount2;
    if (n > 0) {
      k_ins2_hits<<<Blocks(n, 1LL << 30), 256, 0, s>>>(d_hits, n, grid->d_cells, hit_table);
      CSM_LAUNCH_CHECK();
    }
    if (num_rays > 0) {
      k_ins2_rays<<<Blocks(num_rays, 1LL << 30), 256, 0, s>>>(
          begin, reinterpret_cast<const int2*>(d + o_ends), reinterpret_cast<const int*>(d + o_off),
          num_rays, pitch, d_slots);
      CSM_LAUNCH_CHECK();
      k_ins2_misses<<<Blocks(num_slots), 256, 0, s>>>(d_slots, num_slots, grid->d_cells, miss_table);
      CSM_LAUNCH_CHECK();
    }
    k_ins2_finish<<<Blocks(static_cast<long long>(n) + num_slots), 256, 0, s>>>(
        d_hits, n, d_slots, num_slots, grid->d_cells);
    CSM_LAUNCH_CHECK();
  }
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  if (retired) CSM_CUDA(cudaFree(retired));
  // ---- the known-cells box: the old one moved by the growth, plus what this insert set ----
  KnownBox2 known = box_stale ? BoxFrom(h_box.as<int>()) : grid->known;
  if (!known.empty()) {
    known.lo[0] += grow_x;
    known.hi[0] += grow_x;
    known.lo[1] += grow_y;
    known.hi[1] += grow_y;
  }
  known.Extend(touched);
  grid->known = known;
  grid->known_stale = false;
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

}  // extern "C"
