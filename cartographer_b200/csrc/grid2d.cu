// The csm_rt_grid2d handle: a ProbabilityGrid or TSDF2D (2d/grid_2d.h) resident on the device.
// Its allocation and TMA descriptor, uploads and read-back, the known-cells box
// (Grid2D::known_cells_box_, computed on the device for a handle made from cells),
// ProbabilityGrid::ComputeCroppedGrid (2d/probability_grid.cc:91-107) from device to device,
// and Grid2D::GrowLimits (2d/grid_2d.cc:125-164) with the insert transaction that both 2D range
// data inserters end with.  Every kernel here is integer-only.
#include <algorithm>
#include <climits>
#include <cmath>
#include <memory>
#include <vector>

#include "insert2d.cuh"
#include "proto_write.h"
#include "rtgrid.cuh"

namespace csm {

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

// DrawProbabilityGrid's pixel loop (probability_grid_points_processor.cc:185-194): pixel (x, y)
// of row blockIdx.y is cell (x + ox, y + oy), its grey level looked up in the host-computed
// colour table (entry 0, the unknown cell, is 128), written as a cairo ARGB32 word.
__global__ void k_ins2_draw(const uint16_t* __restrict__ cells, int pitch, int ox, int oy, int w,
                            const uint8_t* __restrict__ table, uint32_t* __restrict__ pixels) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= w) return;
  const int y = blockIdx.y;
  const uint32_t v = __ldg(table + (cells[static_cast<size_t>(y + oy) * pitch + (x + ox)] & 0x7fff));
  pixels[static_cast<size_t>(y) * w + x] = 0xFF000000u | v << 16 | v << 8 | v;
}

}  // namespace csm

using namespace csm;

namespace {

// rows are multiples of 16 bytes (TMA global strides)
int Pitch(int nx) { return (nx + 7) / 8 * 8; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn GetEncodeTiled() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// (Re-)encodes the handle's TMA box and descriptor for its current cell array and dimensions.
csm_status EncodeTmap(csm_rt_grid2d* g) {
  RtGridDev& d = g->g;
  // TMA box: as wide as the (padded) grid up to 256 cells, as many rows as fit the tile
  d.bw = std::min(d.pitch, 256);
  d.bh = std::max(1, std::min(std::min(d.ny, 256), kRtTileBytes / (d.bw * 2)));
  g->has_tmap = false;
  if (g->d_wcells) {
    std::memset(&g->tmap, 0, sizeof(g->tmap));
    return CSM_OK;
  }
  EncodeTiledFn encode = GetEncodeTiled();
  if (encode) {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.nx), static_cast<cuuint64_t>(d.ny)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.pitch) * 2};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(d.bw), static_cast<cuuint32_t>(d.bh)};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = encode(&g->tmap, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, g->d_cells, dims,
                              strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    g->has_tmap = r == CUDA_SUCCESS;
  }
  if (!g->has_tmap) {
    SetError("cuTensorMapEncodeTiled is unavailable or failed");
    return CSM_E_CUDA;
  }
  return CSM_OK;
}

// A zero-filled handle of the given limits (caller holds ctx->mu): a ProbabilityGrid or, with
// truncation > 0, a TSDF2D (tsd and weight 0) with that converter.  Its known-cells box is empty.
csm_status NewGrid(Ctx* ctx, int nx, int ny, double resolution, double max_x, double max_y,
                   float truncation, float max_weight, std::unique_ptr<csm_rt_grid2d>* out) {
  std::unique_ptr<csm_rt_grid2d> g(new csm_rt_grid2d);
  g->ctx = ctx;
  g->truncation = truncation;
  g->max_weight = max_weight;
  RtGridDev& d = g->g;
  std::memset(&d, 0, sizeof(d));
  d.nx = nx;
  d.ny = ny;
  d.pitch = Pitch(nx);
  d.resolution = resolution;
  d.max_x = max_x;
  d.max_y = max_y;
  const size_t bytes = static_cast<size_t>(d.pitch) * ny * 2;
  CSM_CUDA(cudaMalloc(&g->d_cells, bytes));
  CSM_CUDA(cudaMemsetAsync(g->d_cells, 0, bytes, ctx->stream));
  if (truncation > 0.f) {
    CSM_CUDA(cudaMalloc(&g->d_wcells, bytes));
    CSM_CUDA(cudaMemsetAsync(g->d_wcells, 0, bytes, ctx->stream));
  }
  d.cells = g->d_cells;
  d.wcells = g->d_wcells;
  CSM_TRY(EncodeTmap(g.get()));
  g->known_stale = false;   // empty
  *out = std::move(g);
  return CSM_OK;
}

// The staging of known-cells boxes: slot k is ints [4k, 4k + 4) of the device and pinned
// "ins2_box" buffers.
csm_status ReserveBoxSlots(Ctx* ctx, int n) {
  CSM_TRY(ctx->D("ins2_box").Reserve(4 * sizeof(int) * static_cast<size_t>(n)));
  CSM_TRY(ctx->P("ins2_box").Reserve(4 * sizeof(int) * static_cast<size_t>(n)));
  return CSM_OK;
}

const int* StagedBox(Ctx* ctx, int slot) { return ctx->P("ins2_box").as<int>() + 4 * slot; }

// Starts the known-box reduction of the handle's (tsd) cells and its copy (min x, min y, max x,
// max y) into slot `slot` of the pinned "ins2_box" buffer on the handle's stream; the caller
// reserved the slot and synchronises before BoxFrom reads it.
csm_status StartKnownBox(csm_rt_grid2d* grid, int slot) {
  Ctx* ctx = grid->ctx;
  int* d_box = ctx->D("ins2_box").as<int>() + 4 * slot;
  int* h_box = ctx->P("ins2_box").as<int>() + 4 * slot;
  const int init[4] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN};
  CSM_CUDA(cudaMemcpyAsync(d_box, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
  const long long total = static_cast<long long>(grid->g.nx) * grid->g.ny;
  k_ins2_known_box<<<Blocks(total, ctx->sm_count * 8), 256, 0, ctx->stream>>>(
      grid->d_cells, grid->g.nx, grid->g.ny, grid->g.pitch, d_box);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(h_box, d_box, 4 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  return CSM_OK;
}

// csm_rt_grid2d_create_empty(_tsdf) after the TSDF parameters' check.
csm_status CreateEmpty(double resolution, double max_x, double max_y, int32_t nx, int32_t ny,
                       float truncation, float max_weight, int32_t device, csm_rt_grid2d** out) {
  CSM_REQUIRE(out != nullptr, "null pointer");
  CSM_REQUIRE(resolution > 0. && std::isfinite(resolution) && std::isfinite(max_x) &&
                  std::isfinite(max_y), "limits");
  CSM_REQUIRE(nx >= 1 && ny >= 1, "sizes");
  CSM_REQUIRE(nx < kMaxCells && ny < kMaxCells, "grid too large");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_rt_grid2d> g;
  CSM_TRY(NewGrid(ctx, nx, ny, resolution, max_x, max_y, truncation, max_weight, &g));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = g.release();
  return CSM_OK;
}

// Brings grid->known up to date (one stream synchronisation when it is stale).  Caller holds
// ctx->mu.
csm_status KnownBox(csm_rt_grid2d* grid) {
  if (!grid->known_stale) return CSM_OK;
  Ctx* ctx = grid->ctx;
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_TRY(ReserveBoxSlots(ctx, 1));
  CSM_TRY(StartKnownBox(grid, 0));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  grid->known = BoxFrom(StagedBox(ctx, 0));
  grid->known_stale = false;
  return CSM_OK;
}

// Grid2D::GrowLimits(point) on the limits alone; the cell offset of the old cells in the new
// array accumulates into (ox, oy).  false if the grid would pass the size guard.
bool GrowLimits(float px, float py, Limits2* L, int* ox, int* oy) {
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

// Allocates and fills the arrays of `grid` for limits L on stream s: the old block at cell
// offset (ox, oy), unknown (0) around it, in both arrays of a TSDF2D.  The handle itself is not
// changed.
csm_status GrowCellArrays2(const csm_rt_grid2d* grid, const Limits2& L, int ox, int oy,
                           cudaStream_t s, CellArrays2* out) {
  CellArrays2 a;
  a.pitch = Pitch(L.nx);
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

// Installs `arrays` and the limits L into the handle and re-encodes its TMA descriptor;
// `arrays` gets the old arrays back, to be freed once the stream is done with them.
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
  return EncodeTmap(grid);
}

// SetProbability(GetProbability(v)) of a known cell (probability_grid.cc:41-49, 78-82): the
// value -> cost -> probability -> cost -> value round trip in float.
const std::vector<uint16_t>& CropTable() {
  static const std::vector<uint16_t> table = [] {
    const ValueConversion cost =
        MakeValueConversion(kMinCorrespondenceCost, kMaxCorrespondenceCost);
    std::vector<uint16_t> t(kValueCount, 0);
    for (int v = 1; v < kValueCount; ++v)
      t[v] = BoundedFloatToValue(1.f - (1.f - cost(v)), kMinCorrespondenceCost,
                                 kMaxCorrespondenceCost);
    return t;
  }();
  return table;
}

// ProbabilityToColor(GetProbability(v)) of every cell value (probability_grid_points_processor.cc
// :51-56, probability_grid.cc:78-82) with the reference's float steps, and kUnknownValue = 128
// for value 0.
const std::vector<uint8_t>& ColorTable() {
  static const std::vector<uint8_t> table = [] {
    const ValueConversion cost =
        MakeValueConversion(kMinCorrespondenceCost, kMaxCorrespondenceCost);
    std::vector<uint8_t> t(kValueCount, 128);
    for (int v = 1; v < kValueCount; ++v) {
      const float probability = 1.f - (1.f - cost(v));
      t[v] = static_cast<uint8_t>(std::lround(
          255 * ((probability - kMinProbability) / (kMaxProbability - kMinProbability))));
    }
    return t;
  }();
  return table;
}

// Grid2D::ComputeCroppedLimits (grid_2d.cc:110-120) of a handle whose box is up to date: the
// known-cells box, or 1 x 1 at offset (0, 0) when it is empty.
void CroppedLimits(const csm_rt_grid2d* g, int* ox, int* oy, int* nx, int* ny) {
  *ox = *oy = 0;
  *nx = *ny = 1;
  if (g->known.empty()) return;
  *ox = g->known.lo[0];
  *oy = g->known.lo[1];
  *nx = g->known.hi[0] - *ox + 1;
  *ny = g->known.hi[1] - *oy + 1;
}

}  // namespace

namespace csm {

csm_status RefreshKnownBox(csm_rt_grid2d* grid) { return KnownBox(grid); }

csm_status ReserveKnownBoxSlots(Ctx* ctx, int n) { return ReserveBoxSlots(ctx, n); }

csm_status UploadCells(csm_rt_grid2d* g, const uint16_t* cells, const uint16_t* wcells,
                       cudaStream_t s) {
  CSM_CUDA(cudaMemcpy2DAsync(g->d_cells, static_cast<size_t>(g->g.pitch) * 2, cells,
                             static_cast<size_t>(g->g.nx) * 2, static_cast<size_t>(g->g.nx) * 2,
                             g->g.ny, cudaMemcpyHostToDevice, s));
  if (wcells)
    CSM_CUDA(cudaMemcpy2DAsync(g->d_wcells, static_cast<size_t>(g->g.pitch) * 2, wcells,
                               static_cast<size_t>(g->g.nx) * 2, static_cast<size_t>(g->g.nx) * 2,
                               g->g.ny, cudaMemcpyHostToDevice, s));
  return CSM_OK;
}

csm_status RtGridCreate(const uint16_t* cells, const uint16_t* wcells, float truncation,
                        float max_weight, int32_t nx, int32_t ny, double resolution, double max_x,
                        double max_y, int32_t device, csm_rt_grid2d** out) {
  CSM_REQUIRE(out != nullptr && cells != nullptr, "null pointer");
  CSM_REQUIRE(nx >= 1 && ny >= 1 && resolution > 0., "sizes");
  CSM_REQUIRE(nx < kMaxCells && ny < kMaxCells, "grid too large");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_rt_grid2d> g;
  CSM_TRY(NewGrid(ctx, nx, ny, resolution, max_x, max_y, truncation, max_weight, &g));
  CSM_TRY(UploadCells(g.get(), cells, wcells, ctx->stream));
  g->known_stale = true;
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = g.release();
  return CSM_OK;
}

GridInsert2::GridInsert2(csm_rt_grid2d* grid, int box_slot)
    : L{grid->g.resolution, grid->g.max_x, grid->g.max_y, grid->g.nx, grid->g.ny},
      arrays{grid->d_cells, grid->d_wcells, grid->g.pitch},
      grid_(grid),
      box_slot_(box_slot) {}

GridInsert2::~GridInsert2() {
  if (!grown_) return;
  cudaStreamSynchronize(grid_->ctx->stream);
  cudaFree(arrays.cells);
  cudaFree(arrays.wcells);
}

bool GridInsert2::Grow(float lo_x, float lo_y, float hi_x, float hi_y) {
  constexpr float kPadding = 1e-6f;   // GrowAsNeeded's padding
  if (!GrowLimits(lo_x - kPadding, lo_y - kPadding, &L, &grow_x_, &grow_y_) ||
      !GrowLimits(hi_x + kPadding, hi_y + kPadding, &L, &grow_x_, &grow_y_))
    return false;
  if (L.nx != grid_->g.nx) arrays = CellArrays2{nullptr, nullptr, Pitch(L.nx)};
  return true;
}

csm_status GridInsert2::Begin() {
  Ctx* ctx = grid_->ctx;
  CSM_CUDA(cudaSetDevice(ctx->device));
  // the known box of a handle made from cells, before its cells move
  box_stale_ = grid_->known_stale;
  if (box_stale_) {
    CSM_TRY(ReserveBoxSlots(ctx, box_slot_ + 1));   // no-op once the caller reserved its slots
    CSM_TRY(StartKnownBox(grid_, box_slot_));
  }
  if (L.nx != grid_->g.nx) {   // the old block at the doubling offset, unknown (0) around it
    CSM_TRY(GrowCellArrays2(grid_, L, grow_x_, grow_y_, ctx->stream, &arrays));
    grown_ = true;
  }
  return CSM_OK;
}

csm_status GridInsert2::Commit(const KnownBox2& touched, csm_stats* stats) {
  Ctx* ctx = grid_->ctx;
  if (grown_) {
    const csm_status st = InstallCellArrays2(grid_, L, &arrays);   // arrays: the old ones now
    grown_ = false;
    cudaFree(arrays.cells);
    cudaFree(arrays.wcells);
    if (st != CSM_OK) return st;
  }
  // the old known box moved by the growth, plus what this insert set
  KnownBox2 known = box_stale_ ? BoxFrom(StagedBox(ctx, box_slot_)) : grid_->known;
  if (!known.empty()) {
    known.lo[0] += grow_x_;
    known.hi[0] += grow_x_;
    known.lo[1] += grow_y_;
    known.hi[1] += grow_y_;
  }
  known.Extend(touched);
  grid_->known = known;
  grid_->known_stale = false;
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

}  // namespace csm

extern "C" {

csm_status csm_rt_grid2d_create(const uint16_t* cells, int32_t nx, int32_t ny, double resolution,
                                double max_x, double max_y, int32_t device, csm_rt_grid2d** out) {
  return RtGridCreate(cells, nullptr, 0.f, 0.f, nx, ny, resolution, max_x, max_y, device, out);
}

csm_status csm_rt_grid2d_create_tsdf(const uint16_t* tsd_cells, const uint16_t* weight_cells,
                                     int32_t nx, int32_t ny, double resolution, double max_x,
                                     double max_y, float truncation_distance, float max_weight,
                                     int32_t device, csm_rt_grid2d** out) {
  CSM_REQUIRE(weight_cells != nullptr, "null weight cells");
  CSM_REQUIRE(truncation_distance > 0.f && max_weight > 0.f, "TSDF parameters");
  return RtGridCreate(tsd_cells, weight_cells, truncation_distance, max_weight, nx, ny, resolution,
                      max_x, max_y, device, out);
}

csm_status csm_rt_grid2d_create_empty(double resolution, double max_x, double max_y,
                                      int32_t num_x_cells, int32_t num_y_cells, int32_t device,
                                      csm_rt_grid2d** out) {
  return CreateEmpty(resolution, max_x, max_y, num_x_cells, num_y_cells, 0.f, 0.f, device, out);
}

csm_status csm_rt_grid2d_create_empty_tsdf(double resolution, double max_x, double max_y,
                                           int32_t num_x_cells, int32_t num_y_cells,
                                           float truncation_distance, float max_weight,
                                           int32_t device, csm_rt_grid2d** out) {
  CSM_REQUIRE(truncation_distance > 0.f && max_weight > 0.f && std::isfinite(truncation_distance) &&
                  std::isfinite(max_weight), "TSDF parameters");
  return CreateEmpty(resolution, max_x, max_y, num_x_cells, num_y_cells, truncation_distance,
                     max_weight, device, out);
}

csm_status csm_rt_grid2d_update(csm_rt_grid2d* grid, const uint16_t* cells) {
  CSM_REQUIRE(grid && cells, "null pointer");
  // the weight cells would go stale
  CSM_REQUIRE(grid->d_wcells == nullptr, "a TSDF2D handle is updated by csm_rt_grid2d_update_tsdf");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  CSM_TRY(UploadCells(grid, cells, nullptr, grid->ctx->stream));
  grid->known_stale = true;
  CSM_CUDA(cudaStreamSynchronize(grid->ctx->stream));
  return CSM_OK;
}

csm_status csm_rt_grid2d_update_tsdf(csm_rt_grid2d* grid, const uint16_t* tsd_cells,
                                     const uint16_t* weight_cells) {
  CSM_REQUIRE(grid && tsd_cells && weight_cells, "null pointer");
  CSM_REQUIRE(grid->d_wcells != nullptr, "the grid is not a TSDF2D");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  CSM_TRY(UploadCells(grid, tsd_cells, weight_cells, grid->ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(grid->ctx->stream));
  return CSM_OK;
}

csm_status csm_rt_grid2d_destroy(csm_rt_grid2d* grid) {
  if (!grid) return CSM_OK;
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  cudaSetDevice(grid->ctx->device);
  cudaStreamSynchronize(grid->ctx->stream);
  delete grid;
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
  CSM_TRY(KnownBox(g));
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

csm_status csm_rt_grid2d_limits(const csm_rt_grid2d* grid, double* resolution, double* max_x,
                                double* max_y, int32_t* num_x_cells, int32_t* num_y_cells) {
  CSM_REQUIRE(grid != nullptr, "null pointer");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);   // an insert may be growing the limits
  const RtGridDev& d = grid->g;
  if (resolution) *resolution = d.resolution;
  if (max_x) *max_x = d.max_x;
  if (max_y) *max_y = d.max_y;
  if (num_x_cells) *num_x_cells = d.nx;
  if (num_y_cells) *num_y_cells = d.ny;
  return CSM_OK;
}

csm_status csm_rt_grid2d_read_weights(const csm_rt_grid2d* grid, uint16_t* weight_cells,
                                      int64_t capacity) {
  CSM_REQUIRE(grid != nullptr && weight_cells != nullptr, "null pointer");
  CSM_REQUIRE(grid->d_wcells != nullptr, "the grid is not a TSDF2D");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  const RtGridDev& d = grid->g;
  CSM_REQUIRE(capacity >= static_cast<int64_t>(d.nx) * d.ny, "capacity");
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  CSM_CUDA(cudaMemcpy2DAsync(weight_cells, static_cast<size_t>(d.nx) * 2, grid->d_wcells,
                             static_cast<size_t>(d.pitch) * 2, static_cast<size_t>(d.nx) * 2,
                             d.ny, cudaMemcpyDeviceToHost, grid->ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(grid->ctx->stream));
  return CSM_OK;
}

csm_status csm_rt_grid2d_to_proto(const csm_rt_grid2d* grid, uint8_t* buf, int64_t capacity,
                                  int64_t* size) {
  using namespace wire;
  CSM_REQUIRE(grid != nullptr && size != nullptr, "null pointer");
  csm_rt_grid2d* g = const_cast<csm_rt_grid2d*>(grid);   // the box is a cache
  Ctx* ctx = g->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_TRY(KnownBox(g));
  const RtGridDev& d = g->g;
  const bool tsdf = g->d_wcells != nullptr;
  const size_t cells = static_cast<size_t>(d.nx) * d.ny;
  PinnedBuf& staging = ctx->P("g2p_cells");
  CSM_TRY(staging.Reserve(sizeof(uint16_t) * cells * (tsdf ? 2 : 1)));
  uint16_t* h = staging.as<uint16_t>();
  const uint16_t* arrays[2] = {g->d_cells, g->d_wcells};
  for (int k = 0; k < (tsdf ? 2 : 1); ++k)
    CSM_CUDA(cudaMemcpy2DAsync(h + k * cells, static_cast<size_t>(d.nx) * 2, arrays[k],
                               static_cast<size_t>(d.pitch) * 2, static_cast<size_t>(d.nx) * 2,
                               d.ny, cudaMemcpyDeviceToHost, ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  auto packed_len = [&](const uint16_t* c) {
    int64_t n = 0;
    for (size_t i = 0; i < cells; ++i) n += VarintSize(c[i]);
    return n;
  };
  // proto::Grid2D (grid_2d.proto): limits = 1 {resolution = 1, max = 2 {x = 1, y = 2},
  // cell_limits = 3 {num_x_cells = 1, num_y_cells = 2}}, cells = 2, known_cells_box = 3
  // {max_x = 1, max_y = 2, min_x = 3, min_y = 4}, probability_grid_2d = 4 {} | tsdf_2d = 5
  // {truncation_distance = 1, max_weight = 2, weight_cells = 3}, min / max_correspondence_cost =
  // 6 / 7.  MapLimits' ToProto always sets max and cell_limits (map_limits.h:98-104).
  const int64_t max_len = DoubleFieldSize(d.max_x) + DoubleFieldSize(d.max_y);
  const int64_t cell_limits_len = Int32FieldSize(d.nx) + Int32FieldSize(d.ny);
  const int64_t limits_len = DoubleFieldSize(d.resolution) + DelimitedSize(max_len) +
                             DelimitedSize(cell_limits_len);
  const int64_t cells_len = packed_len(h);
  const KnownBox2& box = g->known;
  const int32_t box_fields[4] = {box.hi[0], box.hi[1], box.lo[0], box.lo[1]};
  int64_t box_len = 0;
  for (int f = 0; f < 4; ++f) box_len += Int32FieldSize(box_fields[f]);
  int64_t weights_len = 0, tsdf_len = 0;
  if (tsdf) {
    weights_len = packed_len(h + cells);
    tsdf_len = FloatFieldSize(g->truncation) + FloatFieldSize(g->max_weight) +
               DelimitedSize(weights_len);
  }
  const float min_cost = tsdf ? -g->truncation : kMinCorrespondenceCost;
  const float max_cost = tsdf ? g->truncation : kMaxCorrespondenceCost;
  const int64_t total = DelimitedSize(limits_len) + DelimitedSize(cells_len) +
                        (box.empty() ? 0 : DelimitedSize(box_len)) +
                        DelimitedSize(tsdf ? tsdf_len : 0) + FloatFieldSize(min_cost) +
                        FloatFieldSize(max_cost);
  *size = total;
  if (total >= (int64_t(1) << 31)) {
    SetError("a serialized Grid2D of %lld bytes exceeds protobuf's 2 GiB limit",
             static_cast<long long>(total));
    return CSM_E_CAPACITY;
  }
  if (!buf) return CSM_OK;
  if (capacity < total) {
    SetError("capacity %lld is below the %lld bytes of the message",
             static_cast<long long>(capacity), static_cast<long long>(total));
    return CSM_E_CAPACITY;
  }
  uint8_t* p = PutDelimitedHeader(buf, 1, limits_len);
  p = PutDoubleField(p, 1, d.resolution);
  p = PutDelimitedHeader(p, 2, max_len);
  p = PutDoubleField(p, 1, d.max_x);
  p = PutDoubleField(p, 2, d.max_y);
  p = PutDelimitedHeader(p, 3, cell_limits_len);
  p = PutInt32Field(p, 1, d.nx);
  p = PutInt32Field(p, 2, d.ny);
  p = PutDelimitedHeader(p, 2, cells_len);
  for (size_t i = 0; i < cells; ++i) p = PutVarint(p, h[i]);
  if (!box.empty()) {
    p = PutDelimitedHeader(p, 3, box_len);
    for (int f = 0; f < 4; ++f) p = PutInt32Field(p, 1 + f, box_fields[f]);
  }
  if (tsdf) {
    p = PutDelimitedHeader(p, 5, tsdf_len);
    p = PutFloatField(p, 1, g->truncation);
    p = PutFloatField(p, 2, g->max_weight);
    p = PutDelimitedHeader(p, 3, weights_len);
    for (size_t i = 0; i < cells; ++i) p = PutVarint(p, h[cells + i]);
  } else {
    p = PutDelimitedHeader(p, 4, 0);
  }
  p = PutFloatField(p, 6, min_cost);
  PutFloatField(p, 7, max_cost);
  return CSM_OK;
}

csm_status csm_rt_grid2d_crop(const csm_rt_grid2d* grid, csm_rt_grid2d** out) {
  CSM_REQUIRE(grid != nullptr && out != nullptr, "null pointer");
  CSM_REQUIRE(grid->d_wcells == nullptr, "a TSDF2D handle is not cropped here");
  csm_rt_grid2d* src = const_cast<csm_rt_grid2d*>(grid);   // the box is a cache
  Ctx* ctx = src->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_TRY(KnownBox(src));
  int ox, oy, nx, ny;
  CroppedLimits(src, &ox, &oy, &nx, &ny);
  const double resolution = src->g.resolution;
  const double max_x = src->g.max_x - resolution * static_cast<double>(oy);
  const double max_y = src->g.max_y - resolution * static_cast<double>(ox);
  std::unique_ptr<csm_rt_grid2d> g;
  CSM_TRY(NewGrid(ctx, nx, ny, resolution, max_x, max_y, 0.f, 0.f, &g));
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

csm_status csm_rt_grid2d_draw(const csm_rt_grid2d* grid, uint32_t* pixels, int64_t capacity,
                              int32_t* width, int32_t* height, int32_t offset[2],
                              csm_stats* stats) {
  CSM_REQUIRE(grid != nullptr && width != nullptr && height != nullptr && offset != nullptr,
              "null pointer");
  CSM_REQUIRE(grid->d_wcells == nullptr, "a TSDF2D handle is not drawn here");
  csm_rt_grid2d* g = const_cast<csm_rt_grid2d*>(grid);   // the box is a cache
  Ctx* ctx = g->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  if (stats) std::memset(stats, 0, sizeof(*stats));
  CSM_CUDA(cudaSetDevice(ctx->device));
  const int box_syncs = g->known_stale ? 1 : 0;
  CSM_TRY(KnownBox(g));
  int ox, oy, w, h;
  CroppedLimits(g, &ox, &oy, &w, &h);
  *width = w;
  *height = h;
  offset[0] = ox;
  offset[1] = oy;
  if (stats) stats->host_syncs = box_syncs;
  if (!pixels) return CSM_OK;
  const int64_t num_pixels = static_cast<int64_t>(w) * h;
  if (capacity < num_pixels) {
    SetError("a %d x %d image, capacity %lld", w, h, static_cast<long long>(capacity));
    return CSM_E_CAPACITY;
  }
  const std::vector<uint8_t>& table = ColorTable();
  DevBuf& d_table = ctx->D("ins2_draw_table");
  DevBuf& d_pixels = ctx->D("ins2_draw_pixels");
  CSM_TRY(d_table.Reserve(table.size()));
  CSM_TRY(d_pixels.Reserve(sizeof(uint32_t) * num_pixels));
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaMemcpyAsync(d_table.p, table.data(), table.size(), cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  k_ins2_draw<<<dim3((w + 255) / 256, h), 256, 0, s>>>(g->d_cells, g->g.pitch, ox, oy, w,
                                                       d_table.as<uint8_t>(),
                                                       d_pixels.as<uint32_t>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(pixels, d_pixels.p, sizeof(uint32_t) * num_pixels,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  if (stats) {
    stats->host_syncs = box_syncs + 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

csm_status csm_rt_grid2d_draw_table(uint8_t* grey) {
  CSM_REQUIRE(grey != nullptr, "null pointer");
  const std::vector<uint8_t>& table = ColorTable();
  std::memcpy(grey, table.data(), table.size());
  return CSM_OK;
}

}  // extern "C"
