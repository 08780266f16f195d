// ProbabilityGridRangeDataInserter2D::Insert on the device
// (cartographer/mapping/2d/probability_grid_range_data_inserter_2d.cc:35-133) into a
// csm_rt_grid2d handle, growing it as Grid2D::GrowLimits (2d/grid_2d.cc:125-164) does.
//
// The reference applies the hit table to every return's cell, then the miss table to every
// pixel of RayToPixelMask (internal/2d/ray_to_pixel_mask.cc) of each return's ray and each
// miss's ray.  A cell updated once carries kUpdateMarker and is skipped until FinishUpdate
// (grid_2d.cc:99-106), so each touched cell ends at hit_table[v] & 0x7fff if a return hits it,
// else miss_table[v] & 0x7fff, whatever the order inside each phase.  Here:
//   * the host decides growth (it holds the limits), computes every superscaled index, and
//     checks them all, so an invalid call changes nothing; the kernels write grown copies of
//     the cells, installed after the insert's one synchronisation (GridInsert2, grid2d.cu);
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

__global__ void k_ins2_hits(const int* __restrict__ hit_flat, int n, uint16_t* cells,
                            const uint16_t* __restrict__ hit_table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ApplyTable(cells + hit_flat[i], hit_table);
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
    if (flat >= 0) ApplyTable(cells + flat, miss_table);
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
    ClearUpdateMarker(cells, flat);
  }
}

}  // namespace csm

using namespace csm;


extern "C" {

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
  std::vector<uint16_t> tables(2 * kValueCount);
  ComputeLookupTableToApplyCorrespondenceCostOdds(
      Odds(static_cast<float>(options->hit_probability)), tables.data());
  ComputeLookupTableToApplyCorrespondenceCostOdds(
      Odds(static_cast<float>(options->miss_probability)), tables.data() + kValueCount);
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
  GridInsert2 tx(grid);
  CSM_REQUIRE(tx.Grow(lo_x, lo_y, hi_x, hi_y), "the grid would grow past 30000 cells");
  const Limits2& L = tx.L;
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
  const int pitch = tx.arrays.pitch;
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

  CSM_TRY(tx.Begin());
  cudaStream_t s = ctx->stream;
  uint16_t* cells = tx.arrays.cells;
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
    const uint16_t* miss_table = inserter->d_tables + kValueCount;
    if (n > 0) {
      k_ins2_hits<<<Blocks(n, 1LL << 30), 256, 0, s>>>(d_hits, n, cells, hit_table);
      CSM_LAUNCH_CHECK();
    }
    if (num_rays > 0) {
      k_ins2_rays<<<Blocks(num_rays, 1LL << 30), 256, 0, s>>>(
          begin, reinterpret_cast<const int2*>(d + o_ends), reinterpret_cast<const int*>(d + o_off),
          num_rays, pitch, d_slots);
      CSM_LAUNCH_CHECK();
      k_ins2_misses<<<Blocks(num_slots), 256, 0, s>>>(d_slots, num_slots, cells, miss_table);
      CSM_LAUNCH_CHECK();
    }
    k_ins2_finish<<<Blocks(static_cast<long long>(n) + num_slots), 256, 0, s>>>(
        d_hits, n, d_slots, num_slots, cells);
    CSM_LAUNCH_CHECK();
  }
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return tx.Commit(touched, stats);
}

}  // extern "C"
