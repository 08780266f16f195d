// RangeDataInserter3D::Insert on the device
// (cartographer/mapping/3d/range_data_inserter_3d.cc:27-68, 87-114) into the dense device
// copies of a HybridGrid (csm_grid3d) and an IntensityHybridGrid (csm_intensity_grid3d).
//
// The reference walks the returns in order, applying a lookup table to each hit cell and to
// the last num_free_space_voxels samples of each ray (HybridGrid::ApplyLookupTable,
// hybrid_grid.h:502-518): a cell updated once in an insert carries kUpdateMarker and is
// skipped until FinishUpdate (:492-499) clears the markers.  So each touched cell ends at
// hit_table[v] & 0x7fff if a return hits it, else miss_table[v] & 0x7fff — whatever the order
// inside each phase.  Here:
//   * the host computes every cell (GetCellIndex, :428-433) and checks them, so an invalid
//     call changes nothing and the box an insert needs is known before any launch;
//   * GridInsert3 (grid3d.cu) grows the handles' volumes, and installs them only after the
//     insert's one synchronisation;
//   * k_ins3_hits (one thread per return), then k_ins3_misses (one per (return, sample)):
//     a 16-bit atomicCAS applies the table only while the marker is clear; the thread whose
//     CAS set the marker appends the cell to the insert's touched list;
//   * k_ins3_finish clears the markers of exactly the listed cells (a value that carried the
//     marker before the insert keeps it, as in the reference);
//   * intensities (IntensityHybridGrid::AddIntensity, :552-560): (voxel, intensity) pairs in
//     return order are stable-sorted by voxel (CUB radix sort), then one thread per run of
//     equal voxels adds them to the voxel's sum in order and writes sum, count and the mean
//     GetIntensity reads (:562-569).  No float atomics: the order of the adds is the reference's.
#include <algorithm>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "grid3d.cuh"
#include "value_conversion.h"

struct csm_range_inserter3d {
  csm::Ctx* ctx = nullptr;
  csm_range_inserter_options3d options;
  uint16_t* d_tables = nullptr;   // hit table | miss table, 32768 entries each
  ~csm_range_inserter3d() { cudaFree(d_tables); }
};

namespace csm {

__device__ __forceinline__ void Touched(unsigned long long idx, unsigned long long* list,
                                        unsigned long long* count) {
  list[atomicAdd(count, 1ull)] = idx;
}

__global__ void k_ins3_hits(const int* __restrict__ cells, int n, Box3 box, uint16_t* vol,
                            const uint16_t* __restrict__ hit_table, unsigned long long* list,
                            unsigned long long* count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long idx = box.Index(cells[3 * i], cells[3 * i + 1], cells[3 * i + 2]);
  if (ApplyTable(vol + idx, hit_table)) Touched(idx, list, count);
}

// InsertMissesIntoGrid (range_data_inserter_3d.cc:27-52): thread (r, k) takes sample
// position num_samples - 1 - k of return r, k < per_return.
__global__ void k_ins3_misses(const int* __restrict__ cells, int n, int per_return, int ox,
                              int oy, int oz, int num_free_space_voxels, Box3 box, uint16_t* vol,
                              const uint16_t* __restrict__ miss_table, unsigned long long* list,
                              unsigned long long* count) {
  const long long total = static_cast<long long>(n) * per_return;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(t / per_return), k = static_cast<int>(t % per_return);
    const int dx = cells[3 * r] - ox, dy = cells[3 * r + 1] - oy, dz = cells[3 * r + 2] - oz;
    const int num_samples = max(abs(dx), max(abs(dy), abs(dz)));
    const int position = num_samples - 1 - k;
    if (position < max(0, num_samples - num_free_space_voxels)) continue;
    // origin_cell + delta * position / num_samples: truncating integer division per axis
    const unsigned long long idx =
        box.Index(ox + dx * position / num_samples, oy + dy * position / num_samples,
                 oz + dz * position / num_samples);
    if (ApplyTable(vol + idx, miss_table)) Touched(idx, list, count);
  }
}

// FinishUpdate: the listed cells are distinct, but neighbouring 16-bit cells share a word.
__global__ void k_ins3_finish(const unsigned long long* __restrict__ list,
                              const unsigned long long* __restrict__ count, uint16_t* vol) {
  const unsigned long long m = *count;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
       i < m; i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    ClearUpdateMarker(vol, list[i]);
  }
}

__global__ void k_ins3_intensity_keys(const int* __restrict__ cells, int m, Box3 box,
                                      unsigned* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  keys[i] = static_cast<unsigned>(box.Index(cells[3 * i], cells[3 * i + 1], cells[3 * i + 2]));
}

// One thread per run of equal voxels of the sorted pairs: AddIntensity in return order.
__global__ void k_ins3_intensity_runs(const unsigned* __restrict__ keys,
                                      const float* __restrict__ values, int m, float* sum,
                                      int32_t* count, float* mean) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m || (i > 0 && keys[i] == keys[i - 1])) return;
  const unsigned k = keys[i];
  float s = sum[k];
  int c = count[k];
  for (int j = i; j < m && keys[j] == k; ++j) {
    s = __fadd_rn(s, values[j]);
    ++c;
  }
  sum[k] = s;
  count[k] = c;
  mean[k] = __fdiv_rn(s, __int2float_rn(c));
}

}  // namespace csm

using namespace csm;

namespace {

// HybridGridBase::GetCellIndex (hybrid_grid.h:428-433); false outside the 2^14 cube
// (hybrid_grid.h:387) or for a non-finite point.
bool CellIndex(const float* p, float resolution, int* cell) {
  for (int a = 0; a < 3; ++a) {
    const float q = p[a] / resolution;
    if (!(q > -kCube - 0.5f && q < kCube - 0.5f)) return false;
    cell[a] = static_cast<int>(std::lround(q));
  }
  return true;
}

}  // namespace

extern "C" {

csm_status csm_range_inserter3d_create(const csm_range_inserter_options3d* options,
                                       int32_t device, csm_range_inserter3d** out) {
  CSM_REQUIRE(options && out, "null pointer");
  // RangeDataInserter3D's CHECK_GT / CHECK_LT (range_data_inserter_3d.cc:66-67); beyond them,
  // a hit probability of 1 or a negative miss probability would make NaN / negative odds
  CSM_REQUIRE(options->hit_probability > 0.5 && options->hit_probability < 1.0, "hit_probability");
  CSM_REQUIRE(options->miss_probability < 0.5 && options->miss_probability >= 0.0,
              "miss_probability");
  CSM_REQUIRE(options->num_free_space_voxels >= 0, "num_free_space_voxels");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_range_inserter3d> ins(new csm_range_inserter3d);
  ins->ctx = ctx;
  ins->options = *options;
  // Odds(options_.hit_probability()): the double option enters Odds(float)
  std::vector<uint16_t> tables(2 * kValueCount);
  ComputeLookupTableToApplyOdds(Odds(static_cast<float>(options->hit_probability)), tables.data());
  ComputeLookupTableToApplyOdds(Odds(static_cast<float>(options->miss_probability)),
                                tables.data() + kValueCount);
  CSM_CUDA(cudaMalloc(&ins->d_tables, tables.size() * sizeof(uint16_t)));
  CSM_CUDA(cudaMemcpy(ins->d_tables, tables.data(), tables.size() * sizeof(uint16_t),
                      cudaMemcpyHostToDevice));
  *out = ins.release();
  return CSM_OK;
}

csm_status csm_range_inserter3d_destroy(csm_range_inserter3d* inserter) {
  if (!inserter) return CSM_OK;
  std::lock_guard<std::mutex> lock(inserter->ctx->mu);
  cudaSetDevice(inserter->ctx->device);
  cudaStreamSynchronize(inserter->ctx->stream);
  delete inserter;
  return CSM_OK;
}

csm_status csm_range_inserter3d_insert(const csm_range_inserter3d* inserter,
                                       const float origin[3], const float* returns,
                                       const float* intensities, int32_t num_returns,
                                       csm_grid3d* grid, csm_intensity_grid3d* intensity_grid,
                                       csm_stats* stats) {
  CSM_REQUIRE(inserter && origin && grid, "null pointer");
  CSM_REQUIRE(num_returns >= 0 && (num_returns == 0 || returns), "returns");
  Ctx* ctx = inserter->ctx;
  CSM_REQUIRE(grid->ctx == ctx, "grid on another device than the inserter");
  CSM_REQUIRE(!intensity_grid || intensity_grid->ctx == ctx,
              "intensity grid on another device than the inserter");
  const int n = num_returns;
  const int nfsv = inserter->options.num_free_space_voxels;
  std::lock_guard<std::mutex> lock(ctx->mu);
  // ---- every cell, and every check, before anything changes ----
  int origin_cell[3];
  CSM_REQUIRE(CellIndex(origin, grid->g.resolution, origin_cell),
              "origin cell outside the 2^14 cube");
  std::vector<int> cells(3 * static_cast<size_t>(n));
  TightBox3 need = grid->tight;
  int max_samples = 0;
  for (int i = 0; i < n; ++i) {
    int* c = &cells[3 * static_cast<size_t>(i)];
    CSM_REQUIRE(CellIndex(returns + 3 * static_cast<size_t>(i), grid->g.resolution, c),
                "hit cell outside the 2^14 cube");
    const int num_samples = std::max(std::abs(c[0] - origin_cell[0]),
                                     std::max(std::abs(c[1] - origin_cell[1]),
                                              std::abs(c[2] - origin_cell[2])));
    CSM_REQUIRE(num_samples < (1 << 15), "num_samples");   // range_data_inserter_3d.cc:38
    max_samples = std::max(max_samples, num_samples);
    need.Include(c);
  }
  // every miss cell lies between the origin cell and a hit cell
  if (n > 0) need.Include(origin_cell);
  const bool with_intensity = intensity_grid != nullptr && intensities != nullptr;
  std::vector<int> icells;
  std::vector<float> ivalues;
  TightBox3 ineed;
  if (with_intensity) {
    ineed = intensity_grid->tight;
    const float threshold = inserter->options.intensity_threshold;
    for (int i = 0; i < n; ++i) {
      if (intensities[i] > threshold) continue;   // InsertIntensitiesIntoGrid (:57-59)
      int c[3];
      CSM_REQUIRE(CellIndex(returns + 3 * static_cast<size_t>(i), intensity_grid->resolution, c),
                  "intensity cell outside the 2^14 cube");
      icells.insert(icells.end(), c, c + 3);
      ivalues.push_back(intensities[i]);
      ineed.Include(c);
    }
  }
  const int m = static_cast<int>(ivalues.size());
  GridInsert3 tx(grid, with_intensity ? intensity_grid : nullptr);
  CSM_TRY(tx.Grow(need, ineed));
  CSM_TRY(tx.Begin());
  cudaStream_t s = ctx->stream;
  // ---- upload: hit cells | intensity cells | intensities ----
  const size_t o_icell = (sizeof(int) * 3 * static_cast<size_t>(n) + 255) / 256 * 256;
  const size_t o_ival = o_icell + (sizeof(int) * 3 * static_cast<size_t>(m) + 255) / 256 * 256;
  const size_t bytes = o_ival + sizeof(float) * static_cast<size_t>(m);
  if (n > 0) {
    PinnedBuf& up = ctx->P("ins3_upload");
    DevBuf& d_up = ctx->D("ins3_upload");
    CSM_TRY(up.Reserve(bytes));
    CSM_TRY(d_up.Reserve(bytes));
    char* h = up.as<char>();
    std::memcpy(h, cells.data(), sizeof(int) * cells.size());
    std::memcpy(h + o_icell, icells.data(), sizeof(int) * icells.size());
    std::memcpy(h + o_ival, ivalues.data(), sizeof(float) * ivalues.size());
    CSM_CUDA(cudaMemcpyAsync(d_up.p, h, bytes, cudaMemcpyHostToDevice, s));
    const char* d = d_up.as<char>();
    const int* d_cells = reinterpret_cast<const int*>(d);
    // ---- occupancy: hits, misses, FinishUpdate ----
    const int per_return = std::min(nfsv, max_samples);
    const unsigned long long list_cap = std::min<unsigned long long>(
        static_cast<unsigned long long>(n) * (per_return + 1), tx.box.Volume());
    DevBuf& d_list = ctx->D("ins3_touched");
    CSM_TRY(d_list.Reserve(sizeof(unsigned long long) * (list_cap + 1)));
    unsigned long long* d_count = d_list.as<unsigned long long>();
    unsigned long long* d_touched = d_count + 1;
    CSM_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), s));
    const uint16_t* hit_table = inserter->d_tables;
    const uint16_t* miss_table = inserter->d_tables + kValueCount;
    ProfBegin(ctx);
    k_ins3_hits<<<Blocks(n, 1LL << 30), 256, 0, s>>>(d_cells, n, tx.box, tx.vol, hit_table,
                                                    d_touched, d_count);
    CSM_LAUNCH_CHECK();
    ProfEnd(ctx, "k_ins3_hits", n);
    if (per_return > 0) {
      ProfBegin(ctx);
      k_ins3_misses<<<Blocks(static_cast<long long>(n) * per_return), 256, 0, s>>>(
          d_cells, n, per_return, origin_cell[0], origin_cell[1], origin_cell[2], nfsv, tx.box,
          tx.vol, miss_table, d_touched, d_count);
      CSM_LAUNCH_CHECK();
      ProfEnd(ctx, "k_ins3_misses", static_cast<double>(n) * per_return);
    }
    ProfBegin(ctx);
    k_ins3_finish<<<Blocks(static_cast<long long>(list_cap)), 256, 0, s>>>(d_touched, d_count,
                                                                         tx.vol);
    CSM_LAUNCH_CHECK();
    ProfEnd(ctx, "k_ins3_finish", static_cast<double>(list_cap));
    // ---- intensities ----
    if (m > 0) {
      const int* d_icells = reinterpret_cast<const int*>(d + o_icell);
      const float* d_ivals = reinterpret_cast<const float*>(d + o_ival);
      int end_bit = 1;
      while (end_bit < 32 && (tx.ibox.Volume() - 1) >> end_bit) ++end_bit;
      size_t temp_bytes = 0;
      CSM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, static_cast<unsigned*>(nullptr),
                                               static_cast<unsigned*>(nullptr),
                                               static_cast<float*>(nullptr),
                                               static_cast<float*>(nullptr), m, 0, end_bit, s));
      const size_t o_kout = (sizeof(unsigned) * m + 255) / 256 * 256;
      const size_t o_vout = o_kout + o_kout;
      const size_t o_temp = o_vout + (sizeof(float) * m + 255) / 256 * 256;
      DevBuf& d_sort = ctx->D("ins3_sort");
      CSM_TRY(d_sort.Reserve(o_temp + temp_bytes));
      char* w = d_sort.as<char>();
      unsigned* keys = reinterpret_cast<unsigned*>(w);
      unsigned* keys_sorted = reinterpret_cast<unsigned*>(w + o_kout);
      float* vals_sorted = reinterpret_cast<float*>(w + o_vout);
      ProfBegin(ctx);
      k_ins3_intensity_keys<<<Blocks(m, 1LL << 30), 256, 0, s>>>(d_icells, m, tx.ibox, keys);
      CSM_LAUNCH_CHECK();
      CSM_CUDA(cub::DeviceRadixSort::SortPairs(w + o_temp, temp_bytes, keys, keys_sorted, d_ivals,
                                               vals_sorted, m, 0, end_bit, s));
      g_launches.fetch_add(1, std::memory_order_relaxed);
      k_ins3_intensity_runs<<<Blocks(m, 1LL << 30), 256, 0, s>>>(
          keys_sorted, vals_sorted, m, tx.sum, tx.count, tx.mean);
      CSM_LAUNCH_CHECK();
      ProfEnd(ctx, "k_ins3_intensity", m);
    }
  }
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  tx.Commit(stats);
  return CSM_OK;
}

}  // extern "C"
