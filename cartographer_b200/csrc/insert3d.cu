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

struct Box3 {
  int lo[3];
  int n[3];
};

__device__ __forceinline__ unsigned long long BoxIndex(const Box3& b, int x, int y, int z) {
  return (static_cast<unsigned long long>(z - b.lo[2]) * b.n[1] + (y - b.lo[1])) * b.n[0] +
         (x - b.lo[0]);
}

__device__ __forceinline__ void Touched(unsigned long long idx, unsigned long long* list,
                                        unsigned long long* count) {
  list[atomicAdd(count, 1ull)] = idx;
}

__global__ void k_ins3_hits(const int* __restrict__ cells, int n, Box3 box, uint16_t* vol,
                            const uint16_t* __restrict__ hit_table, unsigned long long* list,
                            unsigned long long* count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long idx = BoxIndex(box, cells[3 * i], cells[3 * i + 1], cells[3 * i + 2]);
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
        BoxIndex(box, ox + dx * position / num_samples, oy + dy * position / num_samples,
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
  keys[i] = static_cast<unsigned>(BoxIndex(box, cells[3 * i], cells[3 * i + 1], cells[3 * i + 2]));
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

// Copies the part of box `from` that lies in box `to` (`to` already zero-filled).
template <typename T>
__global__ void k_ins3_copy(const T* __restrict__ src, Box3 from, T* __restrict__ dst, Box3 to) {
  const unsigned long long total =
      static_cast<unsigned long long>(from.n[0]) * from.n[1] * from.n[2];
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
       i < total; i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const int x = from.lo[0] + static_cast<int>(i % from.n[0]);
    const int y = from.lo[1] + static_cast<int>(i / from.n[0] % from.n[1]);
    const int z = from.lo[2] + static_cast<int>(i / (static_cast<unsigned long long>(from.n[0]) * from.n[1]));
    if (x < to.lo[0] || x >= to.lo[0] + to.n[0] || y < to.lo[1] || y >= to.lo[1] + to.n[1] ||
        z < to.lo[2] || z >= to.lo[2] + to.n[2])
      continue;
    dst[BoxIndex(to, x, y, z)] = src[i];
  }
}

__global__ void k_ins3_scatter_made(const int* __restrict__ idx, const float* __restrict__ s,
                                    const int32_t* __restrict__ c, long long m, Box3 box,
                                    float* sum, int32_t* count) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= m) return;
  const unsigned long long k = BoxIndex(box, idx[3 * i], idx[3 * i + 1], idx[3 * i + 2]);
  sum[k] = s[i];
  count[k] = c[i];
}

}  // namespace csm

using namespace csm;

namespace {

// HybridGridBase::GetCellIndex (hybrid_grid.h:428-433); false outside the 2^14 cube
// (hybrid_grid.h:387) or for a non-finite point.
bool CellIndex(const float* p, float resolution, int* cell) {
  for (int a = 0; a < 3; ++a) {
    const float q = p[a] / resolution;
    if (!(q > -8192.5f && q < 8191.5f)) return false;
    cell[a] = static_cast<int>(std::lround(q));
  }
  return true;
}

void Include(TightBox3* t, const int* c) {
  for (int a = 0; a < 3; ++a) {
    if (t->empty || c[a] < t->lo[a]) t->lo[a] = c[a];
    if (t->empty || c[a] > t->hi[a]) t->hi[a] = c[a];
  }
  t->empty = false;
}

bool Covers(const Box3& b, const TightBox3& t) {
  if (t.empty) return true;
  for (int a = 0; a < 3; ++a)
    if (t.lo[a] < b.lo[a] || t.hi[a] >= b.lo[a] + b.n[a]) return false;
  return true;
}

// The box a handle grows to (DESIGN §9): the tight box plus extent / 8 voxels on each side of
// every axis, inside the 2^14 cube — at most 1.25^3 < 2x the tight box's volume, and every
// regrowth extends some axis's tight extent by more than 1/8 since the last one.
Box3 SlackBox(const TightBox3& t) {
  Box3 b;
  for (int a = 0; a < 3; ++a) {
    const int s = (t.hi[a] - t.lo[a] + 1) / 8;
    b.lo[a] = std::max(-8192, t.lo[a] - s);
    b.n[a] = std::min(8191, t.hi[a] + s) - b.lo[a] + 1;
  }
  return b;
}

size_t Volume(const Box3& b) { return static_cast<size_t>(b.n[0]) * b.n[1] * b.n[2]; }

unsigned Blocks(long long work, long long cap = 1 << 16) {
  return static_cast<unsigned>(std::max(1LL, std::min(cap, (work + 255) / 256)));
}

// A zero-filled volume of box `to` holding what `old` held over box `from`.
template <typename T>
csm_status Regrow(T* old, const Box3& from, const Box3& to, cudaStream_t s, T** out) {
  const size_t bytes = std::max<size_t>((Volume(to) * sizeof(T) + 3) / 4 * 4, 256);
  T* p = nullptr;
  CSM_CUDA(cudaMalloc(&p, bytes));
  *out = p;
  CSM_CUDA(cudaMemsetAsync(p, 0, bytes, s));
  if (old) {
    k_ins3_copy<T><<<Blocks(static_cast<long long>(Volume(from))), 256, 0, s>>>(old, from, p, to);
    CSM_LAUNCH_CHECK();
  }
  return CSM_OK;
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
    Include(&need, c);
  }
  // every miss cell lies between the origin cell and a hit cell
  if (n > 0) Include(&need, origin_cell);
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
      Include(&ineed, c);
    }
  }
  const int m = static_cast<int>(ivalues.size());
  Box3 box, grown;
  std::copy(grid->g.lo, grid->g.lo + 3, box.lo);
  std::copy(grid->g.n, grid->g.n + 3, box.n);
  const bool grow = !Covers(box, need);
  if (grow) {
    grown = SlackBox(need);
    CSM_REQUIRE(Volume(grown) < (size_t(8) << 30), "dense volume too large");
  }
  Box3 ibox{}, igrown{};
  bool igrow = false;
  if (with_intensity) {
    std::copy(intensity_grid->lo, intensity_grid->lo + 3, ibox.lo);
    std::copy(intensity_grid->n, intensity_grid->n + 3, ibox.n);
    igrow = !Covers(ibox, ineed);
    if (igrow) {
      igrown = SlackBox(ineed);
      CSM_REQUIRE(Volume(igrown) < (size_t(4) << 30), "dense volume too large");
    }
  }

  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  std::vector<void*> retired;   // freed once the stream has passed the copies
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  // ---- growth ----
  if (grow) {
    uint16_t* p;
    CSM_TRY(Regrow<uint16_t>(grid->d_vol, box, grown, s, &p));
    retired.push_back(grid->d_vol);
    grid->d_vol = p;
    grid->g.p = p;
    std::copy(grown.lo, grown.lo + 3, grid->g.lo);
    std::copy(grown.n, grown.n + 3, grid->g.n);
    box = grown;
  }
  grid->tight = need;
  if (with_intensity) {
    csm_intensity_grid3d* ig = intensity_grid;
    if (!ig->d_sum) {   // first insert: the AverageIntensityData volumes of what it was made from
      CSM_TRY(Regrow<float>(nullptr, ibox, ibox, s, &ig->d_sum));
      CSM_TRY(Regrow<int32_t>(nullptr, ibox, ibox, s, &ig->d_count));
      const long long made = static_cast<long long>(ig->made_sum.size());
      if (made > 0) {
        DevBuf& d_made = ctx->D("ins3_made");
        const size_t o_sum = (sizeof(int) * 3 * made + 255) / 256 * 256;
        const size_t o_cnt = o_sum + (sizeof(float) * made + 255) / 256 * 256;
        CSM_TRY(d_made.Reserve(o_cnt + sizeof(int32_t) * made));
        char* d = d_made.as<char>();
        CSM_CUDA(cudaMemcpyAsync(d, ig->made_idx.data(), sizeof(int) * 3 * made,
                                 cudaMemcpyHostToDevice, s));
        CSM_CUDA(cudaMemcpyAsync(d + o_sum, ig->made_sum.data(), sizeof(float) * made,
                                 cudaMemcpyHostToDevice, s));
        CSM_CUDA(cudaMemcpyAsync(d + o_cnt, ig->made_count.data(), sizeof(int32_t) * made,
                                 cudaMemcpyHostToDevice, s));
        k_ins3_scatter_made<<<Blocks(made, 1LL << 30), 256, 0, s>>>(
            reinterpret_cast<const int*>(d), reinterpret_cast<const float*>(d + o_sum),
            reinterpret_cast<const int32_t*>(d + o_cnt), made, ibox, ig->d_sum, ig->d_count);
        CSM_LAUNCH_CHECK();
      }
    }
    if (igrow) {
      float *mean, *sum;
      int32_t* count;
      CSM_TRY(Regrow<float>(ig->d_vol, ibox, igrown, s, &mean));
      retired.push_back(ig->d_vol);
      ig->d_vol = mean;
      CSM_TRY(Regrow<float>(ig->d_sum, ibox, igrown, s, &sum));
      retired.push_back(ig->d_sum);
      ig->d_sum = sum;
      CSM_TRY(Regrow<int32_t>(ig->d_count, ibox, igrown, s, &count));
      retired.push_back(ig->d_count);
      ig->d_count = count;
      std::copy(igrown.lo, igrown.lo + 3, ig->lo);
      std::copy(igrown.n, igrown.n + 3, ig->n);
      ibox = igrown;
    }
    ig->tight = ineed;
  }
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
        static_cast<unsigned long long>(n) * (per_return + 1), Volume(box));
    DevBuf& d_list = ctx->D("ins3_touched");
    CSM_TRY(d_list.Reserve(sizeof(unsigned long long) * (list_cap + 1)));
    unsigned long long* d_count = d_list.as<unsigned long long>();
    unsigned long long* d_touched = d_count + 1;
    CSM_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned long long), s));
    const uint16_t* hit_table = inserter->d_tables;
    const uint16_t* miss_table = inserter->d_tables + kValueCount;
    ProfBegin(ctx);
    k_ins3_hits<<<Blocks(n, 1LL << 30), 256, 0, s>>>(d_cells, n, box, grid->d_vol, hit_table,
                                                    d_touched, d_count);
    CSM_LAUNCH_CHECK();
    ProfEnd(ctx, "k_ins3_hits", n);
    if (per_return > 0) {
      ProfBegin(ctx);
      k_ins3_misses<<<Blocks(static_cast<long long>(n) * per_return), 256, 0, s>>>(
          d_cells, n, per_return, origin_cell[0], origin_cell[1], origin_cell[2], nfsv, box,
          grid->d_vol, miss_table, d_touched, d_count);
      CSM_LAUNCH_CHECK();
      ProfEnd(ctx, "k_ins3_misses", static_cast<double>(n) * per_return);
    }
    ProfBegin(ctx);
    k_ins3_finish<<<Blocks(static_cast<long long>(list_cap)), 256, 0, s>>>(d_touched, d_count,
                                                                         grid->d_vol);
    CSM_LAUNCH_CHECK();
    ProfEnd(ctx, "k_ins3_finish", static_cast<double>(list_cap));
    // ---- intensities ----
    if (m > 0) {
      const int* d_icells = reinterpret_cast<const int*>(d + o_icell);
      const float* d_ivals = reinterpret_cast<const float*>(d + o_ival);
      int end_bit = 1;
      while (end_bit < 32 && (Volume(ibox) - 1) >> end_bit) ++end_bit;
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
      k_ins3_intensity_keys<<<Blocks(m, 1LL << 30), 256, 0, s>>>(d_icells, m, ibox, keys);
      CSM_LAUNCH_CHECK();
      CSM_CUDA(cub::DeviceRadixSort::SortPairs(w + o_temp, temp_bytes, keys, keys_sorted, d_ivals,
                                               vals_sorted, m, 0, end_bit, s));
      g_launches.fetch_add(1, std::memory_order_relaxed);
      k_ins3_intensity_runs<<<Blocks(m, 1LL << 30), 256, 0, s>>>(
          keys_sorted, vals_sorted, m, intensity_grid->d_sum, intensity_grid->d_count,
          intensity_grid->d_vol);
      CSM_LAUNCH_CHECK();
      ProfEnd(ctx, "k_ins3_intensity", m);
    }
  }
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  for (void* p : retired) CSM_CUDA(cudaFree(p));
  if (with_intensity && !intensity_grid->made_sum.empty()) {
    // the volumes hold it now
    std::vector<int32_t>().swap(intensity_grid->made_idx);
    std::vector<int32_t>().swap(intensity_grid->made_count);
    std::vector<float>().swap(intensity_grid->made_sum);
  }
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

csm_status csm_grid3d_read(const csm_grid3d* grid, int32_t lo[3], int32_t dims[3],
                           uint16_t* out) {
  CSM_REQUIRE(grid && lo && dims, "null pointer");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  for (int a = 0; a < 3; ++a) {
    lo[a] = grid->g.lo[a];
    dims[a] = grid->g.n[a];
  }
  if (!out) return CSM_OK;
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  const size_t vox = static_cast<size_t>(dims[0]) * dims[1] * dims[2];
  CSM_CUDA(cudaMemcpyAsync(out, grid->d_vol, vox * sizeof(uint16_t), cudaMemcpyDeviceToHost,
                           grid->ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(grid->ctx->stream));
  return CSM_OK;
}

csm_status csm_intensity_grid3d_read(const csm_intensity_grid3d* grid, int32_t lo[3],
                                     int32_t dims[3], float* mean, float* sum, int32_t* count) {
  CSM_REQUIRE(grid && lo && dims, "null pointer");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  for (int a = 0; a < 3; ++a) {
    lo[a] = grid->lo[a];
    dims[a] = grid->n[a];
  }
  if (!mean) return CSM_OK;
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  cudaStream_t s = grid->ctx->stream;
  const size_t vox = static_cast<size_t>(dims[0]) * dims[1] * dims[2];
  CSM_CUDA(cudaMemcpyAsync(mean, grid->d_vol, vox * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (grid->d_sum) {
    if (sum) CSM_CUDA(cudaMemcpyAsync(sum, grid->d_sum, vox * 4, cudaMemcpyDeviceToHost, s));
    if (count) CSM_CUDA(cudaMemcpyAsync(count, grid->d_count, vox * 4, cudaMemcpyDeviceToHost, s));
  } else {   // never inserted into: the list it was made from
    if (sum) std::fill(sum, sum + vox, 0.f);
    if (count) std::fill(count, count + vox, 0);
    for (size_t i = 0; i < grid->made_sum.size(); ++i) {
      const int* c = &grid->made_idx[3 * i];
      const size_t k = (static_cast<size_t>(c[2] - lo[2]) * dims[1] + (c[1] - lo[1])) * dims[0] +
                       (c[0] - lo[0]);
      if (sum) sum[k] = grid->made_sum[i];
      if (count) count[k] = grid->made_count[i];
    }
  }
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

}  // extern "C"
