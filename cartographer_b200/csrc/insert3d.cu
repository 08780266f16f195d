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
//
// csm_range_inserter3d_insert_submaps is Submap3D::InsertData (submap_3d.cc:271-294) for every
// active submap at once: the scan is uploaded once and k_ins3_submap_cells, one thread per
// (submap, return), does on the device what the single-grid insert does on the host: the
// transform into the submap frame, the high-resolution range filter, the cells, the checks and
// the boxes.  A stable compaction keeps the filtered returns and the intensity pairs in return
// order; after one small read-back the same hit, miss, finish and intensity kernels run per handle.
#include <algorithm>
#include <climits>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "grid3d.cuh"
#include "rigid3f.h"
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

// One entry of csm_range_inserter3d_insert_submaps as k_ins3_submap_cells reads it.
struct SubmapEntry3 {
  Rigid3f inverse;       // local_pose().inverse().cast<float>()
  float resolution[3];   // of the handles kHigh, kLow, kIntensity
  int with_intensity;
};
enum { kHigh = 0, kLow = 1, kIntensity = 2 };
enum { kFlagCell = 1, kFlagSamples = 2 };

// What k_ins3_submap_cells finds for one entry, read back before any handle changes.  lo / hi:
// the box of the handle's cells in this scan (origin excluded), count: how many there are.
struct SubmapScan3 {
  int flags;
  int origin_cell[2][3];   // kHigh, kLow
  int lo[3][3], hi[3][3];
  int count[3];
  int max_samples[2];
};

// CellIndex below, on the device: the same float quotient, in-cube test and rounding.
__device__ __forceinline__ bool DeviceCellIndex(const Vec3f& p, float resolution, int* cell) {
  const float v[3] = {p.x, p.y, p.z};
  bool ok = true;
  for (int a = 0; a < 3; ++a) {
    const float q = FDiv(v[a], resolution);
    ok = ok && q > -kCube - 0.5f && q < kCube - 0.5f;
    cell[a] = ok ? static_cast<int>(lroundf(q)) : 0;
  }
  return ok;
}

// Adds the cells of the lanes with `on` to handle h's box and count (whole warps call it).
__device__ __forceinline__ void WarpBox(SubmapScan3* r, int h, bool on, const int* c) {
  const unsigned lanes = __ballot_sync(~0u, on);
  if (lanes == 0) return;
  const bool leader = (threadIdx.x & 31) == 0;
  for (int a = 0; a < 3; ++a) {
    const int mn = __reduce_min_sync(~0u, on ? c[a] : INT_MAX);
    const int mx = __reduce_max_sync(~0u, on ? c[a] : INT_MIN);
    if (leader) {
      atomicMin(&r->lo[h][a], mn);
      atomicMax(&r->hi[h][a], mx);
    }
  }
  if (leader) atomicAdd(&r->count[h], __popc(lanes));
}

__device__ __forceinline__ int NumSamples(const int* c, const int* o) {
  return max(abs(c[0] - o[0]), max(abs(c[1] - o[1]), abs(c[2] - o[2])));
}

// Thread (e = blockIdx.y, i) of Submap3D::InsertData for entry e and return i: return i and the
// origin in the submap frame (TransformRangeData), the range filter (FilterRangeDataByMaxRange,
// submap_3d.cc:41-49, in FilterByMaxRange's evaluation order), the cells of the three handles,
// their checks and boxes.  Per flat index j = e * n + i: the low-resolution cell at low_cells
// [3 j], the high-resolution and intensity cells at high_all / intensity_all [3 j], and
// keep[j] = kept | with-intensity << 32 for the compaction.  Threads i >= n only check the
// origin (every entry has at least one block).
__global__ void k_ins3_submap_cells(const float* __restrict__ returns,
                                    const float* __restrict__ intensities, int n, Vec3f origin,
                                    float max_range, float threshold,
                                    const SubmapEntry3* __restrict__ entries, SubmapScan3* scans,
                                    int* __restrict__ low_cells, int* __restrict__ high_all,
                                    int* __restrict__ intensity_all,
                                    unsigned long long* __restrict__ keep) {
  const int e = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const SubmapEntry3& E = entries[e];
  SubmapScan3* r = scans + e;
  const bool valid = i < n;
  const Vec3f o = Rigid3Apply(E.inverse, origin);
  int oc[2][3];
  int flags = 0;
  const bool origin_ok = DeviceCellIndex(o, E.resolution[kHigh], oc[kHigh]) &
                         DeviceCellIndex(o, E.resolution[kLow], oc[kLow]);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int a = 0; a < 3; ++a) {
      r->origin_cell[kHigh][a] = oc[kHigh][a];
      r->origin_cell[kLow][a] = oc[kLow][a];
    }
    if (!origin_ok) flags |= kFlagCell;
  }
  Vec3f p = o;
  if (valid) p = Rigid3Apply(E.inverse, Vec3f{returns[3 * i], returns[3 * i + 1], returns[3 * i + 2]});
  const float dx = FSub(p.x, o.x), dy = FSub(p.y, o.y), dz = FSub(p.z, o.z);
  const bool kept =
      valid && FSqrt(FAdd(FAdd(FMul(dx, dx), FMul(dy, dy)), FMul(dz, dz))) <= max_range;
  int cl[3] = {0, 0, 0}, ch[3] = {0, 0, 0}, ci[3] = {0, 0, 0};
  bool low_on = false, high_on = false, intensity_on = false;
  int low_samples = 0, high_samples = 0;
  if (valid) {   // the low-resolution grid takes every return
    low_on = DeviceCellIndex(p, E.resolution[kLow], cl);
    if (!low_on) flags |= kFlagCell;
    if (low_on && origin_ok) low_samples = NumSamples(cl, oc[kLow]);
  }
  if (kept) {    // the high-resolution and intensity grids the filtered ones
    high_on = DeviceCellIndex(p, E.resolution[kHigh], ch);
    if (!high_on) flags |= kFlagCell;
    if (high_on && origin_ok) high_samples = NumSamples(ch, oc[kHigh]);
    if (E.with_intensity && !(intensities[i] > threshold)) {   // InsertIntensitiesIntoGrid
      intensity_on = DeviceCellIndex(p, E.resolution[kIntensity], ci);
      if (!intensity_on) flags |= kFlagCell;
    }
  }
  if (max(low_samples, high_samples) >= (1 << 15)) flags |= kFlagSamples;   // :38
  if (valid) {
    const long long j = static_cast<long long>(e) * n + i;
    for (int a = 0; a < 3; ++a) {
      low_cells[3 * j + a] = cl[a];
      high_all[3 * j + a] = ch[a];
      intensity_all[3 * j + a] = ci[a];
    }
    keep[j] = static_cast<unsigned long long>(kept) |
              static_cast<unsigned long long>(intensity_on) << 32;
  }
  WarpBox(r, kHigh, high_on, ch);
  WarpBox(r, kLow, low_on, cl);
  WarpBox(r, kIntensity, intensity_on, ci);
  const int ms_high = __reduce_max_sync(~0u, high_samples);
  const int ms_low = __reduce_max_sync(~0u, low_samples);
  flags = __reduce_or_sync(~0u, flags);
  if ((threadIdx.x & 31) == 0) {
    if (ms_high > 0) atomicMax(&r->max_samples[kHigh], ms_high);
    if (ms_low > 0) atomicMax(&r->max_samples[kLow], ms_low);
    if (flags) atomicOr(&r->flags, flags);
  }
}

// The stable compaction: position[j] is the exclusive sum of keep, so the kept returns of all
// entries, and their intensity pairs, follow each other in (entry, return) order.
__global__ void k_ins3_submap_compact(const unsigned long long* __restrict__ keep,
                                      const unsigned long long* __restrict__ position,
                                      long long total, int n, const int* __restrict__ high_all,
                                      const int* __restrict__ intensity_all,
                                      const float* __restrict__ intensities,
                                      int* __restrict__ high_cells,
                                      int* __restrict__ intensity_cells,
                                      float* __restrict__ intensity_values) {
  for (long long j = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; j < total;
       j += static_cast<long long>(gridDim.x) * blockDim.x) {
    const unsigned long long k = keep[j], at = position[j];
    if (k & 1ull) {
      const unsigned long long h = at & 0xffffffffull;
      for (int a = 0; a < 3; ++a) high_cells[3 * h + a] = high_all[3 * j + a];
    }
    if (k >> 32) {
      const unsigned long long m = at >> 32;
      for (int a = 0; a < 3; ++a) intensity_cells[3 * m + a] = intensity_all[3 * j + a];
      intensity_values[m] = intensities[j % n];
    }
  }
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

// Queues RangeDataInserter3D::Insert's occupancy part for the n hit cells d_cells (device,
// {x, y, z} each) from origin_cell into tx's volume: hits, the last num_free_space_voxels
// samples of each ray, FinishUpdate.  max_samples: the largest num_samples of the cells.
csm_status QueueOccupancy3(const csm_range_inserter3d* inserter, const int* d_cells, int n,
                           const int* origin_cell, int max_samples, const GridInsert3& tx) {
  if (n == 0) return CSM_OK;
  Ctx* ctx = inserter->ctx;
  cudaStream_t s = ctx->stream;
  const int nfsv = inserter->options.num_free_space_voxels;
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
  return CSM_OK;
}

// Queues InsertIntensitiesIntoGrid for the m (cell, intensity) pairs d_icells / d_ivals (device,
// in return order) into tx's intensity volumes.
csm_status QueueIntensities3(Ctx* ctx, const int* d_icells, const float* d_ivals, int m,
                             const GridInsert3& tx) {
  if (m == 0) return CSM_OK;
  cudaStream_t s = ctx->stream;
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
  k_ins3_intensity_runs<<<Blocks(m, 1LL << 30), 256, 0, s>>>(keys_sorted, vals_sorted, m, tx.sum,
                                                            tx.count, tx.mean);
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, "k_ins3_intensity", m);
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
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  GridInsert3 tx(grid, with_intensity ? intensity_grid : nullptr);
  CSM_TRY(tx.Grow(need, ineed));
  CSM_TRY(tx.Begin());
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
    CSM_TRY(QueueOccupancy3(inserter, reinterpret_cast<const int*>(d), n, origin_cell,
                            max_samples, tx));
    CSM_TRY(QueueIntensities3(ctx, reinterpret_cast<const int*>(d + o_icell),
                              reinterpret_cast<const float*>(d + o_ival), m, tx));
  }
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  tx.Commit(stats);
  return CSM_OK;
}

csm_status csm_range_inserter3d_insert_submaps(const csm_range_inserter3d* inserter,
                                               const csm_submap_insert3d* submaps,
                                               int32_t num_submaps, const float origin[3],
                                               const float* returns, const float* intensities,
                                               int32_t num_returns,
                                               float high_resolution_max_range,
                                               csm_stats* stats) {
  CSM_REQUIRE(inserter && submaps && origin, "null pointer");
  CSM_REQUIRE(num_submaps >= 1 && num_submaps <= 65535, "num_submaps");
  CSM_REQUIRE(num_returns >= 0 && (num_returns == 0 || returns), "returns");
  const int E = num_submaps, n = num_returns;
  CSM_REQUIRE(static_cast<long long>(E) * n < (1LL << 31), "num_submaps * num_returns");
  Ctx* ctx = inserter->ctx;
  std::vector<const void*> handles;
  for (int e = 0; e < E; ++e) {
    const csm_submap_insert3d& sub = submaps[e];
    CSM_REQUIRE(sub.high_resolution && sub.low_resolution, "null grid");
    CSM_REQUIRE(sub.high_resolution->ctx == ctx && sub.low_resolution->ctx == ctx &&
                    (!sub.intensity || sub.intensity->ctx == ctx),
                "grid on another device than the inserter");
    handles.push_back(sub.high_resolution);
    handles.push_back(sub.low_resolution);
    if (sub.intensity) handles.push_back(sub.intensity);
  }
  std::sort(handles.begin(), handles.end());
  CSM_REQUIRE(std::adjacent_find(handles.begin(), handles.end()) == handles.end(),
              "a handle appears twice");
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  // ---- upload: returns | intensities | entries | zeroed scans ----
  const bool with_intensity = intensities != nullptr;
  auto up256 = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t o_inten = up256(sizeof(float) * 3 * static_cast<size_t>(n));
  const size_t o_entry = o_inten + (with_intensity ? up256(sizeof(float) * n) : 0);
  const size_t o_scan = o_entry + up256(sizeof(SubmapEntry3) * E);
  const size_t up_bytes = o_scan + sizeof(SubmapScan3) * E;
  PinnedBuf& up = ctx->P("ins3s_upload");
  DevBuf& d_up = ctx->D("ins3s_upload");
  PinnedBuf& back = ctx->P("ins3s_scans");
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(d_up.Reserve(up_bytes));
  CSM_TRY(back.Reserve(sizeof(SubmapScan3) * E));
  char* h = up.as<char>();
  if (n > 0) std::memcpy(h, returns, sizeof(float) * 3 * n);
  if (with_intensity && n > 0) std::memcpy(h + o_inten, intensities, sizeof(float) * n);
  SubmapEntry3* entry = reinterpret_cast<SubmapEntry3*>(h + o_entry);
  SubmapScan3* scan0 = reinterpret_cast<SubmapScan3*>(h + o_scan);
  for (int e = 0; e < E; ++e) {
    const csm_submap_insert3d& sub = submaps[e];
    entry[e].inverse = Rigid3dInverseCast(sub.local_pose);
    entry[e].resolution[kHigh] = sub.high_resolution->g.resolution;
    entry[e].resolution[kLow] = sub.low_resolution->g.resolution;
    entry[e].resolution[kIntensity] = sub.intensity ? sub.intensity->resolution : 1.f;
    entry[e].with_intensity = with_intensity && sub.intensity != nullptr;
    SubmapScan3& z = scan0[e];
    std::memset(&z, 0, sizeof(z));
    for (int k = 0; k < 3; ++k)
      for (int a = 0; a < 3; ++a) {
        z.lo[k][a] = INT_MAX;
        z.hi[k][a] = INT_MIN;
      }
  }
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_CUDA(cudaMemcpyAsync(d_up.p, h, up_bytes, cudaMemcpyHostToDevice, s));
  const char* d = d_up.as<char>();
  const float* d_returns = reinterpret_cast<const float*>(d);
  const float* d_inten = with_intensity ? reinterpret_cast<const float*>(d + o_inten) : nullptr;
  SubmapScan3* d_scans = reinterpret_cast<SubmapScan3*>(d_up.as<char>() + o_scan);
  // ---- cells, checks, boxes; the stable compaction ----
  const long long total = static_cast<long long>(E) * n;
  const size_t cells_bytes = up256(sizeof(int) * 3 * static_cast<size_t>(total));
  const size_t flags_bytes = up256(sizeof(unsigned long long) * static_cast<size_t>(total));
  size_t scan_temp = 0;
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_temp,
                                         static_cast<unsigned long long*>(nullptr),
                                         static_cast<unsigned long long*>(nullptr),
                                         static_cast<int>(std::max(1LL, total)), s));
  // low | high (all) | intensity (all) | high (kept) | intensity (kept) | intensity values |
  // keep | position | scan temp
  const size_t o_high_all = cells_bytes, o_int_all = 2 * cells_bytes,
               o_high = 3 * cells_bytes, o_int = 4 * cells_bytes, o_ival = 5 * cells_bytes;
  const size_t o_keep = o_ival + up256(sizeof(float) * static_cast<size_t>(total));
  const size_t o_pos = o_keep + flags_bytes, o_temp = o_pos + flags_bytes;
  DevBuf& d_work = ctx->D("ins3s_work");
  CSM_TRY(d_work.Reserve(o_temp + scan_temp));
  char* w = d_work.as<char>();
  int* d_low = reinterpret_cast<int*>(w);
  int* d_high = reinterpret_cast<int*>(w + o_high);
  int* d_icells = reinterpret_cast<int*>(w + o_int);
  float* d_ivals = reinterpret_cast<float*>(w + o_ival);
  unsigned long long* d_keep = reinterpret_cast<unsigned long long*>(w + o_keep);
  unsigned long long* d_pos = reinterpret_cast<unsigned long long*>(w + o_pos);
  const Vec3f org{origin[0], origin[1], origin[2]};
  ProfBegin(ctx);
  k_ins3_submap_cells<<<dim3(Blocks(std::max(n, 1), 1LL << 30), E), 256, 0, s>>>(
      d_returns, d_inten, n, org, high_resolution_max_range,
      inserter->options.intensity_threshold, reinterpret_cast<const SubmapEntry3*>(d + o_entry),
      d_scans, d_low, reinterpret_cast<int*>(w + o_high_all), reinterpret_cast<int*>(w + o_int_all),
      d_keep);
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, "k_ins3_submap_cells", static_cast<double>(total));
  if (total > 0) {
    CSM_CUDA(cub::DeviceScan::ExclusiveSum(w + o_temp, scan_temp, d_keep, d_pos,
                                           static_cast<int>(total), s));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    ProfBegin(ctx);
    k_ins3_submap_compact<<<Blocks(total), 256, 0, s>>>(
        d_keep, d_pos, total, n, reinterpret_cast<const int*>(w + o_high_all),
        reinterpret_cast<const int*>(w + o_int_all), d_inten, d_high, d_icells, d_ivals);
    CSM_LAUNCH_CHECK();
    ProfEnd(ctx, "k_ins3_submap_compact", static_cast<double>(total));
  }
  SubmapScan3* scans = back.as<SubmapScan3>();
  CSM_CUDA(cudaMemcpyAsync(scans, d_scans, sizeof(SubmapScan3) * E, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  for (int e = 0; e < E; ++e) {
    CSM_REQUIRE(!(scans[e].flags & kFlagCell),
                "origin, hit or intensity cell outside the 2^14 cube, or a non-finite point");
    CSM_REQUIRE(!(scans[e].flags & kFlagSamples), "num_samples");
  }
  // ---- one transaction over every handle: grow all, then begin all ----
  auto call_box = [](const SubmapScan3& sc, int k, TightBox3* t) {
    if (sc.count[k] == 0) return;
    t->Include(sc.lo[k]);
    t->Include(sc.hi[k]);
  };
  std::vector<std::unique_ptr<GridInsert3>> txs;   // entry e: 2 e (high), 2 e + 1 (low)
  for (int e = 0; e < E; ++e) {
    const csm_submap_insert3d& sub = submaps[e];
    const SubmapScan3& sc = scans[e];
    csm_intensity_grid3d* ig = entry[e].with_intensity ? sub.intensity : nullptr;
    TightBox3 need = sub.high_resolution->tight, ineed;
    call_box(sc, kHigh, &need);
    if (sc.count[kHigh] > 0) need.Include(sc.origin_cell[kHigh]);   // the n > 0 rule, per handle
    if (ig) {
      ineed = ig->tight;
      call_box(sc, kIntensity, &ineed);
    }
    txs.emplace_back(new GridInsert3(sub.high_resolution, ig));
    CSM_TRY(txs.back()->Grow(need, ineed));
    TightBox3 low_need = sub.low_resolution->tight;
    call_box(sc, kLow, &low_need);
    if (sc.count[kLow] > 0) low_need.Include(sc.origin_cell[kLow]);
    txs.emplace_back(new GridInsert3(sub.low_resolution, nullptr));
    CSM_TRY(txs.back()->Grow(low_need, TightBox3()));
  }
  for (auto& tx : txs) CSM_TRY(tx->Begin());
  // ---- the single-grid insert's kernels, per handle, on the device-resident cells ----
  int high_base = 0, intensity_base = 0;
  for (int e = 0; e < E; ++e) {
    const SubmapScan3& sc = scans[e];
    GridInsert3& high = *txs[2 * e];
    GridInsert3& low = *txs[2 * e + 1];
    CSM_TRY(QueueOccupancy3(inserter, d_high + 3 * static_cast<size_t>(high_base),
                            sc.count[kHigh], sc.origin_cell[kHigh], sc.max_samples[kHigh], high));
    CSM_TRY(QueueOccupancy3(inserter, d_low + 3 * static_cast<size_t>(e) * n, n,
                            sc.origin_cell[kLow], sc.max_samples[kLow], low));
    if (entry[e].with_intensity)
      CSM_TRY(QueueIntensities3(ctx, d_icells + 3 * static_cast<size_t>(intensity_base),
                                d_ivals + intensity_base, sc.count[kIntensity], high));
    high_base += sc.count[kHigh];
    intensity_base += sc.count[kIntensity];
  }
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  for (auto& tx : txs) tx->Commit(nullptr);
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 2;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

}  // extern "C"
