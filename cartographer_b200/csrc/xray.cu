// io::XRayPointsProcessor (io/xray_points_processor.cc:170-239) on the device, bit for bit: the
// voxels, the column sums and counts, the shared bounding box and every pixel equal the
// reference's.
//
// The reference keeps per aggregation (one per floor) a HybridGridBase<bool> at resolution
// (float)voxel_size and a std::map<(y, z), ColumnData{float sum_r, sum_g, sum_b; uint32 count}>,
// and one bounding box over all of them.  Insert, per point in stream order:
//   p = transform * point (Rigid3f); index = lround(p / resolution) narrowed to int; the voxel is
//   set; the box extends; column (index.y, index.z) adds the colour (black without colours).
// On the device:
//   * one thread per point transforms (rigid3f.h) and rounds, reduces the call's index box and
//     flags an index outside [-8192, 8192)^3, the cube the reference's grid can grow to (its
//     CHECK).  The voxels and columns are only changed by the kernels after it, which return at
//     once when the flag is set, so a refused call changes nothing;
//   * the voxels go into an open-addressing set of 42-bit keys (atomicCAS): a set does not
//     depend on order;
//   * the column sums are sequential float sums, so (28-bit column key, list position) pairs are
//     sorted stably and one thread per run adds its colours in list order onto the column's
//     running sums: the same additions in the same order as the reference.
//   One stream synchronisation per call with points reads back the flag, the box and the voxel
//   and column counts; the next call sizes its growth (a device rehash that keeps both tables at
//   most half full) from those counts.
// Draw (WriteVoxels + IntoImage), per pixel: n = the number of voxels of its column (atomicAdd
// per voxel, order-free); max = max(FLT_MIN, (float)log(n_max)); saturation =
// (float)(log(n) / max * saturation_factor) capped at 1; per channel Mix(1.f, sum / count,
// saturation) with its double and float steps; then the cairo word.  log(n) comes from a table
// that the host fills with glibc's log, so the device never calls log.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "point_batch.cuh"
#include "rigid3f.h"

namespace {

constexpr long long kInitialSlots = 1 << 12;
constexpr int kThreads = 256;
constexpr int kColumnKeyBits = 28;

}  // namespace

namespace csm {

// ColumnData (io/xray_points_processor.h:62-67).
struct XRayColumn {
  float sum_r, sum_g, sum_b;
  unsigned count;
};

// The call block: the refusal flag and the call's index box {min x, y, z, max x, y, z}.
struct XRayCallBlock {
  int outside;
  int box[6];
  int pad;
};

struct XRayAggregation {
  unsigned long long* voxel_keys = nullptr;   // a set of packed voxel keys
  long long voxel_slots = 0;
  long long voxels = 0;                       // read back at the end of every call with points
  unsigned long long* column_keys = nullptr;  // column keys ((z + 8192) << 14 | (y + 8192))
  XRayColumn* columns = nullptr;
  long long column_slots = 0;
  long long num_columns = 0;
};

}  // namespace csm

struct csm_xray {
  csm::Ctx* ctx = nullptr;
  float resolution = 0;                       // HybridGridBase<bool>(voxel_size)
  double saturation_factor = 1;
  csm::Rigid3f transform{};
  std::vector<csm::XRayAggregation> aggregations;
  unsigned long long* d_counts = nullptr;     // per aggregation {voxels, columns}
  // the shared bounding box (Eigen::AlignedBox3i), kept on the host
  bool empty = true;
  int lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  std::vector<double> logs{0.0};              // logs[n] = std::log((double)n), n >= 1
  ~csm_xray() {
    for (csm::XRayAggregation& a : aggregations) {
      cudaFree(a.voxel_keys);
      cudaFree(a.column_keys);
      cudaFree(a.columns);
    }
    cudaFree(d_counts);
  }
};

namespace csm {
namespace {

__device__ inline unsigned ColumnKey(int y, int z) {
  return (static_cast<unsigned>(z + kCubeHalf) << 14) | static_cast<unsigned>(y + kCubeHalf);
}

// Per point: the transformed cell index, its voxel and column keys and its list position; the
// call's box and the refusal flag.
__global__ void k_xr_cells(const float* __restrict__ xyz, int n, Rigid3f transform,
                           float resolution, unsigned long long* voxel_keys,
                           unsigned* column_keys, int* positions, XRayCallBlock* block) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  bool outside = false;
  if (i < n) {
    const Vec3f p = Rigid3Apply(transform, Vec3f{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]});
    const int c[3] = {RoundToInt(FDiv(p.x, resolution)), RoundToInt(FDiv(p.y, resolution)),
                      RoundToInt(FDiv(p.z, resolution))};
    outside = !InCube(c[0]) || !InCube(c[1]) || !InCube(c[2]);
    for (int a = 0; a < 3; ++a) lo[a] = hi[a] = c[a];
    if (!outside) {
      voxel_keys[i] = Pack(c[0], c[1], c[2]);
      column_keys[i] = ColumnKey(c[1], c[2]);
    }
    positions[i] = i;
  }
  for (int a = 0; a < 3; ++a) {
    lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
    hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
  }
  const unsigned any_outside = __ballot_sync(0xffffffffu, outside);
  const unsigned any_point = __ballot_sync(0xffffffffu, i < n);
  if ((threadIdx.x & 31) == 0 && any_point) {
    for (int a = 0; a < 3; ++a) {
      atomicMin(&block->box[a], lo[a]);
      atomicMax(&block->box[3 + a], hi[a]);
    }
    if (any_outside) atomicOr(&block->outside, 1);
  }
}

// mutable_value(index) = true for every point of an accepted call.
__global__ void k_xr_voxels(const unsigned long long* __restrict__ voxel_keys, int n,
                            const XRayCallBlock* __restrict__ block, unsigned long long* keys,
                            unsigned long long mask, unsigned long long* count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || block->outside) return;
  bool inserted;
  Insert(keys, mask, voxel_keys[i], &inserted);
  if (inserted) atomicAdd(count, 1ull);
}

// One thread per run of equal column keys in the stably sorted list: the run's colours are
// added onto the column's sums in list (= stream) order, as column_data[...] += color does.
__global__ void k_xr_runs(const unsigned* __restrict__ sorted_keys,
                          const int* __restrict__ sorted_positions, int n,
                          const float* __restrict__ rgb, const XRayCallBlock* __restrict__ block,
                          unsigned long long* keys, XRayColumn* columns, unsigned long long mask,
                          unsigned long long* count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || block->outside) return;
  const unsigned key = sorted_keys[i];
  if (i > 0 && sorted_keys[i - 1] == key) return;
  bool inserted;
  const unsigned long long h = Insert(keys, mask, key, &inserted);
  if (inserted) atomicAdd(count, 1ull);
  XRayColumn c = columns[h];
  for (int j = i; j < n && sorted_keys[j] == key; ++j) {
    const float* color = rgb + 3 * sorted_positions[j];
    c.sum_r = __fadd_rn(c.sum_r, color[0]);
    c.sum_g = __fadd_rn(c.sum_g, color[1]);
    c.sum_b = __fadd_rn(c.sum_b, color[2]);
    ++c.count;
  }
  columns[h] = c;
}

// WriteVoxels' ++num_occupied_cells_in_column per voxel, and the largest count: the add that
// takes a pixel to its final count returns that count - 1, and no add returns more.
__global__ void k_xr_count(const unsigned long long* __restrict__ keys, long long slots,
                           int max_y, int max_z, int width, unsigned* counts, unsigned* max_count) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  unsigned top = 0;
  if (i < slots) {
    const unsigned long long k = keys[i];
    if (k != kEmptyKey) {
      const int y = static_cast<int>((k >> 14) & 0x3fff) - kCubeHalf;
      const int z = static_cast<int>(k >> 28) - kCubeHalf;
      top = atomicAdd(&counts[static_cast<long long>(max_z - z) * width + (max_y - y)], 1u) + 1;
    }
  }
  top = __reduce_max_sync(0xffffffffu, top);
  if ((threadIdx.x & 31) == 0 && top > 0) atomicMax(max_count, top);
}

// io/color.h FloatComponentToUint8: RoundToInt(Clamp(c, 0.f, 1.f) * 255), then uint8.
__device__ inline unsigned ToUint8(float c) {
  const float clamped = c > 1.f ? 1.f : (c < 0.f ? 0.f : c);
  return static_cast<unsigned>(RoundToInt(__fmul_rn(clamped, 255.f))) & 0xffu;
}

// Mix(1.f, b, t) = 1.f * (1. - t) + t * b: a double product plus a float product, in double,
// returned as float.
__device__ inline float MixFromWhite(float b, float t) {
  const double white = __dmul_rn(1.0, __dsub_rn(1.0, static_cast<double>(t)));
  return __double2float_rn(__dadd_rn(white, static_cast<double>(__fmul_rn(t, b))));
}

// IntoImage, one thread per pixel: the cairo word 0xFF << 24 | r << 16 | g << 8 | b.
__global__ void k_xr_pixels(const unsigned* __restrict__ counts, int width, long long num_pixels,
                            int max_y, int max_z, const unsigned* __restrict__ max_count,
                            const double* __restrict__ logs, double saturation_factor,
                            const unsigned long long* __restrict__ keys,
                            const XRayColumn* __restrict__ columns, unsigned long long mask,
                            unsigned* pixels) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= num_pixels) return;
  const unsigned n = counts[i];
  if (n == 0) {
    pixels[i] = 0xffffffffu;
    return;
  }
  // float max = FLT_MIN; max = std::max<float>(max, std::log(n)) over the pixels with n > 0
  const float top = __double2float_rn(logs[*max_count]);
  const float max = FLT_MIN < top ? top : FLT_MIN;
  // std::min<float>(1.0, std::log(n) / max * saturation_factor)
  const float s =
      __double2float_rn(__dmul_rn(__ddiv_rn(logs[n], static_cast<double>(max)), saturation_factor));
  const float saturation = s < 1.f ? s : 1.f;
  const int y = max_y - static_cast<int>(i % width);
  const int z = max_z - static_cast<int>(i / width);
  const XRayColumn c = columns[Find(keys, mask, ColumnKey(y, z))];
  const float count = __uint2float_rn(c.count);
  const unsigned r = ToUint8(MixFromWhite(__fdiv_rn(c.sum_r, count), saturation));
  const unsigned g = ToUint8(MixFromWhite(__fdiv_rn(c.sum_g, count), saturation));
  const unsigned b = ToUint8(MixFromWhite(__fdiv_rn(c.sum_b, count), saturation));
  pixels[i] = 0xff000000u | r << 16 | g << 8 | b;
}

csm_status CheckAggregation(const csm_xray* h, int32_t aggregation) {
  CSM_REQUIRE(aggregation >= 0 && aggregation < static_cast<int>(h->aggregations.size()),
              "aggregation out of range");
  return CSM_OK;
}

long long SlotsFor(long long current, long long entries) {
  long long slots = std::max(current, kInitialSlots);
  while (2 * entries > slots) slots *= 2;
  return slots;
}

// A table of `slots` keys (all free) and, unless `value_bytes` is 0, zeroed values.
csm_status AllocTable(cudaStream_t s, long long slots, size_t value_bytes,
                      unsigned long long** keys, void** vals) {
  CSM_CUDA(cudaMallocAsync(keys, sizeof(unsigned long long) * slots, s));
  if (value_bytes && cudaMallocAsync(vals, value_bytes * slots, s) != cudaSuccess) {
    cudaFreeAsync(*keys, s);
    SetError("xray: cudaMallocAsync of %lld column slots failed", slots);
    return CSM_E_CAPACITY;
  }
  CSM_CUDA(cudaMemsetAsync(*keys, 0xff, sizeof(unsigned long long) * slots, s));
  if (value_bytes) CSM_CUDA(cudaMemsetAsync(*vals, 0, value_bytes * slots, s));
  return CSM_OK;
}

// Grows the aggregation's voxel set and column map (device rehash) so that `incoming` more
// entries keep each at most half full.  CSM_E_CAPACITY, with nothing changed, when the device
// has not the memory for both.
csm_status Reserve(csm_xray* h, XRayAggregation* a, long long incoming) {
  const long long vslots = SlotsFor(a->voxel_slots, a->voxels + incoming);
  const long long cslots = SlotsFor(a->column_slots, a->num_columns + incoming);
  const bool grow_v = vslots != a->voxel_slots, grow_c = cslots != a->column_slots;
  if (!grow_v && !grow_c) return CSM_OK;
  const size_t bytes =
      (grow_v ? static_cast<size_t>(vslots) * sizeof(unsigned long long) : 0) +
      (grow_c ? static_cast<size_t>(cslots) * (sizeof(unsigned long long) + sizeof(XRayColumn))
              : 0);
  size_t free_bytes = 0, total_bytes = 0;
  CSM_CUDA(cudaMemGetInfo(&free_bytes, &total_bytes));
  if (bytes > free_bytes) {
    SetError("xray: growing to %lld voxel and %lld column slots needs %zu bytes, %zu free",
             vslots, cslots, bytes, free_bytes);
    return CSM_E_CAPACITY;
  }
  cudaStream_t s = h->ctx->stream;
  unsigned long long *vkeys = nullptr, *ckeys = nullptr;
  void* cvals = nullptr;
  if (grow_v) CSM_TRY(AllocTable(s, vslots, 0, &vkeys, nullptr));
  if (grow_c) {
    const csm_status st = AllocTable(s, cslots, sizeof(XRayColumn), &ckeys, &cvals);
    if (st != CSM_OK) {
      if (vkeys) cudaFreeAsync(vkeys, s);
      return st;
    }
  }
  if (grow_v) {
    if (a->voxel_slots > 0) {
      k_rehash<NoValues><<<DivUp(a->voxel_slots, kThreads), kThreads, 0, s>>>(
          a->voxel_keys, nullptr, a->voxel_slots, vkeys, nullptr, vslots - 1);
      CSM_LAUNCH_CHECK();
      CSM_CUDA(cudaFreeAsync(a->voxel_keys, s));
    }
    a->voxel_keys = vkeys;
    a->voxel_slots = vslots;
  }
  if (grow_c) {
    XRayColumn* cols = static_cast<XRayColumn*>(cvals);
    if (a->column_slots > 0) {
      k_rehash<XRayColumn><<<DivUp(a->column_slots, kThreads), kThreads, 0, s>>>(
          a->column_keys, a->columns, a->column_slots, ckeys, cols, cslots - 1);
      CSM_LAUNCH_CHECK();
      CSM_CUDA(cudaFreeAsync(a->column_keys, s));
      CSM_CUDA(cudaFreeAsync(a->columns, s));
    }
    a->column_keys = ckeys;
    a->columns = cols;
    a->column_slots = cslots;
  }
  return CSM_OK;
}

void NoWork(csm_stats* stats) {
  if (stats) std::memset(stats, 0, sizeof(*stats));
}

// Host copies of a table's keys (and values), in slot order.
template <class V>
csm_status Download(Ctx* ctx, const unsigned long long* d_keys, const V* d_vals, long long slots,
                    std::vector<unsigned long long>* keys, std::vector<V>* vals) {
  keys->resize(slots);
  CSM_CUDA(cudaMemcpyAsync(keys->data(), d_keys, sizeof(unsigned long long) * slots,
                           cudaMemcpyDeviceToHost, ctx->stream));
  if (vals) {
    vals->resize(slots);
    CSM_CUDA(cudaMemcpyAsync(vals->data(), d_vals, sizeof(V) * slots, cudaMemcpyDeviceToHost,
                             ctx->stream));
  }
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  return CSM_OK;
}

}  // namespace
}  // namespace csm

using namespace csm;

extern "C" {

csm_status csm_xray_create(double voxel_size, double saturation_factor, const float transform[7],
                           int32_t num_aggregations, int32_t device, csm_xray** out) {
  CSM_REQUIRE(out && transform, "null pointer");
  CSM_REQUIRE(std::isfinite(voxel_size) && voxel_size > 0.0, "voxel_size");
  CSM_REQUIRE(std::isfinite(saturation_factor), "saturation_factor");
  CSM_REQUIRE(Finite(transform, 7), "non-finite transform");
  CSM_REQUIRE(num_aggregations >= 1, "num_aggregations");
  CSM_REQUIRE(static_cast<float>(voxel_size) > 0.f, "voxel_size rounds to 0 in float");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_xray> h(new csm_xray);
  h->ctx = ctx;
  h->resolution = static_cast<float>(voxel_size);
  h->saturation_factor = saturation_factor;
  h->transform = Rigid3f{Vec3f{transform[0], transform[1], transform[2]},
                         Quatf{transform[3], transform[4], transform[5], transform[6]}};
  h->aggregations.resize(num_aggregations);
  CSM_CUDA(cudaMalloc(&h->d_counts, sizeof(unsigned long long) * 2 * num_aggregations));
  CSM_CUDA(cudaMemsetAsync(h->d_counts, 0, sizeof(unsigned long long) * 2 * num_aggregations,
                           ctx->stream));
  for (XRayAggregation& a : h->aggregations) CSM_TRY(Reserve(h.get(), &a, 0));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = h.release();
  return CSM_OK;
}

csm_status csm_xray_destroy(csm_xray* h) {
  if (!h) return CSM_OK;
  std::lock_guard<std::mutex> lock(h->ctx->mu);
  cudaSetDevice(h->ctx->device);
  cudaStreamSynchronize(h->ctx->stream);
  delete h;
  return CSM_OK;
}

csm_status csm_xray_insert(csm_xray* h, int32_t aggregation, const float* const* xyz,
                           const float* const* rgb, const int32_t* num_points,
                           int32_t num_batches, csm_stats* stats) {
  CSM_REQUIRE(h, "null processor");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_TRY(CheckAggregation(h, aggregation));
  CSM_REQUIRE(num_batches >= 0, "num_batches");
  CSM_REQUIRE(num_batches == 0 || (xyz && num_points), "null pointer");
  long long total = 0;
  for (int b = 0; b < num_batches; ++b) {
    CSM_REQUIRE(num_points[b] >= 0, "negative point count");
    const size_t m = 3 * static_cast<size_t>(num_points[b]);
    CSM_REQUIRE(num_points[b] == 0 || xyz[b], "null batch");
    CSM_REQUIRE(Finite(xyz[b], m), "non-finite point");
    CSM_REQUIRE(!rgb || !rgb[b] || Finite(rgb[b], m), "non-finite colour");
    total += num_points[b];
    CSM_REQUIRE(total < (1ll << 30), "more than 2^30 points in one call");
  }
  CSM_CUDA(cudaSetDevice(ctx->device));
  const int n = static_cast<int>(total);
  if (n == 0) {
    NoWork(stats);
    return CSM_OK;
  }
  XRayAggregation* a = &h->aggregations[aggregation];
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_TRY(Reserve(h, a, n));
  size_t sort_bytes = 0;
  CSM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, static_cast<unsigned*>(nullptr),
                                           static_cast<unsigned*>(nullptr),
                                           static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                           n, 0, kColumnKeyBits, s));
  struct Work {
    XRayCallBlock* block;
    float* points;            // xyz (3n), then rgb (3n)
    unsigned long long* voxel_keys;
    unsigned* column_keys;
    unsigned* sorted_keys;
    int* positions;
    int* sorted_positions;
    void* temp;
  };
  auto lay = [&](Carver& w) {
    Work k;
    k.block = w.take<XRayCallBlock>(1);
    k.points = w.take<float>(6 * static_cast<size_t>(n));
    k.voxel_keys = w.take<unsigned long long>(n);
    k.column_keys = w.take<unsigned>(n);
    k.sorted_keys = w.take<unsigned>(n);
    k.positions = w.take<int>(n);
    k.sorted_positions = w.take<int>(n);
    k.temp = w.take<char>(sort_bytes);
    return k;
  };
  Carver sizer;
  lay(sizer);
  DevBuf& ws = ctx->D("xray");
  CSM_TRY(ws.Reserve(sizer.at));
  Carver carver;
  carver.base = ws.as<char>();
  const Work k = lay(carver);
  // the call block and the points and colours, as laid out on the device, in one copy
  const size_t o_points = reinterpret_cast<char*>(k.points) - reinterpret_cast<char*>(k.block);
  const size_t o_rgb = o_points + sizeof(float) * 3 * static_cast<size_t>(n);
  const size_t up_bytes = o_rgb + sizeof(float) * 3 * static_cast<size_t>(n);
  PinnedBuf& up = ctx->P("xray_up");
  CSM_TRY(up.Reserve(up_bytes));
  char* p = up.as<char>();
  const XRayCallBlock init{0, {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN}, 0};
  std::memcpy(p, &init, sizeof(init));
  size_t at = 0;
  for (int b = 0; b < num_batches; ++b) {
    const size_t m = sizeof(float) * 3 * static_cast<size_t>(num_points[b]);
    if (!m) continue;
    std::memcpy(p + o_points + at, xyz[b], m);
    if (rgb && rgb[b]) std::memcpy(p + o_rgb + at, rgb[b], m);
    else std::memset(p + o_rgb + at, 0, m);
    at += m;
  }
  CSM_CUDA(cudaMemcpyAsync(k.block, p, up_bytes, cudaMemcpyHostToDevice, s));
  const float* d_rgb = k.points + 3 * static_cast<size_t>(n);
  k_xr_cells<<<DivUp(n, kThreads), kThreads, 0, s>>>(k.points, n, h->transform, h->resolution,
                                                     k.voxel_keys, k.column_keys, k.positions,
                                                     k.block);
  CSM_LAUNCH_CHECK();
  unsigned long long* counts = h->d_counts + 2 * aggregation;
  k_xr_voxels<<<DivUp(n, kThreads), kThreads, 0, s>>>(k.voxel_keys, n, k.block, a->voxel_keys,
                                                      a->voxel_slots - 1, counts);
  CSM_LAUNCH_CHECK();
  size_t tb = sort_bytes;
  CSM_CUDA(cub::DeviceRadixSort::SortPairs(k.temp, tb, k.column_keys, k.sorted_keys, k.positions,
                                           k.sorted_positions, n, 0, kColumnKeyBits, s));
  k_xr_runs<<<DivUp(n, kThreads), kThreads, 0, s>>>(k.sorted_keys, k.sorted_positions, n, d_rgb,
                                                    k.block, a->column_keys, a->columns,
                                                    a->column_slots - 1, counts + 1);
  CSM_LAUNCH_CHECK();
  PinnedBuf& down = ctx->P("xray_down");
  CSM_TRY(down.Reserve(sizeof(XRayCallBlock) + 2 * sizeof(unsigned long long)));
  char* d = down.as<char>();
  CSM_CUDA(cudaMemcpyAsync(d, k.block, sizeof(XRayCallBlock), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(d + sizeof(XRayCallBlock), counts, 2 * sizeof(unsigned long long),
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  XRayCallBlock block;
  std::memcpy(&block, d, sizeof(block));
  if (block.outside) {
    SetError("xray: a point's cell lies outside the [-8192, 8192)^3 cells the grid can hold");
    return CSM_E_INVALID;
  }
  unsigned long long c[2];
  std::memcpy(c, d + sizeof(XRayCallBlock), sizeof(c));
  a->voxels = static_cast<long long>(c[0]);
  a->num_columns = static_cast<long long>(c[1]);
  for (int i = 0; i < 3; ++i) {
    h->lo[i] = h->empty ? block.box[i] : std::min(h->lo[i], block.box[i]);
    h->hi[i] = h->empty ? block.box[3 + i] : std::max(h->hi[i], block.box[3 + i]);
  }
  h->empty = false;
  return CSM_OK;
}

csm_status csm_xray_bounding_box(const csm_xray* h, int32_t min[3], int32_t max[3],
                                 int32_t* empty) {
  CSM_REQUIRE(h && min && max && empty, "null pointer");
  std::lock_guard<std::mutex> lock(h->ctx->mu);
  *empty = h->empty;
  for (int i = 0; i < 3; ++i) {
    min[i] = h->lo[i];
    max[i] = h->hi[i];
  }
  return CSM_OK;
}

csm_status csm_xray_draw(csm_xray* h, int32_t aggregation, uint32_t* pixels, int64_t capacity,
                         int32_t* width, int32_t* height, csm_stats* stats) {
  CSM_REQUIRE(h && width && height, "null pointer");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_TRY(CheckAggregation(h, aggregation));
  NoWork(stats);
  if (h->empty) {
    *width = *height = 0;
    return CSM_OK;
  }
  // the cube bounds every side by 16384, so the image has at most 2^28 pixels
  const int w = h->hi[1] - h->lo[1] + 1, ht = h->hi[2] - h->lo[2] + 1;
  *width = w;
  *height = ht;
  if (!pixels) return CSM_OK;
  const long long num_pixels = static_cast<long long>(w) * ht;
  if (capacity < num_pixels) {
    SetError("xray: a %d x %d image, capacity %lld", w, ht, static_cast<long long>(capacity));
    return CSM_E_CAPACITY;
  }
  CSM_CUDA(cudaSetDevice(ctx->device));
  const XRayAggregation& a = h->aggregations[aggregation];
  // std::log of every count a column can reach: at most one voxel per x of the box
  const int max_n = h->hi[0] - h->lo[0] + 1;
  for (int n = static_cast<int>(h->logs.size()); n <= max_n; ++n)
    h->logs.push_back(std::log(static_cast<double>(n)));
  struct Work {
    double* logs;
    unsigned* max_count;
    unsigned* counts;
    unsigned* pixels;
  };
  auto lay = [&](Carver& wc) {
    Work k;
    k.logs = wc.take<double>(max_n + 1);
    k.max_count = wc.take<unsigned>(1);
    k.counts = wc.take<unsigned>(num_pixels);
    k.pixels = wc.take<unsigned>(num_pixels);
    return k;
  };
  Carver sizer;
  lay(sizer);
  DevBuf& ws = ctx->D("xray_draw");
  CSM_TRY(ws.Reserve(sizer.at));
  Carver carver;
  carver.base = ws.as<char>();
  const Work k = lay(carver);
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  PinnedBuf& up = ctx->P("xray_logs");
  CSM_TRY(up.Reserve(sizeof(double) * (max_n + 1)));
  std::memcpy(up.p, h->logs.data(), sizeof(double) * (max_n + 1));
  CSM_CUDA(cudaMemcpyAsync(k.logs, up.p, sizeof(double) * (max_n + 1), cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemsetAsync(k.max_count, 0, sizeof(unsigned), s));
  CSM_CUDA(cudaMemsetAsync(k.counts, 0, sizeof(unsigned) * num_pixels, s));
  k_xr_count<<<DivUp(a.voxel_slots, kThreads), kThreads, 0, s>>>(
      a.voxel_keys, a.voxel_slots, h->hi[1], h->hi[2], w, k.counts, k.max_count);
  CSM_LAUNCH_CHECK();
  k_xr_pixels<<<DivUp(num_pixels, kThreads), kThreads, 0, s>>>(
      k.counts, w, num_pixels, h->hi[1], h->hi[2], k.max_count, k.logs, h->saturation_factor,
      a.column_keys, a.columns, a.column_slots - 1, k.pixels);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(pixels, k.pixels, sizeof(unsigned) * num_pixels,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  if (stats) {
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

csm_status csm_xray_voxels(const csm_xray* h, int32_t aggregation, int32_t* indices,
                           int64_t capacity, int64_t* num_voxels) {
  CSM_REQUIRE(h && num_voxels, "null pointer");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_TRY(CheckAggregation(h, aggregation));
  const XRayAggregation& a = h->aggregations[aggregation];
  *num_voxels = a.voxels;
  if (!indices) return CSM_OK;
  if (capacity < a.voxels) {
    SetError("xray: %lld voxels, capacity %lld", a.voxels, static_cast<long long>(capacity));
    return CSM_E_CAPACITY;
  }
  CSM_CUDA(cudaSetDevice(ctx->device));
  std::vector<unsigned long long> keys;
  CSM_TRY(Download<NoValues>(ctx, a.voxel_keys, nullptr, a.voxel_slots, &keys, nullptr));
  keys.erase(std::remove(keys.begin(), keys.end(), kEmptyKey), keys.end());
  std::sort(keys.begin(), keys.end());   // the packed key orders (z, y, x) ascending
  for (size_t j = 0; j < keys.size(); ++j) {
    indices[3 * j] = static_cast<int>(keys[j] & 0x3fff) - kCubeHalf;
    indices[3 * j + 1] = static_cast<int>((keys[j] >> 14) & 0x3fff) - kCubeHalf;
    indices[3 * j + 2] = static_cast<int>(keys[j] >> 28) - kCubeHalf;
  }
  *num_voxels = static_cast<int64_t>(keys.size());
  return CSM_OK;
}

csm_status csm_xray_columns(const csm_xray* h, int32_t aggregation, int32_t* yz, float* sums,
                            uint32_t* counts, int64_t capacity, int64_t* num_columns) {
  CSM_REQUIRE(h && num_columns, "null pointer");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_TRY(CheckAggregation(h, aggregation));
  const XRayAggregation& a = h->aggregations[aggregation];
  *num_columns = a.num_columns;
  if (!yz && !sums && !counts) return CSM_OK;
  if (capacity < a.num_columns) {
    SetError("xray: %lld columns, capacity %lld", a.num_columns, static_cast<long long>(capacity));
    return CSM_E_CAPACITY;
  }
  CSM_CUDA(cudaSetDevice(ctx->device));
  std::vector<unsigned long long> keys;
  std::vector<XRayColumn> vals;
  CSM_TRY(Download(ctx, a.column_keys, a.columns, a.column_slots, &keys, &vals));
  std::vector<long long> order;
  for (long long i = 0; i < a.column_slots; ++i)
    if (keys[i] != kEmptyKey) order.push_back(i);
  // (y, z) ascending, the std::map's order
  auto yz_of = [&](long long i) {
    return std::make_pair(static_cast<int>(keys[i] & 0x3fff), static_cast<int>(keys[i] >> 14));
  };
  std::sort(order.begin(), order.end(), [&](long long p, long long q) { return yz_of(p) < yz_of(q); });
  for (size_t j = 0; j < order.size(); ++j) {
    const XRayColumn& c = vals[order[j]];
    if (yz) {
      yz[2 * j] = yz_of(order[j]).first - kCubeHalf;
      yz[2 * j + 1] = yz_of(order[j]).second - kCubeHalf;
    }
    if (sums) {
      sums[3 * j] = c.sum_r;
      sums[3 * j + 1] = c.sum_g;
      sums[3 * j + 2] = c.sum_b;
    }
    if (counts) counts[j] = c.count;
  }
  *num_columns = static_cast<int64_t>(order.size());
  return CSM_OK;
}

}  // extern "C"
