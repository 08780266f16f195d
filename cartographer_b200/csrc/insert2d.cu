// ProbabilityGridRangeDataInserter2D::Insert on the device
// (cartographer/mapping/2d/probability_grid_range_data_inserter_2d.cc:35-133) into one or several
// csm_rt_grid2d handles, each growing as Grid2D::GrowLimits (2d/grid_2d.cc:125-164) does.
//
// The reference applies the hit table to every return's cell, then the miss table to every
// pixel of RayToPixelMask (internal/2d/ray_to_pixel_mask.cc) of each return's ray and each
// miss's ray.  A cell updated once carries kUpdateMarker and is skipped until FinishUpdate
// (grid_2d.cc:99-106), so each touched cell ends at hit_table[v] & 0x7fff if a return hits it,
// else miss_table[v] & 0x7fff, whatever the order inside each phase.  Several handles take the
// same scan independently; only their limits differ.  Here:
//   * the host makes one pass over the points: finiteness, their bounding box (from which every
//     handle's growth is decided, so a refused call changes nothing) and the sum of the rays'
//     L1 lengths; it computes each handle's superscaled origin cell;
//   * k_ins2_index (one thread per (handle, point)) computes every superscaled end index with
//     the host's Limits2::CellIndex, flags an end outside the grown limits, writes the hit cells
//     and each ray's pixel count, and reduces each handle's touched box: a mask contains both
//     its end pixels and stays inside their bounding box, so the box grows by the hit pixels
//     and, with free space on and at least one ray, by the misses' pixels and the origin's
//     (added on the host);
//   * each ray's mask has at most |dx| + |dy| + 1 pixels (it moves one pixel in x, in y or,
//     across an exact corner, in both per step).  One exclusive sum over the (handle, ray)
//     counts gives the slot offsets; each handle's slots live in a range the host reserved
//     from the L1 lengths (SlotReservation), and a handle whose exact total
//     passes its range raises a flag instead of writing;
//   * k_ins2_rays (one thread per (handle, ray) replays the reference's integer walk into its
//     slots), k_ins2_hits, k_ins2_misses (one thread per slot) and k_ins2_finish (clears the
//     markers of the hit cells and mask pixels again) take every handle in one launch
//     (blockIdx.y) and write nothing once a flag is raised;
//   * a 16-bit atomicCAS applies a table only while the marker is clear;
//   * the kernels write grown copies of the cells (GridInsert2, grid2d.cu), installed after the
//     insert's one synchronisation, when the flags and boxes are read back; a flag refuses the
//     call and every handle keeps its cells, limits and box.
#include <algorithm>
#include <climits>
#include <cmath>

#include <cub/device/device_scan.cuh>

#include "insert2d.cuh"
#include "resident2d.cuh"

struct csm_range_inserter2d {
  csm::Ctx* ctx = nullptr;
  csm_range_inserter_options2d options;
  uint16_t* d_tables = nullptr;   // hit table | miss table, 32768 entries each
  ~csm_range_inserter2d() { cudaFree(d_tables); }
};

namespace csm {

enum : int { kIns2Outside = 1, kIns2TooManyPixels = 2 };   // flag bits in status[0]

// One handle of an insert as the kernels see it.
struct Ins2Target {
  uint16_t* cells;        // what the insert writes: the handle's cells or their grown copy
  Limits2 S;              // the grown limits, superscaled by kSubpixelScale
  int pitch;
  int2 begin;             // the origin's superscaled cell
  long long slot_begin;   // the handle's slot range [slot_begin, slot_begin + slot_cap)
  long long slot_cap;
};

// Status block: status[0] the flags, status[4 + 4h ..] handle h's touched box (min x, min y,
// max x, max y).
constexpr int kIns2BoxBase = 4;

// One thread per (handle blockIdx.y, point i): points are the returns, then (with free space)
// the misses; with free space point i is also ray i.
__global__ void k_ins2_index(const Ins2Target* __restrict__ targets,
                             const float2* __restrict__ pts, int num_points, int n, int num_rays,
                             int* __restrict__ status, int* __restrict__ hit_flat,
                             int2* __restrict__ ends, long long* __restrict__ counts) {
  const int h = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const Ins2Target& t = targets[h];
  const long long ray = static_cast<long long>(h) * num_rays + i;
  bool in = false;
  int x = 0, y = 0;
  if (i < num_points) {
    const float2 p = pts[i];
    long long ix, iy;
    t.S.CellIndex(p.x, p.y, &ix, &iy);
    if (t.S.Contains(ix, iy)) {
      in = true;
      x = static_cast<int>(ix) / kSubpixelScale;
      y = static_cast<int>(iy) / kSubpixelScale;
      if (i < n) hit_flat[static_cast<long long>(h) * n + i] = y * t.pitch + x;
      if (num_rays > 0) {
        ends[ray] = make_int2(static_cast<int>(ix), static_cast<int>(iy));
        counts[ray] = abs(x - t.begin.x / kSubpixelScale) + abs(y - t.begin.y / kSubpixelScale) + 1;
      }
    } else {
      atomicOr(status, kIns2Outside);
      if (num_rays > 0) counts[ray] = 0;
    }
  }
  if (h == 0 && i == 0 && num_rays > 0)   // the sum's last entry: the total of every handle
    counts[static_cast<long long>(gridDim.y) * num_rays] = 0;
  const int lo_x = __reduce_min_sync(0xffffffffu, in ? x : INT_MAX);
  const int lo_y = __reduce_min_sync(0xffffffffu, in ? y : INT_MAX);
  const int hi_x = __reduce_max_sync(0xffffffffu, in ? x : INT_MIN);
  const int hi_y = __reduce_max_sync(0xffffffffu, in ? y : INT_MIN);
  if ((threadIdx.x & 31) == 0 && lo_x <= hi_x) {
    int* box = status + kIns2BoxBase + 4 * h;
    atomicMin(box + 0, lo_x);
    atomicMin(box + 1, lo_y);
    atomicMax(box + 2, hi_x);
    atomicMax(box + 3, hi_y);
  }
}

// RayToPixelMask(begin, end, kSubpixelScale) of ray r of handle blockIdx.y into its slots as
// flat cell indices; the slots it does not fill stay -1.  Writes nothing after an end outside
// the limits, or for a handle whose exact total passes its slot range (which raises the flag).
__global__ void k_ins2_rays(const Ins2Target* __restrict__ targets, const int2* __restrict__ ends,
                            const long long* __restrict__ off, int num_rays, int* status,
                            int* __restrict__ slots) {
  const int h = blockIdx.y;
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= num_rays || (*status & kIns2Outside)) return;
  const Ins2Target& t = targets[h];
  const long long* o = off + static_cast<long long>(h) * num_rays;
  if (o[num_rays] - o[0] > t.slot_cap) {
    if (r == 0) atomicOr(status, kIns2TooManyPixels);
    return;
  }
  int* out = slots + t.slot_begin + (o[r] - o[0]);
  const int cap = static_cast<int>(o[r + 1] - o[r]);
  const int pitch = t.pitch;
  int count = 0;
  RayToPixelMask2(t.begin, ends[static_cast<long long>(h) * num_rays + r], [&](int x, int y) {
    if (count < cap) out[count] = y * pitch + x;
    ++count;
  });
  for (int k = count; k < cap; ++k) out[k] = -1;
}

// The number of slots handle h's rays fill: its exact total.
__device__ __forceinline__ long long HandleSlots(const long long* off, int h, int num_rays) {
  return num_rays > 0 ? off[static_cast<long long>(h + 1) * num_rays] -
                            off[static_cast<long long>(h) * num_rays]
                      : 0;
}

__global__ void k_ins2_hits(const Ins2Target* __restrict__ targets, const int* __restrict__ hit_flat,
                            int n, const int* status, const uint16_t* __restrict__ hit_table) {
  if (*status) return;
  const int h = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) ApplyTable(targets[h].cells + hit_flat[static_cast<long long>(h) * n + i], hit_table);
}

__global__ void k_ins2_misses(const Ins2Target* __restrict__ targets,
                              const long long* __restrict__ off, int num_rays,
                              const int* __restrict__ slots, const int* status,
                              const uint16_t* __restrict__ miss_table) {
  if (*status) return;
  const int h = blockIdx.y;
  const long long num_slots = HandleSlots(off, h, num_rays);
  const int* s = slots + targets[h].slot_begin;
  uint16_t* cells = targets[h].cells;
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < num_slots;
       i += gridDim.x * blockDim.x) {
    const int flat = s[i];
    if (flat >= 0) ApplyTable(cells + flat, miss_table);
  }
}

// FinishUpdate: clears the marker of every hit cell and mask pixel (the same cell may be
// listed many times; neighbouring 16-bit cells share a word).
__global__ void k_ins2_finish(const Ins2Target* __restrict__ targets,
                              const int* __restrict__ hit_flat, int n,
                              const long long* __restrict__ off, int num_rays,
                              const int* __restrict__ slots, const int* status) {
  if (*status) return;
  const int h = blockIdx.y;
  const long long total = n + HandleSlots(off, h, num_rays);
  const int* hits = hit_flat + static_cast<long long>(h) * n;
  const int* s = slots + targets[h].slot_begin;
  uint16_t* cells = targets[h].cells;
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += gridDim.x * blockDim.x) {
    const int flat = i < n ? hits[i] : s[i - n];
    if (flat < 0) continue;
    ClearUpdateMarker(cells, flat);
  }
}

// The slots handle h reserves for rays whose L1 lengths sum to l1 (in metres), at
// resolution res.  A point's pixel is floor((max - p) / res) per axis (the superscaled index
// rounds within one subpixel of it and drops the subpixels), so a ray's |dx| + |dy| + 1 is
// below its L1 length in cells + 3.  The relative and the + 1 margins absorb the double
// rounding of the lengths and of the cell coordinates on exact cell borders.  Capped at
// 2^31 - 1: an exact total past that is refused anyway ("too many ray pixels").
long long SlotReservation(double l1, double res, int num_rays) {
  const double bound = l1 / res * (1. + 1e-9) + 3. * num_rays + 1.;
  return bound >= static_cast<double>(INT_MAX) ? INT_MAX : static_cast<long long>(bound);
}

}  // namespace csm

using namespace csm;

namespace {

// The handles of one insert: 1 .. 65535 distinct ProbabilityGrid handles on the inserter's device.
csm_status CheckGrids(const csm_range_inserter2d* inserter, csm_rt_grid2d* const* grids,
                      int32_t num_grids) {
  CSM_REQUIRE(num_grids >= 1 && num_grids <= 65535, "num_grids");
  const int H = num_grids;
  for (int h = 0; h < H; ++h) {
    CSM_REQUIRE(grids[h] != nullptr, "null grid");
    for (int k = 0; k < h; ++k) CSM_REQUIRE(grids[k] != grids[h], "a grid appears twice");
  }
  for (int h = 0; h < H; ++h) {
    CSM_REQUIRE(grids[h]->d_wcells == nullptr, "a TSDF2D handle takes the TSDF inserter");
    CSM_REQUIRE(grids[h]->ctx == inserter->ctx, "grid on another device than the inserter");
  }
  return CSM_OK;
}

// Every handle's insert from the points' box and ray lengths: the host's points (returns,
// misses) are uploaded, or points.d_pts already holds them on the device.
csm_status InsertSubmaps(const csm_range_inserter2d* inserter, const float origin[3],
                         const InsertPoints2& points, const float* returns, const float* misses,
                         int n, int m, csm_rt_grid2d* const* grids, int32_t num_grids,
                         csm_stats* stats) {
  const int H = num_grids;
  Ctx* ctx = inserter->ctx;
  const bool free_space = inserter->options.insert_free_space != 0;
  const int num_points = free_space ? n + m : n;   // what the kernels index
  const int num_rays = free_space ? n + m : 0;
  const float lo_x = points.lo_x, lo_y = points.lo_y, hi_x = points.hi_x, hi_y = points.hi_y;
  const double l1 = free_space ? points.l1 : 0.;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  // ---- every handle grows, and its origin is checked, before anything changes ----
  std::vector<std::unique_ptr<GridInsert2>> tx(H);
  std::vector<Ins2Target> targets(H);
  long long num_slots = 0;
  for (int h = 0; h < H; ++h) {
    tx[h].reset(new GridInsert2(grids[h], h));
    CSM_REQUIRE(tx[h]->Grow(lo_x, lo_y, hi_x, hi_y), "the grid would grow past 30000 cells");
    const Limits2& L = tx[h]->L;
    Ins2Target& t = targets[h];
    // the superscaled limits (:58-65)
    t.S = Limits2{L.resolution / kSubpixelScale, L.max_x, L.max_y, L.nx * kSubpixelScale,
                  L.ny * kSubpixelScale};
    long long ix, iy;
    t.S.CellIndex(origin[0], origin[1], &ix, &iy);
    CSM_REQUIRE(t.S.Contains(ix, iy), "origin outside the grown limits");
    t.begin = make_int2(static_cast<int>(ix), static_cast<int>(iy));
    t.pitch = tx[h]->arrays.pitch;
    t.slot_begin = num_slots;
    t.slot_cap = num_rays > 0 ? SlotReservation(l1, L.resolution, num_rays) : 0;
    num_slots += t.slot_cap;
  }

  // ---- workspaces, before any transaction queues a copy into pinned memory ----
  cudaStream_t s = ctx->stream;
  auto align = [](size_t b) { return (b + 255) / 256 * 256; };
  const size_t hn = static_cast<size_t>(H) * n, hr = static_cast<size_t>(H) * num_rays;
  const size_t status_bytes = sizeof(int) * (kIns2BoxBase + 4 * static_cast<size_t>(H));
  const size_t o_targets = align(status_bytes);
  const size_t o_pts = o_targets + align(sizeof(Ins2Target) * H);
  const size_t up_bytes =
      o_pts + (points.d_pts ? 0 : align(sizeof(float2) * static_cast<size_t>(num_points)));
  const size_t o_hits = up_bytes;
  const size_t o_ends = o_hits + align(sizeof(int) * hn);
  const size_t o_counts = o_ends + align(sizeof(int2) * hr);
  const size_t o_off = o_counts + align(sizeof(long long) * (hr + 1));
  const size_t o_scan = o_off + align(sizeof(long long) * (hr + 1));
  size_t scan_bytes = 0;
  if (num_rays > 0)
    CSM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<long long*>(nullptr),
                                           static_cast<long long*>(nullptr),
                                           static_cast<long long>(hr + 1), s));
  const size_t o_slots = o_scan + align(scan_bytes);
  const size_t work_bytes = o_slots + sizeof(int) * static_cast<size_t>(num_slots);
  PinnedBuf& up = ctx->P("ins2_upload");
  PinnedBuf& down = ctx->P("ins2_status");
  DevBuf& d_work = ctx->D("ins2_work");
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(down.Reserve(status_bytes));
  CSM_TRY(d_work.Reserve(work_bytes));
  CSM_TRY(ReserveKnownBoxSlots(ctx, H));

  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  for (int h = 0; h < H; ++h) {
    CSM_TRY(tx[h]->Begin());
    targets[h].cells = tx[h]->arrays.cells;
  }
  // ---- upload: status | targets | points ----
  char* hp = up.as<char>();
  int* h_status = reinterpret_cast<int*>(hp);
  std::fill(h_status, h_status + kIns2BoxBase, 0);
  for (int h = 0; h < H; ++h) {
    int* box = h_status + kIns2BoxBase + 4 * h;
    box[0] = box[1] = INT_MAX;
    box[2] = box[3] = INT_MIN;
  }
  std::memcpy(hp + o_targets, targets.data(), sizeof(Ins2Target) * H);
  if (!points.d_pts) {
    float2* h_pts = reinterpret_cast<float2*>(hp + o_pts);
    for (int i = 0; i < num_points; ++i) {
      const float* q = i < n ? returns + 3 * static_cast<size_t>(i)
                             : misses + 3 * static_cast<size_t>(i - n);
      h_pts[i] = make_float2(q[0], q[1]);
    }
  }
  CSM_CUDA(cudaMemcpyAsync(d_work.p, hp, up_bytes, cudaMemcpyHostToDevice, s));
  char* d = d_work.as<char>();
  int* d_status = reinterpret_cast<int*>(d);
  const Ins2Target* d_targets = reinterpret_cast<const Ins2Target*>(d + o_targets);
  int* d_hits = reinterpret_cast<int*>(d + o_hits);
  int2* d_ends = reinterpret_cast<int2*>(d + o_ends);
  long long* d_counts = reinterpret_cast<long long*>(d + o_counts);
  long long* d_off = reinterpret_cast<long long*>(d + o_off);
  int* d_slots = reinterpret_cast<int*>(d + o_slots);
  if (num_points > 0) {
    const dim3 per_point(DivUp(num_points, 256), H);
    k_ins2_index<<<per_point, 256, 0, s>>>(d_targets,
                                           points.d_pts ? points.d_pts
                                                        : reinterpret_cast<const float2*>(d + o_pts),
                                           num_points, n, num_rays, d_status, d_hits, d_ends,
                                           d_counts);
    CSM_LAUNCH_CHECK();
    if (num_rays > 0) {
      CSM_CUDA(cub::DeviceScan::ExclusiveSum(d + o_scan, scan_bytes, d_counts, d_off,
                                             static_cast<long long>(hr + 1), s));
      k_ins2_rays<<<per_point, 256, 0, s>>>(d_targets, d_ends, d_off, num_rays, d_status,
                                            d_slots);
      CSM_LAUNCH_CHECK();
    }
    if (n > 0) {
      k_ins2_hits<<<dim3(DivUp(n, 256), H), 256, 0, s>>>(d_targets, d_hits, n, d_status,
                                                         inserter->d_tables);
      CSM_LAUNCH_CHECK();
    }
    long long max_cap = 0;
    for (const Ins2Target& t : targets) max_cap = std::max(max_cap, t.slot_cap);
    if (num_rays > 0) {
      k_ins2_misses<<<dim3(Blocks(max_cap), H), 256, 0, s>>>(
          d_targets, d_off, num_rays, d_slots, d_status, inserter->d_tables + kValueCount);
      CSM_LAUNCH_CHECK();
    }
    k_ins2_finish<<<dim3(Blocks(n + max_cap), H), 256, 0, s>>>(d_targets, d_hits, n, d_off,
                                                               num_rays, d_slots, d_status);
    CSM_LAUNCH_CHECK();
  }
  CSM_CUDA(cudaMemcpyAsync(down.p, d_status, status_bytes, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  const int flags = down.as<int>()[0];
  CSM_REQUIRE(!(flags & kIns2Outside), "a point outside the grown limits");
  CSM_REQUIRE(!(flags & kIns2TooManyPixels), "too many ray pixels");
  for (int h = 0; h < H; ++h) {
    KnownBox2 touched = BoxFrom(down.as<int>() + kIns2BoxBase + 4 * h);
    if (num_rays > 0)
      touched.Extend(targets[h].begin.x / kSubpixelScale, targets[h].begin.y / kSubpixelScale);
    CSM_TRY(tx[h]->Commit(touched, stats));
  }
  return CSM_OK;
}

}  // namespace

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

csm_status csm_range_inserter2d_insert_submaps(const csm_range_inserter2d* inserter,
                                                const float origin[3], const float* returns,
                                                int32_t num_returns, const float* misses,
                                                int32_t num_misses, csm_rt_grid2d* const* grids,
                                                int32_t num_grids, csm_stats* stats) {
  CSM_REQUIRE(inserter && origin && grids, "null pointer");
  CSM_REQUIRE(num_returns >= 0 && (num_returns == 0 || returns), "returns");
  CSM_REQUIRE(num_misses >= 0 && (num_misses == 0 || misses), "misses");
  CSM_TRY(CheckGrids(inserter, grids, num_grids));
  const int n = num_returns, m = num_misses;
  // ---- one pass over the points: finite, bounding box (GrowAsNeeded, :35-50), ray lengths ----
  CSM_REQUIRE(Finite(origin, 3), "non-finite point");
  float lo_x = origin[0], lo_y = origin[1], hi_x = origin[0], hi_y = origin[1];
  double l1 = 0.;
  bool finite = true;
  auto scan = [&](const float* p, int k) {
    for (int i = 0; i < k; ++i) {
      const float* q = p + 3 * static_cast<size_t>(i);
      finite = finite && std::isfinite(q[0]) && std::isfinite(q[1]) && std::isfinite(q[2]);
      lo_x = std::min(lo_x, q[0]);
      lo_y = std::min(lo_y, q[1]);
      hi_x = std::max(hi_x, q[0]);
      hi_y = std::max(hi_y, q[1]);
      l1 += std::abs(static_cast<double>(q[0]) - origin[0]) +
            std::abs(static_cast<double>(q[1]) - origin[1]);
    }
  };
  scan(returns, n);
  scan(misses, m);
  CSM_REQUIRE(finite, "non-finite point");
  const InsertPoints2 points{nullptr, lo_x, lo_y, hi_x, hi_y, l1};
  return InsertSubmaps(inserter, origin, points, returns, misses, n, m, grids, num_grids, stats);
}

}  // extern "C"

csm_status csm::InsertSubmapsResident(const csm_range_inserter2d* inserter, const float origin[3],
                                      const InsertPoints2& points, int32_t num_returns,
                                      int32_t num_misses, csm_rt_grid2d* const* grids,
                                      int32_t num_grids, csm_stats* stats) {
  CSM_REQUIRE(inserter && origin && grids && points.d_pts, "null pointer");
  CSM_TRY(CheckGrids(inserter, grids, num_grids));
  return InsertSubmaps(inserter, origin, points, nullptr, nullptr, num_returns, num_misses, grids,
                       num_grids, stats);
}

extern "C" {
csm_status csm_range_inserter2d_insert(const csm_range_inserter2d* inserter,
                                       const float origin[3], const float* returns,
                                       int32_t num_returns, const float* misses,
                                       int32_t num_misses, csm_rt_grid2d* grid,
                                       csm_stats* stats) {
  CSM_REQUIRE(grid, "null pointer");
  return csm_range_inserter2d_insert_submaps(inserter, origin, returns, num_returns, misses,
                                             num_misses, &grid, 1, stats);
}

}  // extern "C"
