// io::OutlierRemovingPointsProcessor (io/outlier_removing_points_processor.cc:53-129) on the
// device, bit for bit: the voxel counts after every phase and the kept points equal the
// reference's.
//
// The reference keeps a HybridGridBase<VoxelData> at resolution (float)voxel_size:
//   phase 1  ++hits of every point's voxel (GetCellIndex = lround(p / resolution), narrowed);
//   phase 2  for (float x = 0; x < length; x += voxel_size) per point, voxel_size a double, so
//            x_{k+1} = (float)((double)x_k + voxel_size): ++rays of the voxel of
//            origin + (x / length) * delta when that voxel has hits;
//   phase 3  drop the point iff !(rays < miss_per_hit_limit * hits), in double.
// Counts are integers whose order of addition does not matter, and every float step is per
// point, so the device reproduces them exactly with:
//   * an open-addressing hash map of the hit voxels (42-bit packed key, int32 {hits, rays})
//     that phase 1 fills with atomicCAS / atomicAdd.  The grid can only grow to [-8192, 8192)^3
//     (DynamicGrid::Grow's CHECK), so phase 1 refuses a point outside that cube; phase 2 and 3
//     read an absent voxel, inside the cube or not, as {0, 0}, which is what the reference's
//     value() returns, so they never insert;
//   * the x_k table, built on the host once per processor and extended on demand: a ray takes
//     the x_k < length, counted by binary search, and a prefix sum over the rays gives one
//     thread per sample (ray lengths vary by two orders of magnitude);
//   * per point a probe and a stable compaction of the kept indices.
// The host checks every input before anything is launched, so a refused call changes nothing.
// The map grows by a device rehash at the start of a phase-1 call, sized from the voxel count
// that the previous call read back, so every call is one stream synchronisation.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "common.cuh"
#include "point_batch.cuh"

namespace {

constexpr long long kInitialSlots = 1 << 12;
constexpr int kThreads = 256;

enum Phase : int { kHits = 1, kRays = 2, kFilter = 3 };

}  // namespace

struct csm_outlier_remover {
  csm::Ctx* ctx = nullptr;
  double voxel_size = 0, miss_per_hit_limit = 0;
  float resolution = 0;                     // HybridGridBase(float resolution)
  int phase = kHits;
  unsigned long long* keys = nullptr;       // slots, kEmptyKey when free
  int2* vals = nullptr;                     // {hits, rays}
  long long slots = 0;
  long long voxels = 0;                     // read back at the end of every phase-1 call
  unsigned long long* d_voxels = nullptr;
  // x_0 = 0, x_1, ... strictly increasing; `absorbed` once x_{k+1} == x_k for the last entry
  std::vector<float> xs{0.f};
  bool absorbed = false;
  float* d_xs = nullptr;
  size_t d_xs_len = 0, d_xs_cap = 0;
  ~csm_outlier_remover() {
    cudaFree(keys);
    cudaFree(vals);
    cudaFree(d_voxels);
    cudaFree(d_xs);
  }
};

namespace csm {
namespace {

// GetCellIndex (hybrid_grid.h:428-433) of (x, y, z) and its packed key; false outside the cube.
__device__ inline bool VoxelKey(float x, float y, float z, float resolution,
                                unsigned long long* key) {
  const int ix = RoundToInt(x / resolution);
  const int iy = RoundToInt(y / resolution);
  const int iz = RoundToInt(z / resolution);
  if (!InCube(ix) || !InCube(iy) || !InCube(iz)) return false;
  *key = Pack(ix, iy, iz);
  return true;
}

// Phase 1 (ProcessInPhaseOne): every point is inside the cube (checked on the host).
__global__ void k_or_hits(const float* __restrict__ xyz, int n, float resolution,
                          unsigned long long* keys, int2* vals, unsigned long long mask,
                          unsigned long long* voxels) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long key;
  if (!VoxelKey(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], resolution, &key)) return;
  bool inserted;
  const unsigned long long h = Insert(keys, mask, key, &inserted);
  atomicAdd(&vals[h].x, 1);
  if (inserted) atomicAdd(voxels, 1ull);
}

// Phase 2, per ray: delta = point - origin, its norm (Eigen's fixed-size norm), and the number
// of samples, #{k : x_k < length}.
__global__ void k_or_lengths(const float* __restrict__ xyz, const int* __restrict__ off, int nb,
                             const float* __restrict__ origins, int n,
                             const float* __restrict__ xs, int num_xs, float* lengths,
                             long long* samples) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* o = origins + 3 * CloudOf(off, nb, i);
  const float dx = xyz[3 * i] - o[0], dy = xyz[3 * i + 1] - o[1], dz = xyz[3 * i + 2] - o[2];
  const float length = sqrtf((dx * dx + dy * dy) + dz * dz);
  int lo = 0, hi = num_xs;
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (xs[mid] < length) lo = mid + 1; else hi = mid;
  }
  lengths[i] = length;
  samples[i] = lo;
}

// The last ray r in [lo, hi) with start[r] <= t.
__device__ inline int RayOf(const long long* __restrict__ start, int lo, int hi, long long t) {
  while (hi - lo > 1) {
    const int mid = (lo + hi) / 2;
    if (start[mid] <= t) lo = mid; else hi = mid;
  }
  return lo;
}

// Phase 2 (ProcessInPhaseTwo), one thread per sample: a fixed grid strides over tiles of
// blockDim samples; the tile's first and last rays bound every thread's search.
__global__ void k_or_rays(const float* __restrict__ xyz, const int* __restrict__ off, int nb,
                          const float* __restrict__ origins, const float* __restrict__ lengths,
                          const long long* __restrict__ start, int n,
                          const float* __restrict__ xs, float resolution,
                          const unsigned long long* __restrict__ keys, int2* vals,
                          unsigned long long mask) {
  __shared__ int tile_ray[2];
  const long long total = start[n];
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long base = static_cast<long long>(blockIdx.x) * blockDim.x; base < total;
       base += stride) {
    if (threadIdx.x < 2) {
      const long long t = threadIdx.x == 0 ? base : min(base + blockDim.x, total) - 1;
      tile_ray[threadIdx.x] = RayOf(start, 0, n, t);
    }
    __syncthreads();
    const long long t = base + threadIdx.x;
    if (t < total) {
      const int r = RayOf(start, tile_ray[0], tile_ray[1] + 1, t);
      const float x = xs[t - start[r]];
      const float* o = origins + 3 * CloudOf(off, nb, r);
      const float dx = xyz[3 * r] - o[0], dy = xyz[3 * r + 1] - o[1], dz = xyz[3 * r + 2] - o[2];
      const float s = x / lengths[r];
      unsigned long long key;
      if (VoxelKey(o[0] + s * dx, o[1] + s * dy, o[2] + s * dz, resolution, &key)) {
        const long long h = Find(keys, mask, key);
        if (h >= 0 && vals[h].x > 0) atomicAdd(&vals[h].y, 1);
      }
    }
    __syncthreads();
  }
}

// Phase 3 (ProcessInPhaseThree): keep iff rays < miss_per_hit_limit * hits, in double.
__global__ void k_or_keep(const float* __restrict__ xyz, const int* __restrict__ off, int nb,
                          int n, float resolution, const unsigned long long* __restrict__ keys,
                          const int2* __restrict__ vals, unsigned long long mask, double limit,
                          unsigned char* kept, int* num_kept) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int2 v = make_int2(0, 0);
  unsigned long long key;
  if (VoxelKey(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], resolution, &key)) {
    const long long h = Find(keys, mask, key);
    if (h >= 0) v = vals[h];
  }
  const bool keep = static_cast<double>(v.y) < limit * static_cast<double>(v.x);
  kept[i] = keep;
  if (keep) atomicAdd(&num_kept[CloudOf(off, nb, i)], 1);
}

__global__ void k_or_localize(const int* __restrict__ off, int nb,
                              const int* __restrict__ num_out, int n, int* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n || t >= *num_out) return;
  out[t] -= off[CloudOf(off, nb, out[t])];
}

int HostCell(float v, float resolution) {
  return static_cast<int>(std::lround(v / resolution));   // LONG_MIN narrows to 0, as on device
}

float HostLength(const float* p, const float* o) {
  const float dx = p[0] - o[0], dy = p[1] - o[1], dz = p[2] - o[2];
  return std::sqrt((dx * dx + dy * dy) + dz * dz);
}

// The checks every phase makes on its batches; *off gets the flat offsets.
csm_status ValidateBatches(const csm_outlier_remover* h, int phase, const float* const* xyz,
                           const int32_t* num_points, int32_t num_batches,
                           std::vector<int>* off) {
  CSM_REQUIRE(num_batches >= 0, "num_batches");
  CSM_REQUIRE(num_batches == 0 || (xyz && num_points), "null pointer");
  if (h->phase > phase) {
    SetError("outlier remover: a phase-%d call after phase %d has begun", phase, h->phase);
    return CSM_E_INVALID;
  }
  off->assign(1, 0);
  long long total = 0;
  for (int b = 0; b < num_batches; ++b) {
    CSM_REQUIRE(num_points[b] >= 0, "negative point count");
    CSM_REQUIRE(num_points[b] == 0 || xyz[b], "null batch");
    CSM_REQUIRE(Finite(xyz[b], 3 * static_cast<size_t>(num_points[b])), "non-finite point");
    total += num_points[b];
    CSM_REQUIRE(total < (1ll << 30), "more than 2^30 points in one call");
    off->push_back(static_cast<int>(total));
  }
  return CSM_OK;
}

// Grows the map (device rehash) until `incoming` more voxels keep it at most half full.
csm_status Reserve(csm_outlier_remover* h, long long incoming) {
  long long slots = std::max(h->slots, kInitialSlots);
  while (2 * (h->voxels + incoming) > slots) slots *= 2;
  if (slots == h->slots) return CSM_OK;
  const size_t bytes = static_cast<size_t>(slots) * (sizeof(unsigned long long) + sizeof(int2));
  size_t free_bytes = 0, total_bytes = 0;
  CSM_CUDA(cudaMemGetInfo(&free_bytes, &total_bytes));
  if (bytes > free_bytes) {
    SetError("outlier remover: growing the voxel map to %lld slots needs %zu bytes, %zu free",
             slots, bytes, free_bytes);
    return CSM_E_CAPACITY;
  }
  cudaStream_t s = h->ctx->stream;
  unsigned long long* keys = nullptr;
  int2* vals = nullptr;
  CSM_CUDA(cudaMallocAsync(&keys, sizeof(unsigned long long) * slots, s));
  if (cudaMallocAsync(&vals, sizeof(int2) * slots, s) != cudaSuccess) {
    cudaFreeAsync(keys, s);
    SetError("outlier remover: cudaMallocAsync of %lld voxel slots failed", slots);
    return CSM_E_CAPACITY;
  }
  CSM_CUDA(cudaMemsetAsync(keys, 0xff, sizeof(unsigned long long) * slots, s));
  CSM_CUDA(cudaMemsetAsync(vals, 0, sizeof(int2) * slots, s));
  if (h->slots > 0) {
    k_rehash<<<DivUp(h->slots, kThreads), kThreads, 0, s>>>(h->keys, h->vals, h->slots, keys,
                                                           vals, slots - 1);
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cudaFreeAsync(h->keys, s));
    CSM_CUDA(cudaFreeAsync(h->vals, s));
  }
  h->keys = keys;
  h->vals = vals;
  h->slots = slots;
  return CSM_OK;
}

// Extends the x_k table to cover `max_length` and brings the device copy up to date.  False
// when x stops growing below max_length: the reference's loop would never end.
csm_status ExtendSamples(csm_outlier_remover* h, float max_length, bool* covered) {
  std::vector<float>& xs = h->xs;
  while (!h->absorbed && xs.back() < max_length) {
    const float next = static_cast<float>(static_cast<double>(xs.back()) + h->voxel_size);
    if (next == xs.back()) h->absorbed = true; else xs.push_back(next);
  }
  *covered = !(xs.back() < max_length);
  if (!*covered || xs.size() == h->d_xs_len) return CSM_OK;
  cudaStream_t s = h->ctx->stream;
  if (xs.size() > h->d_xs_cap) {
    const size_t cap = std::max(xs.size(), 2 * h->d_xs_cap);
    float* d = nullptr;
    CSM_CUDA(cudaMallocAsync(&d, sizeof(float) * cap, s));
    if (h->d_xs) CSM_CUDA(cudaFreeAsync(h->d_xs, s));
    h->d_xs = d;
    h->d_xs_cap = cap;
    h->d_xs_len = 0;
  }
  // a pageable copy: the host table is not touched again before this call synchronises
  CSM_CUDA(cudaMemcpyAsync(h->d_xs + h->d_xs_len, xs.data() + h->d_xs_len,
                           sizeof(float) * (xs.size() - h->d_xs_len), cudaMemcpyHostToDevice, s));
  h->d_xs_len = xs.size();
  return CSM_OK;
}

struct Staged {
  float* xyz;
  int* off;
  float* origins;
};

// Uploads the batches (and the origins, when given) into `a`.
csm_status Upload(Ctx* ctx, const float* const* xyz, const std::vector<int>& off,
                  const float* origins, const Staged& a) {
  const int nb = static_cast<int>(off.size()) - 1;
  const int n = off.back();
  const size_t o_off = Align(sizeof(float) * 3 * static_cast<size_t>(n));
  const size_t o_org = o_off + Align(sizeof(int) * (nb + 1));
  const size_t bytes = o_org + sizeof(float) * 3 * std::max(nb, 1);
  PinnedBuf& up = ctx->P("outlier3d_up");
  CSM_TRY(up.Reserve(bytes));
  char* p = up.as<char>();
  for (int b = 0; b < nb; ++b)
    if (off[b + 1] > off[b])
      std::memcpy(p + sizeof(float) * 3 * off[b], xyz[b], sizeof(float) * 3 * (off[b + 1] - off[b]));
  std::memcpy(p + o_off, off.data(), sizeof(int) * (nb + 1));
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaMemcpyAsync(a.xyz, p, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(a.off, p + o_off, sizeof(int) * (nb + 1), cudaMemcpyHostToDevice, s));
  if (origins && nb > 0) {
    std::memcpy(p + o_org, origins, sizeof(float) * 3 * nb);
    CSM_CUDA(cudaMemcpyAsync(a.origins, p + o_org, sizeof(float) * 3 * nb, cudaMemcpyHostToDevice,
                             s));
  }
  return CSM_OK;
}

csm_status Finish(Ctx* ctx, csm_stats* stats) {
  CSM_CUDA(cudaEventRecord(ctx->ev1, ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

void NoWork(csm_stats* stats) {
  if (stats) std::memset(stats, 0, sizeof(*stats));
}

}  // namespace
}  // namespace csm

using namespace csm;

extern "C" {

csm_status csm_outlier_remover_create(double voxel_size, double miss_per_hit_limit,
                                      int32_t device, csm_outlier_remover** out) {
  CSM_REQUIRE(out, "null pointer");
  CSM_REQUIRE(std::isfinite(voxel_size) && voxel_size > 0.0, "voxel_size");
  CSM_REQUIRE(std::isfinite(miss_per_hit_limit), "miss_per_hit_limit");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_outlier_remover> h(new csm_outlier_remover);
  h->ctx = ctx;
  h->voxel_size = voxel_size;
  h->miss_per_hit_limit = miss_per_hit_limit;
  h->resolution = static_cast<float>(voxel_size);
  CSM_CUDA(cudaMalloc(&h->d_voxels, sizeof(unsigned long long)));
  CSM_CUDA(cudaMemsetAsync(h->d_voxels, 0, sizeof(unsigned long long), ctx->stream));
  CSM_TRY(Reserve(h.get(), 0));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = h.release();
  return CSM_OK;
}

csm_status csm_outlier_remover_destroy(csm_outlier_remover* h) {
  if (!h) return CSM_OK;
  std::lock_guard<std::mutex> lock(h->ctx->mu);
  cudaSetDevice(h->ctx->device);
  cudaStreamSynchronize(h->ctx->stream);
  delete h;
  return CSM_OK;
}

csm_status csm_outlier_remover_add_hits(csm_outlier_remover* h, const float* const* xyz,
                                        const int32_t* num_points, int32_t num_batches,
                                        csm_stats* stats) {
  CSM_REQUIRE(h, "null processor");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  std::vector<int> off;
  CSM_TRY(ValidateBatches(h, kHits, xyz, num_points, num_batches, &off));
  for (int b = 0; b < num_batches; ++b)
    for (int i = 0; i < 3 * num_points[b]; ++i)
      CSM_REQUIRE(InCube(HostCell(xyz[b][i], h->resolution)),
                  "hit outside the [-8192, 8192)^3 voxels the grid can hold");
  CSM_CUDA(cudaSetDevice(ctx->device));
  const int n = off.back();
  if (n == 0) {
    NoWork(stats);
    return CSM_OK;
  }
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_TRY(Reserve(h, n));
  Carver sizer;
  auto lay = [&](Carver& w) {
    Staged a;
    a.xyz = w.take<float>(3 * static_cast<size_t>(n));
    a.off = w.take<int>(num_batches + 1);
    a.origins = nullptr;
    return a;
  };
  lay(sizer);
  DevBuf& ws = ctx->D("outlier3d");
  CSM_TRY(ws.Reserve(sizer.at));
  Carver carver;
  carver.base = ws.as<char>();
  const Staged a = lay(carver);
  CSM_TRY(Upload(ctx, xyz, off, nullptr, a));
  k_or_hits<<<DivUp(n, kThreads), kThreads, 0, s>>>(a.xyz, n, h->resolution, h->keys, h->vals,
                                                    h->slots - 1, h->d_voxels);
  CSM_LAUNCH_CHECK();
  PinnedBuf& down = ctx->P("outlier3d_down");
  CSM_TRY(down.Reserve(sizeof(unsigned long long)));
  CSM_CUDA(cudaMemcpyAsync(down.p, h->d_voxels, sizeof(unsigned long long),
                           cudaMemcpyDeviceToHost, s));
  CSM_TRY(Finish(ctx, stats));
  h->voxels = static_cast<long long>(*down.as<unsigned long long>());
  return CSM_OK;
}

csm_status csm_outlier_remover_count_rays(csm_outlier_remover* h, const float* origins,
                                          const float* const* xyz, const int32_t* num_points,
                                          int32_t num_batches, csm_stats* stats) {
  CSM_REQUIRE(h, "null processor");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  std::vector<int> off;
  CSM_TRY(ValidateBatches(h, kRays, xyz, num_points, num_batches, &off));
  CSM_REQUIRE(num_batches == 0 || origins, "null origins");
  CSM_REQUIRE(Finite(origins, 3 * static_cast<size_t>(num_batches)), "non-finite origin");
  float max_length = 0.f;
  for (int b = 0; b < num_batches; ++b)
    for (int i = 0; i < num_points[b]; ++i)
      max_length = std::max(max_length, HostLength(xyz[b] + 3 * i, origins + 3 * b));
  CSM_CUDA(cudaSetDevice(ctx->device));
  bool covered;
  CSM_TRY(ExtendSamples(h, max_length, &covered));
  if (!covered) {
    SetError("outlier remover: x += voxel_size stops growing at %g, below a ray of length %g "
             "(the reference would loop forever)", h->xs.back(), max_length);
    return CSM_E_INVALID;
  }
  h->phase = kRays;
  const int n = off.back();
  if (n == 0) {
    NoWork(stats);
    return CSM_OK;
  }
  const int nb = num_batches;
  size_t scan_bytes = 0;
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<long long*>(nullptr),
                                         static_cast<long long*>(nullptr), n + 1, ctx->stream));
  struct Rays {
    Staged in;
    float* lengths;
    long long* samples;
    long long* start;
    void* temp;
  };
  auto lay = [&](Carver& w) {
    Rays a;
    a.in.xyz = w.take<float>(3 * static_cast<size_t>(n));
    a.in.off = w.take<int>(nb + 1);
    a.in.origins = w.take<float>(3 * static_cast<size_t>(nb));
    a.lengths = w.take<float>(n);
    a.samples = w.take<long long>(n + 1);
    a.start = w.take<long long>(n + 1);
    a.temp = w.take<char>(scan_bytes);
    return a;
  };
  Carver sizer;
  lay(sizer);
  DevBuf& ws = ctx->D("outlier3d");
  CSM_TRY(ws.Reserve(sizer.at));
  Carver carver;
  carver.base = ws.as<char>();
  const Rays a = lay(carver);
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_TRY(Upload(ctx, xyz, off, origins, a.in));
  k_or_lengths<<<DivUp(n, kThreads), kThreads, 0, s>>>(a.in.xyz, a.in.off, nb, a.in.origins, n,
                                                       h->d_xs, static_cast<int>(h->d_xs_len),
                                                       a.lengths, a.samples);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemsetAsync(a.samples + n, 0, sizeof(long long), s));
  size_t tb = scan_bytes;
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(a.temp, tb, a.samples, a.start, n + 1, s));
  k_or_rays<<<ctx->sm_count * 8, kThreads, 0, s>>>(a.in.xyz, a.in.off, nb, a.in.origins,
                                                   a.lengths, a.start, n, h->d_xs,
                                                   h->resolution, h->keys, h->vals,
                                                   h->slots - 1);
  CSM_LAUNCH_CHECK();
  return Finish(ctx, stats);
}

csm_status csm_outlier_remover_filter(csm_outlier_remover* h, const float* const* xyz,
                                      const int32_t* num_points, int32_t num_batches,
                                      int32_t* kept_indices, int32_t* num_kept,
                                      csm_stats* stats) {
  CSM_REQUIRE(h, "null processor");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  std::vector<int> off;
  CSM_TRY(ValidateBatches(h, kFilter, xyz, num_points, num_batches, &off));
  CSM_REQUIRE(num_batches == 0 || num_kept, "null num_kept");
  const int n = off.back();
  CSM_REQUIRE(n == 0 || kept_indices, "null kept_indices");
  CSM_CUDA(cudaSetDevice(ctx->device));
  h->phase = kFilter;
  if (n == 0) {
    for (int b = 0; b < num_batches; ++b) num_kept[b] = 0;
    NoWork(stats);
    return CSM_OK;
  }
  const int nb = num_batches;
  size_t sel_bytes = 0;
  CSM_CUDA(cub::DeviceSelect::Flagged(nullptr, sel_bytes, cub::CountingInputIterator<int>(0),
                                      static_cast<unsigned char*>(nullptr),
                                      static_cast<int*>(nullptr), static_cast<int*>(nullptr), n,
                                      ctx->stream));
  struct Keep {
    Staged in;
    unsigned char* kept;
    int* out;
    int* num_out;
    int* counts;
    void* temp;
  };
  auto lay = [&](Carver& w) {
    Keep a;
    a.in.xyz = w.take<float>(3 * static_cast<size_t>(n));
    a.in.off = w.take<int>(nb + 1);
    a.in.origins = nullptr;
    a.kept = w.take<unsigned char>(n);
    a.out = w.take<int>(n);
    a.num_out = w.take<int>(1);
    a.counts = w.take<int>(nb);
    a.temp = w.take<char>(sel_bytes);
    return a;
  };
  Carver sizer;
  lay(sizer);
  DevBuf& ws = ctx->D("outlier3d");
  CSM_TRY(ws.Reserve(sizer.at));
  Carver carver;
  carver.base = ws.as<char>();
  const Keep a = lay(carver);
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_TRY(Upload(ctx, xyz, off, nullptr, a.in));
  CSM_CUDA(cudaMemsetAsync(a.counts, 0, sizeof(int) * nb, s));
  k_or_keep<<<DivUp(n, kThreads), kThreads, 0, s>>>(a.in.xyz, a.in.off, nb, n, h->resolution,
                                                    h->keys, h->vals, h->slots - 1,
                                                    h->miss_per_hit_limit, a.kept, a.counts);
  CSM_LAUNCH_CHECK();
  size_t tb = sel_bytes;
  CSM_CUDA(cub::DeviceSelect::Flagged(a.temp, tb, cub::CountingInputIterator<int>(0), a.kept,
                                      a.out, a.num_out, n, s));
  k_or_localize<<<DivUp(n, kThreads), kThreads, 0, s>>>(a.in.off, nb, a.num_out, n, a.out);
  CSM_LAUNCH_CHECK();
  const size_t o_cnt = Align(sizeof(int) * n);
  PinnedBuf& down = ctx->P("outlier3d_down");
  CSM_TRY(down.Reserve(o_cnt + sizeof(int) * nb));
  char* d = down.as<char>();
  CSM_CUDA(cudaMemcpyAsync(d, a.out, sizeof(int) * n, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(d + o_cnt, a.counts, sizeof(int) * nb, cudaMemcpyDeviceToHost, s));
  CSM_TRY(Finish(ctx, stats));
  const int* counts = reinterpret_cast<const int*>(d + o_cnt);
  long long total = 0;
  for (int b = 0; b < nb; ++b) total += counts[b];
  std::memcpy(kept_indices, d, sizeof(int) * total);
  std::memcpy(num_kept, counts, sizeof(int) * nb);
  return CSM_OK;
}

csm_status csm_outlier_remover_voxels(const csm_outlier_remover* h, int32_t* indices,
                                      int32_t* hits, int32_t* rays, int64_t capacity,
                                      int64_t* num_voxels) {
  CSM_REQUIRE(h && num_voxels, "null pointer");
  Ctx* ctx = h->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  *num_voxels = h->voxels;
  if (!indices && !hits && !rays) return CSM_OK;
  if (capacity < h->voxels) {
    SetError("outlier remover: %lld voxels, capacity %lld", h->voxels,
             static_cast<long long>(capacity));
    return CSM_E_CAPACITY;
  }
  CSM_CUDA(cudaSetDevice(ctx->device));
  std::vector<unsigned long long> keys(h->slots);
  std::vector<int2> vals(h->slots);
  CSM_CUDA(cudaMemcpyAsync(keys.data(), h->keys, sizeof(unsigned long long) * h->slots,
                           cudaMemcpyDeviceToHost, ctx->stream));
  CSM_CUDA(cudaMemcpyAsync(vals.data(), h->vals, sizeof(int2) * h->slots, cudaMemcpyDeviceToHost,
                           ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  std::vector<long long> order;
  for (long long i = 0; i < h->slots; ++i)
    if (keys[i] != kEmptyKey) order.push_back(i);
  // the packed key orders (z, y, x) ascending
  std::sort(order.begin(), order.end(), [&](long long a, long long b) { return keys[a] < keys[b]; });
  for (size_t j = 0; j < order.size(); ++j) {
    const unsigned long long k = keys[order[j]];
    if (indices) {
      indices[3 * j] = static_cast<int>(k & 0x3fff) - kCubeHalf;
      indices[3 * j + 1] = static_cast<int>((k >> 14) & 0x3fff) - kCubeHalf;
      indices[3 * j + 2] = static_cast<int>(k >> 28) - kCubeHalf;
    }
    if (hits) hits[j] = vals[order[j]].x;
    if (rays) rays[j] = vals[order[j]].y;
  }
  *num_voxels = static_cast<int64_t>(order.size());
  return CSM_OK;
}

csm_status csm_outlier_remover_info(const csm_outlier_remover* h, int32_t* phase,
                                    int64_t* num_voxels, int64_t* slots) {
  CSM_REQUIRE(h, "null processor");
  std::lock_guard<std::mutex> lock(h->ctx->mu);
  if (phase) *phase = h->phase;
  if (num_voxels) *num_voxels = h->voxels;
  if (slots) *slots = h->slots;
  return CSM_OK;
}

}  // extern "C"
