// The 3D grid handles: csm_grid3d (a HybridGrid) and csm_intensity_grid3d (an
// IntensityHybridGrid) as dense device boxes.  Creation from voxel lists, read-back, growth
// (GridInsert3, the part of csm_range_inserter3d_insert that changes the handles), and the
// non-zero voxels of a csm_grid3d in HybridGrid's iteration order, with the proto written
// from them.
#include <algorithm>
#include <climits>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "grid3d.cuh"
#include "proto_write.h"
#include "value_conversion.h"

namespace csm {

template <typename T>
__global__ void k3_scatter(const int* __restrict__ idx, const T* __restrict__ values, long long n,
                           Box3 box, T* __restrict__ vol) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  vol[box.Index(idx[3 * i], idx[3 * i + 1], idx[3 * i + 2])] = values[i];
}

// Copies the part of box `from` that lies in box `to` (`to` already zero-filled).
template <typename T>
__global__ void k_ins3_copy(const T* __restrict__ src, Box3 from, T* __restrict__ dst, Box3 to) {
  const unsigned long long total = from.Volume();
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
       i < total; i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const int x = from.lo[0] + static_cast<int>(i % from.n[0]);
    const int y = from.lo[1] + static_cast<int>(i / from.n[0] % from.n[1]);
    const int z = from.lo[2] + static_cast<int>(i / (static_cast<unsigned long long>(from.n[0]) * from.n[1]));
    if (x < to.lo[0] || x >= to.lo[0] + to.n[0] || y < to.lo[1] || y >= to.lo[1] + to.n[1] ||
        z < to.lo[2] || z >= to.lo[2] + to.n[2])
      continue;
    dst[to.Index(x, y, z)] = src[i];
  }
}

// The bounding box of the non-zero cells of `b`, as offsets from b.lo: mn[0..2] receives the
// min (atomicMin; the caller sets them to 0xffffffff), mx[0..2] the max + 1 (atomicMax; the
// caller zeroes them), so mx[0] != 0 is the "any non-zero cell" flag.  Per thread, then per
// block (warp reductions + shared memory), then six atomics per block that saw a cell.
// Launched with RowGrid.
__global__ void __launch_bounds__(256)
k3_nonzero_box(Box16 b, unsigned* __restrict__ mn_out, unsigned* __restrict__ mx_out) {
  __shared__ unsigned s[6][8];
  unsigned mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u};
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const long long rows = static_cast<long long>(b.n[1]) * b.n[2];
  if (x < b.n[0]) {
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
      if (__ldg(b.p + r * b.n[0] + x) == 0) continue;
      const unsigned y = static_cast<unsigned>(r % b.n[1]), z = static_cast<unsigned>(r / b.n[1]);
      const unsigned c[3] = {static_cast<unsigned>(x), y, z};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        mn[a] = min(mn[a], c[a]);
        mx[a] = max(mx[a], c[a] + 1u);
      }
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
    if (lane == 0) {
      s[a][warp] = mn[a];
      s[3 + a][warp] = mx[a];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned v[6];
    for (int a = 0; a < 6; ++a) {
      v[a] = s[a][0];
      for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w)
        v[a] = a < 3 ? min(v[a], s[a][w]) : max(v[a], s[a][w]);
    }
    if (v[3] != 0u)
      for (int a = 0; a < 3; ++a) {
        atomicMin(&mn_out[a], v[a]);
        atomicMax(&mx_out[a], v[3 + a]);
      }
  }
}

// ---- the non-zero voxels of a csm_grid3d in HybridGrid's iteration order (csm_grid3d_voxels) ----
// HybridGrid is DynamicGrid<NestedGrid<FlatGrid<uint16, 3>, 3>> (hybrid_grid.h), and each level
// walks its cells in ToFlatIndex order, z outermost (:40-43), skipping null meta cells and value 0
// (:57, :106-115).  The DynamicGrid shifts an index by grid_size() / 2 = 2^(bits - 1) * 64, a
// multiple of 64 (:263-264), so its meta cells are the 64^3 blocks floor(index / 64) in z, y, x
// order, whatever bits_ is and however the grid grew; inside them come the NestedGrid's 8^3 blocks
// and inside those the cells, both in z, y, x order.  The kernels below enumerate the 64-aligned
// cover of the non-zero box in that blocked order and compact the non-zero cells stably: tile t is
// kVoxTile consecutive cells of the enumeration (4 of the 8^3 blocks, 128 tiles per 64^3 block),
// and thread k of a tile holds the x-row (z & 7, y & 7) = ((k & 63) >> 3, k & 7) of its block
// k >> 6.  No sort is needed.
constexpr int kVoxThreads = 256;
constexpr int kVoxTile = 8 * kVoxThreads;

struct VoxCover {
  Box16 src;
  int lo[3];   // multiples of 64
  int nb[3];   // 64^3 blocks per axis
};

// The 8 cells x .. x + 7 of this thread's row in tile t, and their values in v.
__device__ __forceinline__ void VoxRow(const VoxCover& c, long long t, int* x, int* y, int* z,
                                       uint16_t v[8]) {
  const long long m = t >> 7;                                          // the 64^3 block
  const int f = static_cast<int>(t & 127) * 4 + (threadIdx.x >> 6);    // the 8^3 block in it
  const int r = threadIdx.x & 63;
  const long long bxy = static_cast<long long>(c.nb[0]) * c.nb[1];
  const int bz = static_cast<int>(m / bxy);
  const int by = static_cast<int>((m % bxy) / c.nb[0]);
  const int bx = static_cast<int>(m % c.nb[0]);
  *x = c.lo[0] + 64 * bx + 8 * (f & 7);
  *y = c.lo[1] + 64 * by + 8 * ((f >> 3) & 7) + (r & 7);
  *z = c.lo[2] + 64 * bz + 8 * (f >> 6) + (r >> 3);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = Val16(c.src, *x + i, *y, *z);
}

// Pass 1: counts[t] = the non-zero cells of tile t.
__global__ void __launch_bounds__(kVoxThreads)
k3_voxel_count(VoxCover c, long long* __restrict__ counts) {
  __shared__ int s[kVoxThreads / 32];
  int x, y, z;
  uint16_t v[8];
  VoxRow(c, blockIdx.x, &x, &y, &z, v);
  int n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) n += v[i] != 0;
  n = __reduce_add_sync(0xffffffffu, n);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int total = 0;
    for (int w = 0; w < kVoxThreads / 32; ++w) total += s[w];
    counts[blockIdx.x] = total;
  }
}

// Pass 2: the non-zero cells of tile t written from offsets[t] on, in enumeration order:
// idx as {x, y, z}, val as held.
__global__ void __launch_bounds__(kVoxThreads)
k3_voxel_write(VoxCover c, const long long* __restrict__ counts,
               const long long* __restrict__ offsets, int* __restrict__ idx,
               uint16_t* __restrict__ val) {
  typedef cub::BlockScan<int, kVoxThreads> Scan;
  __shared__ typename Scan::TempStorage scan;
  if (counts[blockIdx.x] == 0) return;   // uniform over the block
  int x, y, z;
  uint16_t v[8];
  VoxRow(c, blockIdx.x, &x, &y, &z, v);
  int n = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) n += v[i] != 0;
  int before;
  Scan(scan).ExclusiveSum(n, before);
  long long o = offsets[blockIdx.x] + before;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (v[i] == 0) continue;
    idx[3 * o] = x + i;
    idx[3 * o + 1] = y;
    idx[3 * o + 2] = z;
    val[o] = v[i];
    ++o;
  }
}

TightBox3 ListBox3(const int32_t* idx, int64_t n) {
  TightBox3 t;
  for (int64_t i = 0; i < n; ++i) t.Include(idx + 3 * i);
  return t;
}

Grid3Dev MakeGrid3Dev(const uint16_t* p, const Box3& box, float resolution) {
  const ValueConversion probability = MakeValueConversion(kMinProbability, kMaxProbability);
  Grid3Dev d;
  d.p = p;
  for (int a = 0; a < 3; ++a) {
    d.lo[a] = box.lo[a];
    d.n[a] = box.n[a];
  }
  d.resolution = resolution;
  d.k_scale = probability.scale;
  d.bias = probability.bias;
  d.min_probability = kMinProbability;
  return d;
}

template <typename T>
csm_status ScatterVoxels3(Ctx* ctx, const int32_t* idx, const T* values, long long n,
                          const Box3& box, T* vol) {
  if (n == 0) return CSM_OK;
  cudaStream_t s = ctx->stream;
  DevBuf& d_idx = ctx->D("g3_idx");
  DevBuf& d_val = ctx->D("g3_val");
  CSM_TRY(d_idx.Reserve(sizeof(int) * 3 * n));
  CSM_TRY(d_val.Reserve(sizeof(T) * n));
  CSM_CUDA(cudaMemcpyAsync(d_idx.p, idx, sizeof(int) * 3 * n, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(d_val.p, values, sizeof(T) * n, cudaMemcpyHostToDevice, s));
  k3_scatter<T><<<Blocks(n, 1LL << 30), 256, 0, s>>>(d_idx.as<int>(), d_val.as<T>(), n, box, vol);
  CSM_LAUNCH_CHECK();
  return CSM_OK;
}

template csm_status ScatterVoxels3<uint16_t>(Ctx*, const int32_t*, const uint16_t*, long long,
                                             const Box3&, uint16_t*);

csm_status QueueNonZeroBox3(const csm_grid3d* g, unsigned* mn, unsigned* mx) {
  Ctx* ctx = g->ctx;
  cudaStream_t s = ctx->stream;
  const Box16 b = HandleBox(g);
  CSM_CUDA(cudaMemsetAsync(mn, 0xff, 3 * sizeof(unsigned), s));
  CSM_CUDA(cudaMemsetAsync(mx, 0, 3 * sizeof(unsigned), s));
  const long long rows = static_cast<long long>(b.n[1]) * b.n[2];
  k3_nonzero_box<<<RowGrid(b.n[0], rows, ctx->sm_count * 8), 256, 0, s>>>(b, mn, mx);
  CSM_LAUNCH_CHECK();
  return CSM_OK;
}

// One stream synchronisation for the non-zero box and, if the grid has a non-zero voxel, one
// for the count.
csm_status DeviceVoxels3D(const csm_grid3d* g, long long list_capacity, long long* n,
                          const int** d_idx, const uint16_t** d_val) {
  Ctx* ctx = g->ctx;
  cudaStream_t s = ctx->stream;
  VoxCover c;
  c.src = HandleBox(g);
  DevBuf* d_box;
  CSM_TRY(ctx->Reserve("g3v_box", 6 * sizeof(unsigned), &d_box));
  unsigned* box = d_box->as<unsigned>();
  CSM_TRY(QueueNonZeroBox3(g, box, box + 3));
  PinnedBuf& pin = ctx->P("g3v_box");
  CSM_TRY(pin.Reserve(6 * sizeof(unsigned) + sizeof(long long)));
  unsigned* h = pin.as<unsigned>();
  CSM_CUDA(cudaMemcpyAsync(h, box, 6 * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  *n = 0;
  if (h[3] == 0u) return CSM_OK;   // no non-zero cell
  // the 64-aligned cover of the non-zero box (floor division: indices may be negative)
  long long tiles = static_cast<long long>(262144 / kVoxTile);
  for (int a = 0; a < 3; ++a) {
    const int b0 = (c.src.lo[a] + static_cast<int>(h[a]) + kCube) / 64 - kCube / 64;
    const int b1 = (c.src.lo[a] + static_cast<int>(h[3 + a]) - 1 + kCube) / 64 - kCube / 64;
    c.lo[a] = 64 * b0;
    c.nb[a] = b1 - b0 + 1;
    tiles *= c.nb[a];
  }
  if (tiles >= INT_MAX) {   // one block per tile
    SetError("the non-zero box of the grid is too large to enumerate");
    return CSM_E_CAPACITY;
  }
  // counts[tiles] stays 0, so that the exclusive scan's last entry is the total
  size_t scan_bytes = 0;
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<long long*>(nullptr),
                                         static_cast<long long*>(nullptr), tiles + 1, s));
  const size_t o_off = (sizeof(long long) * (tiles + 1) + 255) / 256 * 256;
  const size_t o_temp = 2 * o_off;
  DevBuf* d_work;
  CSM_TRY(ctx->Reserve("g3v_scan", o_temp + scan_bytes, &d_work));
  long long* counts = d_work->as<long long>();
  long long* offsets = reinterpret_cast<long long*>(d_work->as<char>() + o_off);
  CSM_CUDA(cudaMemsetAsync(counts + tiles, 0, sizeof(long long), s));
  k3_voxel_count<<<static_cast<unsigned>(tiles), kVoxThreads, 0, s>>>(c, counts);
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(d_work->as<char>() + o_temp, scan_bytes, counts, offsets,
                                         tiles + 1, s));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  long long* h_n = reinterpret_cast<long long*>(h + 6);
  CSM_CUDA(cudaMemcpyAsync(h_n, offsets + tiles, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  *n = *h_n;
  if (*n > list_capacity) return CSM_OK;
  DevBuf* out_idx;
  DevBuf* out_val;
  CSM_TRY(ctx->Reserve("g3v_idx", sizeof(int) * 3 * *n, &out_idx));
  CSM_TRY(ctx->Reserve("g3v_val", sizeof(uint16_t) * *n, &out_val));
  k3_voxel_write<<<static_cast<unsigned>(tiles), kVoxThreads, 0, s>>>(
      c, counts, offsets, out_idx->as<int>(), out_val->as<uint16_t>());
  CSM_LAUNCH_CHECK();
  *d_idx = out_idx->as<int>();
  *d_val = out_val->as<uint16_t>();
  return CSM_OK;
}

}  // namespace csm

using namespace csm;

namespace {

// A zero-filled volume of `box` in *out: whole 32-bit words, since the inserter clears update
// markers with 32-bit atomics (insert3d.cu), and at least 256 bytes.  *out is set once the
// volume is allocated, so the caller owns it even if the fill fails to queue.
template <typename T>
csm_status NewVolume3(const Box3& box, cudaStream_t s, T** out) {
  const size_t bytes = std::max<size_t>((box.Volume() * sizeof(T) + 3) / 4 * 4, 256);
  T* p = nullptr;
  CSM_CUDA(cudaMalloc(&p, bytes));
  *out = p;
  CSM_CUDA(cudaMemsetAsync(p, 0, bytes, s));
  return CSM_OK;
}

// *out: a zero-filled volume of box `to` holding what `old` held over box `from`.
template <typename T>
csm_status Regrow(const T* old, const Box3& from, const Box3& to, cudaStream_t s, T** out) {
  CSM_TRY(NewVolume3(to, s, out));
  k_ins3_copy<T><<<Blocks(static_cast<long long>(from.Volume())), 256, 0, s>>>(old, from, *out,
                                                                              to);
  CSM_LAUNCH_CHECK();
  return CSM_OK;
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
    b.lo[a] = std::max(-kCube, t.lo[a] - s);
    b.n[a] = std::min(kCube - 1, t.hi[a] + s) - b.lo[a] + 1;
  }
  return b;
}

// Installs volume p in *slot, freeing the one it replaces.
template <typename T>
void Install(T* p, T** slot) {
  if (p == *slot) return;
  cudaFree(*slot);
  *slot = p;
}

template <typename Handle>
csm_status Destroy(Handle* grid) {
  if (!grid) return CSM_OK;
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  cudaSetDevice(grid->ctx->device);
  cudaStreamSynchronize(grid->ctx->stream);
  delete grid;
  return CSM_OK;
}

}  // namespace

namespace csm {

GridInsert3::GridInsert3(csm_grid3d* grid, csm_intensity_grid3d* intensity_grid)
    : box(BoxOf(grid->g)), vol(grid->d_vol), grid_(grid), igrid_(intensity_grid) {
  if (!igrid_) return;
  ibox = igrid_->box;
  mean = igrid_->d_vol;
  sum = igrid_->d_sum;
  count = igrid_->d_count;
}

GridInsert3::~GridInsert3() {
  const bool own = vol != grid_->d_vol ||
                   (igrid_ && (mean != igrid_->d_vol || sum != igrid_->d_sum ||
                               count != igrid_->d_count));
  if (!own) return;
  cudaStreamSynchronize(grid_->ctx->stream);
  if (vol != grid_->d_vol) cudaFree(vol);
  if (!igrid_) return;
  if (mean != igrid_->d_vol) cudaFree(mean);
  if (sum != igrid_->d_sum) cudaFree(sum);
  if (count != igrid_->d_count) cudaFree(count);
}

csm_status GridInsert3::Grow(const TightBox3& need, const TightBox3& intensity_need) {
  need_ = need;
  grow_ = !Covers(box, need);
  if (grow_) {
    box = SlackBox(need);
    CSM_REQUIRE(box.Volume() < kMaxVoxels3, "dense volume too large");
  }
  if (!igrid_) return CSM_OK;
  ineed_ = intensity_need;
  igrow_ = !Covers(ibox, intensity_need);
  if (igrow_) {
    ibox = SlackBox(intensity_need);
    CSM_REQUIRE(ibox.Volume() < kMaxIntensityVoxels3, "dense volume too large");
  }
  return CSM_OK;
}

csm_status GridInsert3::Begin() {
  Ctx* ctx = grid_->ctx;
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaSetDevice(ctx->device));
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  if (grow_) CSM_TRY(Regrow(grid_->d_vol, BoxOf(grid_->g), box, s, &vol));
  if (!igrid_) return CSM_OK;
  const Box3& iold = igrid_->box;
  if (igrow_) CSM_TRY(Regrow(igrid_->d_vol, iold, ibox, s, &mean));
  if (!igrid_->d_sum) {   // first insert: the AverageIntensityData of the voxels it was made from
    const long long made = static_cast<long long>(igrid_->made_sum.size());
    CSM_TRY(NewVolume3(ibox, s, &sum));
    CSM_TRY(NewVolume3(ibox, s, &count));
    CSM_TRY(ScatterVoxels3(ctx, igrid_->made_idx.data(), igrid_->made_sum.data(), made, ibox, sum));
    CSM_TRY(ScatterVoxels3(ctx, igrid_->made_idx.data(), igrid_->made_count.data(), made, ibox,
                           count));
  } else if (igrow_) {
    CSM_TRY(Regrow(igrid_->d_sum, iold, ibox, s, &sum));
    CSM_TRY(Regrow(igrid_->d_count, iold, ibox, s, &count));
  }
  return CSM_OK;
}

void GridInsert3::Commit(csm_stats* stats) {
  Ctx* ctx = grid_->ctx;
  Install(vol, &grid_->d_vol);
  grid_->g = MakeGrid3Dev(vol, box, grid_->g.resolution);
  grid_->tight = need_;
  if (igrid_) {
    Install(mean, &igrid_->d_vol);
    Install(sum, &igrid_->d_sum);
    Install(count, &igrid_->d_count);
    igrid_->box = ibox;
    igrid_->tight = ineed_;
    // the volumes hold the list it was made from now
    std::vector<int32_t>().swap(igrid_->made_idx);
    std::vector<int32_t>().swap(igrid_->made_count);
    std::vector<float>().swap(igrid_->made_sum);
  }
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
}

}  // namespace csm

extern "C" {

csm_status csm_grid3d_create(const int32_t* idx, const uint16_t* values, int64_t n,
                             float resolution, int32_t device, csm_grid3d** out) {
  CSM_REQUIRE(out != nullptr, "null pointer");
  CSM_REQUIRE(n >= 0 && (n == 0 || (idx && values)), "voxel list");
  CSM_REQUIRE(resolution > 0.f, "resolution");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_grid3d> g(new csm_grid3d);
  g->ctx = ctx;
  g->tight = ListBox3(idx, n);
  CSM_REQUIRE(g->tight.InCube(), "voxel index outside the 2^14 cube");
  const Box3 box = g->tight.Dense();
  CSM_REQUIRE(box.Volume() < kMaxVoxels3, "dense volume too large");
  CSM_TRY(NewVolume3(box, ctx->stream, &g->d_vol));
  g->g = MakeGrid3Dev(g->d_vol, box, resolution);
  CSM_TRY(ScatterVoxels3(ctx, idx, values, n, box, g->d_vol));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  *out = g.release();
  return CSM_OK;
}

csm_status csm_grid3d_destroy(csm_grid3d* grid) { return Destroy(grid); }

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
  CSM_CUDA(cudaMemcpyAsync(out, grid->d_vol, BoxOf(grid->g).Volume() * sizeof(uint16_t),
                           cudaMemcpyDeviceToHost, grid->ctx->stream));
  CSM_CUDA(cudaStreamSynchronize(grid->ctx->stream));
  return CSM_OK;
}

csm_status csm_grid3d_voxels(const csm_grid3d* grid, int32_t* indices, uint16_t* values,
                             int64_t capacity, int64_t* num_voxels) {
  CSM_REQUIRE(grid && num_voxels, "null pointer");
  CSM_REQUIRE((indices == nullptr) == (values == nullptr), "indices and values go together");
  Ctx* ctx = grid->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  long long n = 0;
  const int* d_idx = nullptr;
  const uint16_t* d_val = nullptr;
  CSM_TRY(DeviceVoxels3D(grid, indices ? capacity : -1, &n, &d_idx, &d_val));
  *num_voxels = n;
  if (!indices || n == 0) return CSM_OK;
  if (capacity < n) {
    SetError("capacity %lld is below the %lld non-zero voxels", static_cast<long long>(capacity), n);
    return CSM_E_CAPACITY;
  }
  cudaStream_t s = ctx->stream;
  CSM_CUDA(cudaMemcpyAsync(indices, d_idx, sizeof(int) * 3 * n, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaMemcpyAsync(values, d_val, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

csm_status csm_grid3d_to_proto(const csm_grid3d* grid, uint8_t* buf, int64_t capacity,
                               int64_t* size) {
  using namespace wire;
  CSM_REQUIRE(grid && size, "null pointer");
  Ctx* ctx = grid->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  long long n = 0;
  const int* d_idx = nullptr;
  const uint16_t* d_val = nullptr;
  CSM_TRY(DeviceVoxels3D(grid, LLONG_MAX, &n, &d_idx, &d_val));
  PinnedBuf& h_idx = ctx->P("g3v_idx");
  PinnedBuf& h_val = ctx->P("g3v_val");
  if (n > 0) {
    CSM_TRY(h_idx.Reserve(sizeof(int) * 3 * n));
    CSM_TRY(h_val.Reserve(sizeof(uint16_t) * n));
    cudaStream_t s = ctx->stream;
    CSM_CUDA(cudaMemcpyAsync(h_idx.p, d_idx, sizeof(int) * 3 * n, cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaMemcpyAsync(h_val.p, d_val, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaStreamSynchronize(s));
  }
  const int* idx = h_idx.as<int>();
  const uint16_t* val = h_val.as<uint16_t>();
  // proto::HybridGrid (hybrid_grid.proto): resolution = 1, packed sint32 x / y / z_indices =
  // 3 / 4 / 5, packed int32 values = 6; HybridGrid::ToProto adds the voxels in iteration order
  int64_t len[4] = {0, 0, 0, 0};
  for (long long i = 0; i < n; ++i) {
    for (int a = 0; a < 3; ++a) len[a] += VarintSize(ZigZag32(idx[3 * i + a]));
    len[3] += VarintSize(val[i]);
  }
  const float resolution = grid->g.resolution;
  int64_t total = FloatFieldSize(resolution);
  if (n > 0)
    for (int f = 0; f < 4; ++f) total += DelimitedSize(len[f]);
  *size = total;
  if (total >= (int64_t(1) << 31)) {
    SetError("a serialized HybridGrid of %lld bytes exceeds protobuf's 2 GiB limit",
             static_cast<long long>(total));
    return CSM_E_CAPACITY;
  }
  if (!buf) return CSM_OK;
  if (capacity < total) {
    SetError("capacity %lld is below the %lld bytes of the message",
             static_cast<long long>(capacity), static_cast<long long>(total));
    return CSM_E_CAPACITY;
  }
  uint8_t* p = PutFloatField(buf, 1, resolution);
  if (n > 0) {
    for (int a = 0; a < 3; ++a) {
      p = PutDelimitedHeader(p, 3 + a, len[a]);
      for (long long i = 0; i < n; ++i) p = PutVarint(p, ZigZag32(idx[3 * i + a]));
    }
    p = PutDelimitedHeader(p, 6, len[3]);
    for (long long i = 0; i < n; ++i) p = PutVarint(p, val[i]);
  }
  return CSM_OK;
}

csm_status csm_intensity_grid3d_create(const int32_t* idx, const float* sum, const int32_t* count,
                                       int64_t n, float resolution, int32_t device,
                                       csm_intensity_grid3d** out) {
  CSM_REQUIRE(out != nullptr, "null pointer");
  CSM_REQUIRE(n >= 0 && (n == 0 || (idx && sum && count)), "voxel list");
  CSM_REQUIRE(resolution > 0.f, "resolution");
  Ctx* ctx;
  CSM_TRY(GetCtx(device, &ctx));
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(device));
  std::unique_ptr<csm_intensity_grid3d> g(new csm_intensity_grid3d);
  g->ctx = ctx;
  g->tight = ListBox3(idx, n);
  CSM_REQUIRE(g->tight.InCube(), "voxel index outside the 2^14 cube");
  g->box = g->tight.Dense();
  CSM_REQUIRE(g->box.Volume() < kMaxIntensityVoxels3, "dense volume too large");
  // IntensityHybridGrid::GetIntensity (hybrid_grid.h:562-569): the float mean, 0 where no
  // intensity was added
  std::vector<float> value(static_cast<size_t>(n));
  for (int64_t i = 0; i < n; ++i) {
    CSM_REQUIRE(count[i] >= 0, "negative intensity count");
    value[i] = count[i] == 0 ? 0.f : sum[i] / static_cast<float>(count[i]);
  }
  CSM_TRY(NewVolume3(g->box, ctx->stream, &g->d_vol));
  g->resolution = resolution;
  CSM_TRY(ScatterVoxels3(ctx, idx, value.data(), n, g->box, g->d_vol));
  CSM_CUDA(cudaStreamSynchronize(ctx->stream));
  // what a first insert fills its sum / count volumes from
  g->made_idx.assign(idx, idx + 3 * n);
  g->made_sum.assign(sum, sum + n);
  g->made_count.assign(count, count + n);
  *out = g.release();
  return CSM_OK;
}

csm_status csm_intensity_grid3d_destroy(csm_intensity_grid3d* grid) { return Destroy(grid); }

csm_status csm_intensity_grid3d_read(const csm_intensity_grid3d* grid, int32_t lo[3],
                                     int32_t dims[3], float* mean, float* sum, int32_t* count) {
  CSM_REQUIRE(grid && lo && dims, "null pointer");
  std::lock_guard<std::mutex> lock(grid->ctx->mu);
  for (int a = 0; a < 3; ++a) {
    lo[a] = grid->box.lo[a];
    dims[a] = grid->box.n[a];
  }
  if (!mean) return CSM_OK;
  CSM_CUDA(cudaSetDevice(grid->ctx->device));
  cudaStream_t s = grid->ctx->stream;
  const size_t vox = grid->box.Volume();
  CSM_CUDA(cudaMemcpyAsync(mean, grid->d_vol, vox * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (grid->d_sum) {
    if (sum) CSM_CUDA(cudaMemcpyAsync(sum, grid->d_sum, vox * 4, cudaMemcpyDeviceToHost, s));
    if (count) CSM_CUDA(cudaMemcpyAsync(count, grid->d_count, vox * 4, cudaMemcpyDeviceToHost, s));
  } else {   // never inserted into: the list it was made from
    if (sum) std::fill(sum, sum + vox, 0.f);
    if (count) std::fill(count, count + vox, 0);
    for (size_t i = 0; i < grid->made_sum.size(); ++i) {
      const int* c = &grid->made_idx[3 * i];
      const size_t k = grid->box.Index(c[0], c[1], c[2]);
      if (sum) sum[k] = grid->made_sum[i];
      if (count) count[k] = grid->made_count[i];
    }
  }
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

}  // extern "C"
