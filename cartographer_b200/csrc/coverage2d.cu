// The coverage pass of OverlappingSubmapsTrimmer2D (mapping/internal/2d/
// overlapping_submaps_trimmer_2d.cc:27-102, 145-182) straight from the submaps' device grids.
//
// The reference files every known cell of every finished submap, moved into the global frame, in
// a std::map keyed by global cell, keeps the fresh_submaps_count freshest entries of each cell and
// counts them per submap.  Here the list of entries is built in the reference's order (submap
// order, then the cells of the cropped limits with x fastest: two passes, a per-tile count and a
// block-scan write), stably radix-sorted by packed cell key, and cut per run of equal keys.  The
// cut is exact on the device except where the reference's std::sort is not stable and the choice
// matters: a cell of more than 16 entries (libstdc++ insertion-sorts 16 or fewer) with a freshness
// tie between different submaps across the cut.  Those cells are read back and sorted on the host
// with the reference's comparator.  Built with -fmad=false: every double expression is the
// reference's, uncontracted.
#include <algorithm>
#include <climits>
#include <cmath>
#include <utility>
#include <vector>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "insert2d.cuh"
#include "rtgrid.cuh"

namespace csm {
namespace {

constexpr int kCovThreads = 256;
constexpr int kCovItems = 4;                           // consecutive cells per thread
constexpr int kCovTile = kCovThreads * kCovItems;      // cells per block
constexpr int kStableSortLimit = 16;                   // libstdc++'s _S_threshold

// One participating submap.  The walk covers the known-cells box (ComputeCroppedLimits); a
// handle whose box was never computed is walked whole, which finds the same cells in the same
// order, since its box is by definition the bounding box of its non-zero cells.
struct CovSubmap {
  const uint16_t* cells;
  int pitch, ox, oy, w;
  long long cells_in_walk;                 // w * h
  double max_x, max_y, resolution;         // the submap grid's own limits
  double t[3], q[4];                       // global_frame_from_local_frame: t, (w, x, y, z)
  long long time;                          // freshness, common::Time ticks
};

struct CovArgs {
  const CovSubmap* sub;
  const long long* tile_start;             // n + 1: the first tile of each submap
  int n;
  double off_x, off_y, res;                // the first submap's limits
};

// Device-side totals read back with the counts.
struct CovHeader {
  unsigned long long coverage_cells;
  unsigned long long device_tie_cells;     // ties across the cut settled in list order
  unsigned long long host_cells;           // ambiguous cells left to the host
  unsigned long long host_entries;
  int overflow;                            // a key outside int32
  int pad;
};

__device__ __forceinline__ int SubmapOfTile(const CovArgs& a, long long tile) {
  int lo = 0, hi = a.n - 1;   // the last submap whose first tile is <= tile
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.tile_start[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The known flags of this thread's kCovItems consecutive cells of the block's tile.
__device__ __forceinline__ int TileCells(const CovArgs& a, int* sub, long long* first,
                                         bool known[kCovItems]) {
  const long long tile = blockIdx.x;
  const int i = SubmapOfTile(a, tile);
  const CovSubmap& s = a.sub[i];
  *sub = i;
  *first = (tile - a.tile_start[i]) * kCovTile + threadIdx.x * kCovItems;
  int n = 0;
#pragma unroll
  for (int k = 0; k < kCovItems; ++k) {
    const long long c = *first + k;
    known[k] = false;
    if (c < s.cells_in_walk) {
      const int x = static_cast<int>(c % s.w), y = static_cast<int>(c / s.w);
      known[k] = s.cells[static_cast<size_t>(y + s.oy) * s.pitch + (x + s.ox)] != 0;   // IsKnown
    }
    n += known[k];
  }
  return n;
}

// Pass 1: counts[tile] = the known cells of the tile.
__global__ void __launch_bounds__(kCovThreads) k_cov_count(CovArgs a, long long* __restrict__ counts) {
  typedef cub::BlockReduce<int, kCovThreads> Reduce;
  __shared__ typename Reduce::TempStorage red;
  int sub;
  long long first;
  bool known[kCovItems];
  const int n = Reduce(red).Sum(TileCells(a, &sub, &first, known));
  if (threadIdx.x == 0) counts[blockIdx.x] = n;
}

// Eigen's _transformVector (uv = vec x c; uv += uv; c + w * uv + vec x uv) and then + t, the
// translation of Rigid3d operator* (rigid_transform.h:184-189) for a rotation-free right side.
__device__ __forceinline__ void Transform(const double* q, const double* t, const double c[3],
                                          double p[3]) {
  const double w = q[0], v[3] = {q[1], q[2], q[3]};
  double uv[3] = {__dsub_rn(__dmul_rn(v[1], c[2]), __dmul_rn(v[2], c[1])),
                  __dsub_rn(__dmul_rn(v[2], c[0]), __dmul_rn(v[0], c[2])),
                  __dsub_rn(__dmul_rn(v[0], c[1]), __dmul_rn(v[1], c[0]))};
  for (int k = 0; k < 3; ++k) uv[k] = __dadd_rn(uv[k], uv[k]);
  const double x[3] = {__dsub_rn(__dmul_rn(v[1], uv[2]), __dmul_rn(v[2], uv[1])),
                       __dsub_rn(__dmul_rn(v[2], uv[0]), __dmul_rn(v[0], uv[2])),
                       __dsub_rn(__dmul_rn(v[0], uv[1]), __dmul_rn(v[1], uv[0]))};
  for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(__dadd_rn(__dadd_rn(c[k], __dmul_rn(w, uv[k])), x[k]), t[k]);
}

// RoundToInt64((offset - p) / resolution) (SubmapCoverageGrid2D::AddPoint) into an
// order-preserving 32-bit image; false outside int32.
__device__ __forceinline__ bool CellKey(double offset, double p, double res, unsigned* key) {
  const double v = __ddiv_rn(__dsub_rn(offset, p), res);
  if (!(v > -4.0e9 && v < 4.0e9)) return false;
  const long long k = llround(v);   // half away from zero, as std::lround
  if (k < INT_MIN || k > INT_MAX) return false;
  *key = static_cast<unsigned>(static_cast<int>(k)) ^ 0x80000000u;
  return true;
}

// Pass 2: the entries of the tile from offsets[tile] on, in walk order: the packed global cell
// key (x key high, y key low: std::map's pair order), the entry's list position and its submap.
__global__ void __launch_bounds__(kCovThreads)
k_cov_write(CovArgs a, const long long* __restrict__ counts, const long long* __restrict__ offsets,
            unsigned long long* __restrict__ keys, unsigned* __restrict__ pos,
            int* __restrict__ entry_sub, CovHeader* __restrict__ hdr) {
  typedef cub::BlockScan<int, kCovThreads> Scan;
  __shared__ typename Scan::TempStorage scan;
  if (counts[blockIdx.x] == 0) return;   // uniform over the block
  int i;
  long long first;
  bool known[kCovItems];
  const int n = TileCells(a, &i, &first, known);
  int before;
  Scan(scan).ExclusiveSum(n, before);
  long long o = offsets[blockIdx.x] + before;
  const CovSubmap& s = a.sub[i];
  bool overflow = false;
#pragma unroll
  for (int k = 0; k < kCovItems; ++k) {
    if (!known[k]) continue;
    const long long c = first + k;
    const int ix = static_cast<int>(c % s.w) + s.ox, iy = static_cast<int>(c / s.w) + s.oy;
    // the cell centre in the local frame (overlapping_submaps_trimmer_2d.cc:83-88)
    const double centre[3] = {
        __dsub_rn(s.max_x, __dmul_rn(s.resolution, __dadd_rn(static_cast<double>(iy), 0.5))),
        __dsub_rn(s.max_y, __dmul_rn(s.resolution, __dadd_rn(static_cast<double>(ix), 0.5))), 0.};
    double p[3];
    Transform(s.q, s.t, centre, p);
    unsigned kx = 0, ky = 0;
    if (!CellKey(a.off_x, p[0], a.res, &kx) || !CellKey(a.off_y, p[1], a.res, &ky)) overflow = true;
    keys[o] = (static_cast<unsigned long long>(kx) << 32) | ky;
    pos[o] = static_cast<unsigned>(o);
    entry_sub[o] = i;
    ++o;
  }
  if (overflow) atomicOr(&hdr->overflow, 1);
}

struct HostCell {   // a cell left to the host: its entries' submaps at [offset, offset + n)
  unsigned offset, n;
};

// FindSubmapIdsToTrim's per-cell cut (:150-170), one thread per run of equal keys in the stably
// sorted list, whose entries are then in list order.  Adds each kept entry to its submap's count,
// or hands the cell to the host.
__global__ void __launch_bounds__(kCovThreads)
k_cov_cut(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ pos,
          long long total, const int* __restrict__ entry_sub, const CovSubmap* __restrict__ sub,
          int fresh, unsigned* __restrict__ counts, CovHeader* __restrict__ hdr,
          HostCell* __restrict__ host_cells, int* __restrict__ host_subs) {
  const long long j = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (j >= total) return;
  const unsigned long long key = keys[j];
  if (j > 0 && keys[j - 1] == key) return;
  long long end = j + 1;
  while (end < total && keys[end] == key) ++end;
  const int n = static_cast<int>(end - j);
  atomicAdd(&hdr->coverage_cells, 1ull);
  if (n <= fresh) {   // no cut
    for (long long k = j; k < end; ++k) atomicAdd(&counts[entry_sub[pos[k]]], 1u);
    return;
  }
  if (fresh == 0) return;   // erase(begin() + 0, end())
  // the fresh-th largest time T*, walking the distinct times downwards; `newer` entries are above
  long long t_star = 0;
  int newer = 0, tied = 0;
  bool first = true;
  for (;;) {
    long long v = LLONG_MIN;
    bool any = false;
    for (long long k = j; k < end; ++k) {
      const long long t = sub[entry_sub[pos[k]]].time;
      if ((first || t < t_star) && (!any || t > v)) {
        v = t;
        any = true;
      }
    }
    int c = 0;
    for (long long k = j; k < end; ++k) c += sub[entry_sub[pos[k]]].time == v;
    first = false;
    t_star = v;
    if (newer + c >= fresh) {
      tied = c;
      break;
    }
    newer += c;
  }
  const int take = fresh - newer;   // of the `tied` entries at T*
  int tie_sub = -1;
  bool one_submap = true;
  for (long long k = j; k < end; ++k) {
    const int s = entry_sub[pos[k]];
    if (sub[s].time != t_star) continue;
    if (tie_sub < 0) tie_sub = s; else if (s != tie_sub) one_submap = false;
  }
  if (take < tied && !one_submap) {
    if (n > kStableSortLimit) {   // std::sort's order among the tied entries is not list order
      const unsigned slot = static_cast<unsigned>(atomicAdd(&hdr->host_cells, 1ull));
      const unsigned at = static_cast<unsigned>(atomicAdd(&hdr->host_entries,
                                                          static_cast<unsigned long long>(n)));
      host_cells[slot] = HostCell{at, static_cast<unsigned>(n)};
      for (long long k = j; k < end; ++k) host_subs[at + (k - j)] = entry_sub[pos[k]];
      return;
    }
    atomicAdd(&hdr->device_tie_cells, 1ull);   // insertion sort: stable
  }
  int taken = 0;
  for (long long k = j; k < end; ++k) {
    const int s = entry_sub[pos[k]];
    const long long t = sub[s].time;
    if (t > t_star || (t == t_star && taken++ < take)) atomicAdd(&counts[s], 1u);
  }
}

}  // namespace
}  // namespace csm

using namespace csm;

extern "C" {

csm_status csm_trim_overlapping_submaps2d(const csm_coverage_submap2d* submaps, int32_t n,
                                          double first_max_x, double first_max_y,
                                          double first_resolution, uint16_t fresh_submaps_count,
                                          uint16_t min_covered_cells_count, uint8_t* trim,
                                          uint32_t* covered_entries, csm_coverage_stats2d* stats) {
  CSM_REQUIRE(n >= 0, "negative submap count");
  CSM_REQUIRE(n == 0 || (submaps != nullptr && trim != nullptr && covered_entries != nullptr),
              "null pointer");
  CSM_REQUIRE(std::isfinite(first_max_x) && std::isfinite(first_max_y) &&
                  std::isfinite(first_resolution) && first_resolution > 0., "first limits");
  if (stats) *stats = csm_coverage_stats2d{};
  if (n == 0) return CSM_OK;
  for (int32_t i = 0; i < n; ++i) {
    const csm_coverage_submap2d& s = submaps[i];
    CSM_REQUIRE(s.grid != nullptr, "null grid");
    CSM_REQUIRE(Finite(s.translation, 3) && Finite(s.rotation, 4), "non-finite pose");
    CSM_REQUIRE(s.grid->ctx == submaps[0].grid->ctx, "handles on more than one device");
  }
  Ctx* ctx = submaps[0].grid->ctx;
  std::lock_guard<std::mutex> lock(ctx->mu);
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  int syncs = 0;

  // the submap records and their first tiles, uploaded in one copy
  const size_t o_tiles = (sizeof(CovSubmap) * n + 255) / 256 * 256;
  const size_t rec_bytes = o_tiles + sizeof(long long) * (n + 1);
  PinnedBuf& h_rec = ctx->P("cov_rec");
  CSM_TRY(h_rec.Reserve(rec_bytes));
  CovSubmap* rec = h_rec.as<CovSubmap>();
  long long* tile_start = reinterpret_cast<long long*>(h_rec.as<char>() + o_tiles);
  long long tiles = 0;
  for (int32_t i = 0; i < n; ++i) {
    const csm_rt_grid2d* g = submaps[i].grid;
    CovSubmap& r = rec[i];
    r.cells = g->d_cells;
    r.pitch = g->g.pitch;
    if (g->known_stale) {   // the bounding box of the non-zero cells: walk the whole grid
      r.ox = r.oy = 0;
      r.w = g->g.nx;
      r.cells_in_walk = static_cast<long long>(g->g.nx) * g->g.ny;
    } else if (g->known.empty()) {   // ComputeCroppedLimits: 1 x 1 at offset (0, 0)
      r.ox = r.oy = 0;
      r.w = 1;
      r.cells_in_walk = 1;
    } else {
      r.ox = g->known.lo[0];
      r.oy = g->known.lo[1];
      r.w = g->known.hi[0] - r.ox + 1;
      r.cells_in_walk = static_cast<long long>(r.w) * (g->known.hi[1] - r.oy + 1);
    }
    r.max_x = g->g.max_x;
    r.max_y = g->g.max_y;
    r.resolution = g->g.resolution;
    for (int k = 0; k < 3; ++k) r.t[k] = submaps[i].translation[k];
    for (int k = 0; k < 4; ++k) r.q[k] = submaps[i].rotation[k];
    r.time = submaps[i].freshness;
    tile_start[i] = tiles;
    tiles += (r.cells_in_walk + kCovTile - 1) / kCovTile;
  }
  tile_start[n] = tiles;
  if (tiles >= INT_MAX) {   // one block per tile
    SetError("%lld cell tiles are too many to walk", tiles);
    return CSM_E_CAPACITY;
  }
  DevBuf* d_rec;
  CSM_TRY(ctx->Reserve("cov_rec", rec_bytes, &d_rec));
  CSM_CUDA(cudaMemcpyAsync(d_rec->p, rec, rec_bytes, cudaMemcpyHostToDevice, s));
  CovArgs a;
  a.sub = d_rec->as<CovSubmap>();
  a.tile_start = reinterpret_cast<const long long*>(d_rec->as<char>() + o_tiles);
  a.n = n;
  a.off_x = first_max_x;
  a.off_y = first_max_y;
  a.res = first_resolution;

  // pass 1 and the exclusive scan of the tile counts (counts[tiles] stays 0: the total)
  size_t scan_bytes = 0;
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<long long*>(nullptr),
                                         static_cast<long long*>(nullptr), tiles + 1, s));
  const size_t o_off = (sizeof(long long) * (tiles + 1) + 255) / 256 * 256;
  const size_t o_hdr = 2 * o_off;
  const size_t o_scan = o_hdr + 256;
  DevBuf* d_tiles;
  CSM_TRY(ctx->Reserve("cov_tiles", o_scan + scan_bytes, &d_tiles));
  long long* tile_counts = d_tiles->as<long long>();
  long long* tile_offsets = reinterpret_cast<long long*>(d_tiles->as<char>() + o_off);
  CovHeader* d_hdr = reinterpret_cast<CovHeader*>(d_tiles->as<char>() + o_hdr);
  CSM_CUDA(cudaMemsetAsync(tile_counts + tiles, 0, sizeof(long long), s));
  CSM_CUDA(cudaMemsetAsync(d_hdr, 0, sizeof(CovHeader), s));
  if (tiles > 0) {
    k_cov_count<<<static_cast<unsigned>(tiles), kCovThreads, 0, s>>>(a, tile_counts);
    CSM_LAUNCH_CHECK();
  }
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(d_tiles->as<char>() + o_scan, scan_bytes, tile_counts,
                                         tile_offsets, tiles + 1, s));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  PinnedBuf& h_total = ctx->P("cov_total");
  CSM_TRY(h_total.Reserve(sizeof(long long)));
  CSM_CUDA(cudaMemcpyAsync(h_total.p, tile_offsets + tiles, sizeof(long long),
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  ++syncs;
  const long long total = *h_total.as<long long>();

  std::vector<uint32_t> count(n, 0u);
  CovHeader hdr{};
  if (total > 0) {
    if (total >= INT_MAX) {   // the sort's item count
      SetError("%lld coverage entries are too many to sort", total);
      return CSM_E_CAPACITY;
    }
    // keys and positions twice (the sort's double buffers), the entries' submaps, the counts,
    // the cells left to the host (each holds more than kStableSortLimit entries: at most
    // total / 17 records and total entries' submaps) and the sort's scratch, each region
    // rounded up to 256 bytes
    size_t sort_bytes = 0;
    cub::DoubleBuffer<unsigned long long> k0(nullptr, nullptr);
    cub::DoubleBuffer<unsigned> v0(nullptr, nullptr);
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, k0, v0, static_cast<int>(total),
                                             0, 64, s));
    auto lane = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t o_k1 = lane(sizeof(unsigned long long) * total);
    const size_t o_v0 = 2 * o_k1;
    const size_t o_v1 = o_v0 + lane(sizeof(unsigned) * total);
    const size_t o_sub = o_v1 + lane(sizeof(unsigned) * total);
    const size_t o_cnt = o_sub + lane(sizeof(int) * total);
    const size_t o_hsub = o_cnt + lane(sizeof(unsigned) * n);
    const size_t o_hcell = o_hsub + lane(sizeof(int) * total);
    const size_t o_sort =
        o_hcell + lane(sizeof(HostCell) * (total / (kStableSortLimit + 1) + 1));
    const size_t need = o_sort + sort_bytes;
    DevBuf& work = ctx->D("cov_work");
    if (need > work.cap) {
      size_t free_bytes = 0, total_bytes = 0;
      CSM_CUDA(cudaMemGetInfo(&free_bytes, &total_bytes));
      if (need > free_bytes + work.cap) {
        SetError("%lld coverage entries need %zu bytes of device memory, %zu are free", total,
                 need, free_bytes + work.cap);
        return CSM_E_CAPACITY;
      }
    }
    CSM_TRY(work.Reserve(need));
    char* base = work.as<char>();
    unsigned long long* keys0 = reinterpret_cast<unsigned long long*>(base);
    unsigned long long* keys1 = reinterpret_cast<unsigned long long*>(base + o_k1);
    unsigned* pos0 = reinterpret_cast<unsigned*>(base + o_v0);
    unsigned* pos1 = reinterpret_cast<unsigned*>(base + o_v1);
    int* entry_sub = reinterpret_cast<int*>(base + o_sub);
    unsigned* d_count = reinterpret_cast<unsigned*>(base + o_cnt);
    CSM_CUDA(cudaMemsetAsync(d_count, 0, sizeof(unsigned) * n, s));
    k_cov_write<<<static_cast<unsigned>(tiles), kCovThreads, 0, s>>>(
        a, tile_counts, tile_offsets, keys0, pos0, entry_sub, d_hdr);
    CSM_LAUNCH_CHECK();
    cub::DoubleBuffer<unsigned long long> dk(keys0, keys1);
    cub::DoubleBuffer<unsigned> dv(pos0, pos1);
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(base + o_sort, sort_bytes, dk, dv,
                                             static_cast<int>(total), 0, 64, s));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    int* host_subs = reinterpret_cast<int*>(base + o_hsub);
    HostCell* host_cells = reinterpret_cast<HostCell*>(base + o_hcell);
    k_cov_cut<<<DivUp(total, kCovThreads), kCovThreads, 0, s>>>(
        dk.Current(), dv.Current(), total, entry_sub, a.sub, fresh_submaps_count, d_count, d_hdr,
        host_cells, host_subs);
    CSM_LAUNCH_CHECK();
    PinnedBuf& h_out = ctx->P("cov_out");
    CSM_TRY(h_out.Reserve(sizeof(CovHeader) + sizeof(unsigned) * n));
    CSM_CUDA(cudaMemcpyAsync(h_out.p, d_hdr, sizeof(CovHeader), cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaMemcpyAsync(h_out.as<char>() + sizeof(CovHeader), d_count, sizeof(unsigned) * n,
                             cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaStreamSynchronize(s));
    ++syncs;
    std::memcpy(&hdr, h_out.p, sizeof(CovHeader));
    std::memcpy(count.data(), h_out.as<char>() + sizeof(CovHeader), sizeof(unsigned) * n);
    if (hdr.overflow) {
      SetError("a submap cell lies outside the int32 range of global cell keys");
      return CSM_E_CAPACITY;
    }
    if (hdr.host_cells > 0) {
      // the reference's std::sort on each ambiguous cell's entries in list order
      const size_t cell_bytes = sizeof(HostCell) * hdr.host_cells;
      const size_t sub_bytes = sizeof(int) * hdr.host_entries;
      PinnedBuf& h_host = ctx->P("cov_host");
      CSM_TRY(h_host.Reserve(cell_bytes + sub_bytes));
      CSM_CUDA(cudaMemcpyAsync(h_host.p, host_cells, cell_bytes, cudaMemcpyDeviceToHost, s));
      CSM_CUDA(cudaMemcpyAsync(h_host.as<char>() + cell_bytes, host_subs, sub_bytes,
                               cudaMemcpyDeviceToHost, s));
      CSM_CUDA(cudaStreamSynchronize(s));
      ++syncs;
      const HostCell* cells = h_host.as<HostCell>();
      const int* subs = reinterpret_cast<const int*>(h_host.as<char>() + cell_bytes);
      std::vector<std::pair<int, int64_t>> entries;
      for (unsigned long long c = 0; c < hdr.host_cells; ++c) {
        entries.clear();
        for (unsigned k = 0; k < cells[c].n; ++k) {
          const int i = subs[cells[c].offset + k];
          entries.emplace_back(i, submaps[i].freshness);
        }
        std::sort(entries.begin(), entries.end(),
                  [](const std::pair<int, int64_t>& left, const std::pair<int, int64_t>& right) {
                    return left.second > right.second;
                  });
        for (int k = 0; k < fresh_submaps_count; ++k) ++count[entries[k].first];
      }
    }
  }
  // std::map<SubmapId, uint16>: absent (0 entries) or a wrapped count below the minimum
  for (int32_t i = 0; i < n; ++i) {
    covered_entries[i] = count[i];
    trim[i] = count[i] == 0u || static_cast<uint16_t>(count[i]) < min_covered_cells_count;
  }
  if (stats) {
    stats->entries = total;
    stats->coverage_cells = static_cast<int64_t>(hdr.coverage_cells);
    stats->device_tie_cells = static_cast<int64_t>(hdr.device_tie_cells);
    stats->host_sorted_cells = static_cast<int64_t>(hdr.host_cells);
    stats->host_syncs = syncs;
  }
  return CSM_OK;
}

}  // extern "C"
