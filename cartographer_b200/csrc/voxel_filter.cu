// sensor::VoxelFilter and sensor::AdaptiveVoxelFilter (sensor/internal/voxel_filter.cc) on the
// device, bit for bit: the kept input indices equal what the reference's reservoir sampling keeps.
//
// The reference walks the cloud once with one std::minstd_rand0 (seed 1, fresh per call): the
// m-th point, in input order, whose voxel already holds a point draws
// uniform_int_distribution<int>(1, k)(generator), k its 1-based rank in that voxel, and replaces
// the voxel's sample when the draw is k.  libstdc++ draws for this generator's range by scaling
// (scaling = (2^31 - 3) / k, past = k * scaling; ret = g() - 1 until ret < past; ret / scaling + 1),
// and the generator's j-th output is 16807^j mod (2^31 - 1).  So with the voxels' ranks from a
// stable sort, every call's draw is found by skip-ahead, and the only sequential coupling is a
// rejected draw (ret >= past), which shifts every later call by one raw draw.  Rejections are rare
// (about k / 2^31 per call): each call tests 64 shifts at once, one thread per cloud walks the few
// calls that reject under some shift and fixes the shifts in order, and past 63 extra draws in one
// cloud it steps the remaining calls one by one.  DESIGN §9 has the argument.
//
// The adaptive search (voxel_filter.cc:38-75) only needs the number of distinct voxel keys per
// trial length, counted with a per-cloud hash set; its per-cloud state lives on the device, so
// a batch is one fixed launch sequence and one stream synchronisation.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "common.cuh"
#include "point_batch.cuh"
#include "voxel_filter.cuh"

namespace csm {
namespace {

constexpr uint64_t kModulus = 2147483647ull;      // minstd_rand0: 16807^j mod (2^31 - 1)
constexpr uint64_t kUrngRange = 2147483645ull;    // max() - min() = (2^31 - 2) - 1
constexpr int kShiftWindow = 64;                  // shifts one call tests at once
constexpr unsigned long long kEmptySlot = ~0ull;  // hash-set sentinel (that key is flagged aside)
constexpr int kHalvingSteps = 7;                  // high > 1e-2 * max_length: L .. L / 64
constexpr int kBisectionSteps = 8;                // the ratio halves per step from 1 to <= 0.1
constexpr int kThreads = 256;

__host__ __device__ inline uint64_t MulMod(uint64_t a, uint64_t b) {
  uint64_t x = a * b;                              // < 2^62
  x = (x & kModulus) + (x >> 31);
  x = (x & kModulus) + (x >> 31);
  return x >= kModulus ? x - kModulus : x;
}

// The generator's j-th output (j >= 1): 16807^j mod (2^31 - 1).
__device__ inline uint64_t Draw(uint64_t j) {
  uint64_t r = 1, b = 16807;
  while (j) {
    if (j & 1) r = MulMod(r, b);
    b = MulMod(b, b);
    j >>= 1;
  }
  return r;
}

__device__ inline uint64_t Past(int k) {
  const uint64_t uk = static_cast<uint64_t>(k);
  return uk * (kUrngRange / uk);
}

// GetVoxelCellIndex (voxel_filter.cc:79-86), wrapping.
__device__ inline unsigned long long VoxelKey(const float* p, float resolution) {
  const uint64_t x = static_cast<uint64_t>(static_cast<int64_t>(RoundToInt(p[0] / resolution)));
  const uint64_t y = static_cast<uint64_t>(static_cast<int64_t>(RoundToInt(p[1] / resolution)));
  const uint64_t z = static_cast<uint64_t>(static_cast<int64_t>(RoundToInt(p[2] / resolution)));
  return (x << 42) + (y << 21) + z;
}

// Per-cloud search state (voxel_filter.cc:38-75).  The output is VoxelFilter(length) of the
// range-filtered cloud, or that cloud itself when `keep_all`.
enum Phase : int { kFirst = 0, kHalving = 1, kBisection = 2, kDone = 3 };
struct CloudState {
  float max_length, min_num_points, high, low, mid, length;
  int phase, keep_all, bisection_steps, error;
};

// ---- range filter and the adaptive search --------------------------------------------------

// A point outside `pre_active` (when given) is not in the cloud at all: the batch then filters
// the subsequence of points it flags, in order.
__global__ void k_vf_range(const float* __restrict__ xyz, const int* __restrict__ off, int nc,
                           const float* __restrict__ max_range,
                           const unsigned char* __restrict__ pre_active, int n,
                           unsigned char* active, int* num_active) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = CloudOf(off, nc, i);
  const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
  const bool in = (pre_active == nullptr || pre_active[i]) &&
                  sqrtf((x * x + y * y) + z * z) <= max_range[c];   // FilterByMaxRange (:31-36)
  active[i] = in;
  if (in) atomicAdd(&num_active[c], 1);
}

__global__ void k_vf_start(CloudState* st, const int* num_active, int nc) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  CloudState& s = st[c];
  if (static_cast<float>(num_active[c]) <= s.min_num_points) {   // :40-43
    s.keep_all = 1;
    s.phase = kDone;
  } else {
    s.length = s.max_length;
    s.phase = kFirst;
  }
}

// Inserts the key of every active point of a searching cloud into that cloud's hash set and
// counts the keys inserted first.
__global__ void k_vf_count(const float* __restrict__ xyz, const int* __restrict__ off, int nc,
                           const unsigned char* __restrict__ active, int n,
                           const CloudState* __restrict__ st, unsigned long long* table,
                           const long long* __restrict__ table_off, int* empty_key_seen,
                           int* distinct) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !active[i]) return;
  const int c = CloudOf(off, nc, i);
  if (st[c].phase == kDone) return;
  const unsigned long long key = VoxelKey(xyz + 3 * i, st[c].length);
  bool inserted;
  if (key == kEmptySlot) {
    inserted = atomicExch(&empty_key_seen[c], 1) == 0;
  } else {
    unsigned long long* t = table + table_off[c];
    const uint64_t mask = static_cast<uint64_t>(table_off[c + 1] - table_off[c]) - 1;
    uint64_t h = Mix(key) & mask;
    for (;;) {
      const unsigned long long old = atomicCAS(&t[h], kEmptySlot, key);
      if (old == kEmptySlot) { inserted = true; break; }
      if (old == key) { inserted = false; break; }
      h = (h + 1) & mask;
    }
  }
  if (inserted) atomicAdd(&distinct[c], 1);
}

// One step of AdaptivelyVoxelFiltered's search per cloud, from the distinct-key count of the
// length just tried; resets the counters for the next trial.
__global__ void k_vf_decide(CloudState* st, int* distinct, int* empty_key_seen, int nc) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  CloudState& s = st[c];
  const bool dense = static_cast<float>(distinct[c]) >= s.min_num_points;
  distinct[c] = 0;
  empty_key_seen[c] = 0;
  const float L = s.max_length;
  switch (s.phase) {
    case kFirst:                                           // :44-48
      if (dense) { s.phase = kDone; break; }
      s.high = L;
      s.low = s.high / 2.f;                                // high > 1e-2 * L holds for L > 0
      s.length = s.low;
      s.phase = kHalving;
      break;
    case kHalving:                                         // :52-71
      if (dense) {
        if ((s.high - s.low) / s.low > 1e-1f) {
          s.mid = (s.low + s.high) / 2.f;
          s.length = s.mid;
          s.phase = kBisection;
        } else {
          s.phase = kDone;                                 // result = VoxelFilter(low)
        }
        break;
      }
      s.high /= 2.f;
      if (s.high > 1e-2f * L) {
        s.low = s.high / 2.f;
        s.length = s.low;
      } else {
        s.phase = kDone;                                   // :74: the last VoxelFilter(low)
      }
      break;
    case kBisection:                                       // :59-68
      if (dense) s.low = s.mid; else s.high = s.mid;
      if ((s.high - s.low) / s.low > 1e-1f) {
        if (++s.bisection_steps >= kBisectionSteps) {
          s.error = 1;
          s.phase = kDone;
          break;
        }
        s.mid = (s.low + s.high) / 2.f;
        s.length = s.mid;
      } else {
        s.length = s.low;
        s.phase = kDone;
      }
      break;
    default:
      break;
  }
}

// ---- VoxelFilter(length) of the active points ------------------------------------------------

// Sort keys: the voxel key, then (second, stable pass) the cloud, with the active points of
// keep-all clouds and the inactive points behind every cloud (cloud id nc).
__global__ void k_vf_keys(const float* __restrict__ xyz, const int* __restrict__ off, int nc,
                          const unsigned char* __restrict__ active, int n,
                          const CloudState* __restrict__ st, unsigned long long* keys,
                          int* vals, unsigned char* kept) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = CloudOf(off, nc, i);
  const bool in = active == nullptr || active[i];
  const bool all = in && st[c].keep_all;
  keys[i] = (in && !all) ? VoxelKey(xyz + 3 * i, st[c].length) : 0ull;
  vals[i] = i;
  kept[i] = all;
}

__global__ void k_vf_cloud_ids(const int* __restrict__ off, int nc,
                               const unsigned char* __restrict__ active,
                               const CloudState* __restrict__ st, const int* __restrict__ vals,
                               int n, unsigned* cid) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int i = vals[j];
  const int c = CloudOf(off, nc, i);
  const bool in = (active == nullptr || active[i]) && !st[c].keep_all;
  cid[j] = in ? c : nc;
}

// Group starts in (cloud, key, index) order.
__global__ void k_vf_starts(const unsigned* __restrict__ cid, const int* __restrict__ vals,
                            const unsigned long long* __restrict__ keys, int nc, int n,
                            int* start) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const unsigned c = cid[j];
  start[j] = c != static_cast<unsigned>(nc) &&
             (j == 0 || cid[j - 1] != c || keys[vals[j - 1]] != keys[vals[j]]);
}

__global__ void k_vf_group_starts(const int* __restrict__ start, const int* __restrict__ group,
                                  int n, int* group_start) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n && start[j]) group_start[group[j] - 1] = j;
}

// Per active point, in input order: its rank in its voxel and its voxel (group) number.
__global__ void k_vf_ranks(const unsigned* __restrict__ cid, const int* __restrict__ vals,
                           const int* __restrict__ group, const int* __restrict__ group_start,
                           int nc, int n, int* rank_in, int* group_in, int* is_call) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || cid[j] == static_cast<unsigned>(nc)) return;
  const int g = group[j] - 1;
  const int i = vals[j];
  const int rank = j - group_start[g] + 1;
  rank_in[i] = rank;
  group_in[i] = g;
  is_call[i] = rank >= 2;
}

// One record per distribution call: its k, its cloud and its call number within the cloud;
// the shifts (0 .. 63 extra raw draws before it) under which its first draw is rejected.
__global__ void k_vf_calls(const int* __restrict__ off, int nc, const int* __restrict__ rank_in,
                           const int* __restrict__ call, int n, int* call_k,
                           unsigned long long* call_mask, unsigned char* call_flag,
                           unsigned long long* ecode) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = rank_in[i];
  if (k < 2) return;
  const int c = CloudOf(off, nc, i);
  const int m = call[i];
  const int local = m - call[off[c]];
  call_k[m] = k;
  const uint64_t past = Past(k);
  uint64_t x = Draw(static_cast<uint64_t>(local) + 1);
  unsigned long long mask = 0;
  for (int e = 0; e < kShiftWindow; ++e) {
    if (x - 1 >= past) mask |= 1ull << e;
    x = MulMod(x, 16807);
  }
  call_mask[m] = mask;
  call_flag[m] = mask != 0;
  ecode[m] = static_cast<unsigned long long>(c) << 32;
}

// One thread per cloud: the calls that reject under some shift, in order.  E is the number of
// extra raw draws before the current call; a call whose draw at E is rejected draws on until one
// is accepted, and records the new E (as cloud << 32 | E) for the max-scan that hands every later
// call its E.  Beyond the tested window the thread checks every remaining call itself.
__global__ void k_vf_walk(const int* __restrict__ off, int nc, const int* __restrict__ call,
                          const int* __restrict__ cand, const int* __restrict__ num_cand,
                          const int* __restrict__ call_k,
                          const unsigned long long* __restrict__ call_mask,
                          unsigned long long* ecode) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  const int first = call[off[c]], end = call[off[c + 1]];
  int lo = 0, hi = *num_cand;                      // first candidate >= first
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (cand[mid] < first) lo = mid + 1; else hi = mid;
  }
  uint64_t E = 0;
  int m = -1;
  for (int t = lo; t < *num_cand && cand[t] < end && E < kShiftWindow; ++t) {
    m = cand[t];
    if (!((call_mask[m] >> E) & 1)) continue;
    const uint64_t past = Past(call_k[m]);
    uint64_t x = Draw(static_cast<uint64_t>(m - first) + 1 + E);
    while (x - 1 >= past) {
      ++E;
      x = MulMod(x, 16807);
    }
    ecode[m] = (static_cast<unsigned long long>(c) << 32) | E;
  }
  if (E < kShiftWindow) return;
  uint64_t x = 0;
  for (int mm = m + 1; mm < end; ++mm) {           // past the window: every call in turn
    x = x ? MulMod(x, 16807) : Draw(static_cast<uint64_t>(mm - first) + 1 + E);
    const uint64_t past = Past(call_k[mm]);
    bool rejected = false;
    while (x - 1 >= past) {
      ++E;
      x = MulMod(x, 16807);
      rejected = true;
    }
    if (rejected) ecode[mm] = (static_cast<unsigned long long>(c) << 32) | E;
  }
}

// Each call's accepted draw; a call drawing k bids for its voxel with its rank.
__global__ void k_vf_hits(const int* __restrict__ off, int nc, const int* __restrict__ rank_in,
                          const int* __restrict__ group_in, const int* __restrict__ call,
                          const unsigned long long* __restrict__ eincl, int n, int* best) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = rank_in[i];
  if (k < 2) return;
  const int c = CloudOf(off, nc, i);
  const int m = call[i];
  const unsigned long long e = eincl[m];
  const uint64_t E = (e >> 32) == static_cast<unsigned long long>(c) ? (e & 0xffffffffull) : 0;
  const uint64_t j = static_cast<uint64_t>(m - call[off[c]]) + 1 + E;
  const uint64_t uk = static_cast<uint64_t>(k);
  const uint64_t ret = Draw(j) - 1;
  if (ret / (kUrngRange / uk) + 1 == uk) atomicMax(&best[group_in[i]], k);
}

// The voxel keeps its highest-ranked point that drew its own rank, else its first point.
__global__ void k_vf_keep(const unsigned* __restrict__ cid, const int* __restrict__ vals,
                          const int* __restrict__ rank_in, const int* __restrict__ group_in,
                          const int* __restrict__ best, int nc, int n, unsigned char* kept) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || cid[j] == static_cast<unsigned>(nc)) return;
  const int i = vals[j];
  if (rank_in[i] == max(1, best[group_in[i]])) kept[i] = 1;
}

// Kept counts per cloud, then the kept indices made relative to their cloud.
__global__ void k_vf_counts(const int* __restrict__ off, int nc, const int* __restrict__ out,
                            const int* __restrict__ num_out, int* counts) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nc) return;
  auto lower = [&](int v) {
    int lo = 0, hi = *num_out;
    while (lo < hi) {
      const int mid = (lo + hi) / 2;
      if (out[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
  };
  counts[c] = lower(off[c + 1]) - lower(off[c]);
}

__global__ void k_vf_localize(const int* __restrict__ off, int nc, const int* __restrict__ num_out,
                              int n, int* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n || t >= *num_out) return;
  out[t] -= off[CloudOf(off, nc, out[t])];
}

struct MaxOp {
  __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const {
    return a > b ? a : b;
  }
};

csm_status ValidateClouds(const float* const* xyz, const int32_t* num_points, int32_t num_clouds,
                          const int32_t* kept_indices, const int32_t* num_kept,
                          std::vector<int>* off) {
  CSM_REQUIRE(num_clouds >= 0, "num_clouds");
  CSM_REQUIRE(num_clouds == 0 || (xyz && num_points && num_kept), "null pointer");
  off->assign(1, 0);
  long long total = 0;
  for (int c = 0; c < num_clouds; ++c) {
    CSM_REQUIRE(num_points[c] >= 0, "negative point count");
    CSM_REQUIRE(num_points[c] == 0 || xyz[c], "null cloud");
    CSM_REQUIRE(Finite(xyz[c], 3 * static_cast<size_t>(num_points[c])), "non-finite point");
    total += num_points[c];
    CSM_REQUIRE(total < (1ll << 30), "more than 2^30 points in one batch");
    off->push_back(static_cast<int>(total));
  }
  CSM_REQUIRE(total == 0 || kept_indices, "null kept_indices");
  return CSM_OK;
}

}  // namespace

size_t VoxelFilterStateBytes() { return sizeof(CloudState); }

csm_status VoxelFilterCheckStates(const void* states, int num_clouds) {
  const CloudState* rst = static_cast<const CloudState*>(states);
  for (int c = 0; c < num_clouds; ++c) {
    if (rst[c].error) {
      SetError("adaptive voxel filter: cloud %d did not settle in %d bisection steps", c,
               kBisectionSteps);
      return CSM_E_INTERNAL;
    }
    if (rst[c].phase != kDone) {
      SetError("adaptive voxel filter: cloud %d did not finish its search", c);
      return CSM_E_INTERNAL;
    }
  }
  return CSM_OK;
}

// The whole batch on ctx's stream, up to its device outputs: `options` null for VoxelFilter at
// `resolution`, else the adaptive filter.  The points come from the host clouds `xyz`, or are
// already on the device at d_xyz (off.back() x {x, y, z}).
csm_status VoxelFilterEnqueue(Ctx* ctx, const char* workspace, const float* const* xyz,
                              const float* d_xyz, const std::vector<int>& off,
                              const float* resolution,
                              const csm_adaptive_voxel_filter_options* options,
                              const unsigned char* d_pre_active, cudaEvent_t start,
                              VoxelFilterDeviceOut* result) {
  const int nc = static_cast<int>(off.size()) - 1;
  const int n = off.back();
  cudaStream_t s = ctx->stream;
  const bool adaptive = options != nullptr;

  std::vector<CloudState> st(nc);
  std::vector<float> max_range(nc);
  std::vector<long long> table_off(nc + 1, 0);
  for (int c = 0; c < nc; ++c) {
    CloudState& q = st[c];
    std::memset(&q, 0, sizeof(q));
    if (adaptive) {
      q.max_length = options[c].max_length;
      q.min_num_points = options[c].min_num_points;
      max_range[c] = options[c].max_range;
      q.phase = kFirst;
    } else {
      q.length = resolution[c];
      q.phase = kDone;
    }
    long long cap = 16;
    while (cap < 2ll * (off[c + 1] - off[c])) cap *= 2;
    table_off[c + 1] = table_off[c] + (adaptive ? cap : 0);
  }
  const long long table_slots = table_off[nc];

  // ---- temporary storage of the cub calls ----
  size_t sort_bytes = 0, sort2_bytes = 0, scan_bytes = 0, escan_bytes = 0, sel_bytes = 0;
  CSM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes,
                                           static_cast<unsigned long long*>(nullptr),
                                           static_cast<unsigned long long*>(nullptr),
                                           static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                           n, 0, 64, s));
  CSM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort2_bytes, static_cast<unsigned*>(nullptr),
                                           static_cast<unsigned*>(nullptr),
                                           static_cast<int*>(nullptr), static_cast<int*>(nullptr),
                                           n, 0, 32, s));
  CSM_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, static_cast<int*>(nullptr),
                                         static_cast<int*>(nullptr), n + 1, s));
  size_t ex_bytes = 0;
  CSM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, ex_bytes, static_cast<int*>(nullptr),
                                         static_cast<int*>(nullptr), n + 1, s));
  scan_bytes = std::max(scan_bytes, ex_bytes);
  CSM_CUDA(cub::DeviceScan::InclusiveScan(nullptr, escan_bytes,
                                          static_cast<unsigned long long*>(nullptr),
                                          static_cast<unsigned long long*>(nullptr), MaxOp(), n,
                                          s));
  CSM_CUDA(cub::DeviceSelect::Flagged(nullptr, sel_bytes, cub::CountingInputIterator<int>(0),
                                      static_cast<unsigned char*>(nullptr),
                                      static_cast<int*>(nullptr), static_cast<int*>(nullptr), n,
                                      s));
  const size_t temp_bytes =
      std::max(std::max(sort_bytes, sort2_bytes), std::max(std::max(scan_bytes, escan_bytes), sel_bytes));

  // ---- one workspace ----
  const size_t un = static_cast<size_t>(n) + 1;
  Carver sizer;
  auto lay = [&](Carver& w) {
    struct {
      float* xyz; int* off; CloudState* st; float* max_range; long long* table_off;
      unsigned long long* table; int* empty_seen; int* distinct; int* num_active;
      unsigned char* active; unsigned long long* keys; unsigned long long* keys_s; int* vals;
      int* vals_s; unsigned* cid; unsigned* cid_s; int* vals2; int* start; int* group;
      int* group_start; int* rank_in; int* group_in; int* is_call; int* call; int* call_k;
      unsigned long long* call_mask; unsigned char* call_flag;
      unsigned long long* ecode; unsigned long long* eincl; int* cand; int* num_cand; int* best;
      unsigned char* kept; int* out; int* num_out; int* counts; void* temp;
    } a;
    a.xyz = w.take<float>(3 * un);
    a.off = w.take<int>(nc + 1);
    a.st = w.take<CloudState>(nc);
    a.max_range = w.take<float>(nc);
    a.table_off = w.take<long long>(nc + 1);
    a.table = w.take<unsigned long long>(table_slots);
    a.empty_seen = w.take<int>(nc);
    a.distinct = w.take<int>(nc);
    a.num_active = w.take<int>(nc);
    a.active = w.take<unsigned char>(un);
    a.keys = w.take<unsigned long long>(un);
    a.keys_s = w.take<unsigned long long>(un);
    a.vals = w.take<int>(un);
    a.vals_s = w.take<int>(un);
    a.cid = w.take<unsigned>(un);
    a.cid_s = w.take<unsigned>(un);
    a.vals2 = w.take<int>(un);
    a.start = w.take<int>(un);
    a.group = w.take<int>(un);
    a.group_start = w.take<int>(un);
    a.rank_in = w.take<int>(un);
    a.group_in = w.take<int>(un);
    a.is_call = w.take<int>(un);
    a.call = w.take<int>(un);
    a.call_k = w.take<int>(un);
    a.call_mask = w.take<unsigned long long>(un);
    a.call_flag = w.take<unsigned char>(un);
    a.ecode = w.take<unsigned long long>(un);
    a.eincl = w.take<unsigned long long>(un);
    a.cand = w.take<int>(un);
    a.num_cand = w.take<int>(1);
    a.best = w.take<int>(un);
    a.kept = w.take<unsigned char>(un);
    a.out = w.take<int>(un);
    a.num_out = w.take<int>(1);
    a.counts = w.take<int>(nc);
    a.temp = w.take<char>(temp_bytes);
    return a;
  };
  lay(sizer);
  DevBuf& ws = ctx->D(workspace);
  CSM_TRY(ws.Reserve(sizer.at));
  Carver carver;
  carver.base = ws.as<char>();
  const auto a = lay(carver);

  // ---- upload: points, offsets, states, ranges, table offsets in one staging copy ----
  const size_t o_off = Align(sizeof(float) * 3 * static_cast<size_t>(n));
  const size_t o_st = o_off + Align(sizeof(int) * (nc + 1));
  const size_t o_mr = o_st + Align(sizeof(CloudState) * std::max(nc, 1));
  const size_t o_to = o_mr + Align(sizeof(float) * std::max(nc, 1));
  const size_t up_bytes = o_to + sizeof(long long) * (nc + 1);
  PinnedBuf& up = ctx->P((std::string(workspace) + "_up").c_str());
  CSM_TRY(up.Reserve(up_bytes));
  char* h = up.as<char>();
  if (d_xyz == nullptr)
    for (int c = 0; c < nc; ++c)
      if (off[c + 1] > off[c])
        std::memcpy(h + sizeof(float) * 3 * off[c], xyz[c], sizeof(float) * 3 * (off[c + 1] - off[c]));
  std::memcpy(h + o_off, off.data(), sizeof(int) * (nc + 1));
  if (nc > 0) {
    std::memcpy(h + o_st, st.data(), sizeof(CloudState) * nc);
    std::memcpy(h + o_mr, max_range.data(), sizeof(float) * nc);
  }
  std::memcpy(h + o_to, table_off.data(), sizeof(long long) * (nc + 1));

  if (start) CSM_CUDA(cudaEventRecord(start, s));
  const float* pts = d_xyz ? d_xyz : a.xyz;
  if (d_xyz == nullptr && n > 0)
    CSM_CUDA(cudaMemcpyAsync(a.xyz, h, o_off, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemcpyAsync(a.off, h + o_off, sizeof(int) * (nc + 1), cudaMemcpyHostToDevice, s));
  if (nc > 0) {
    CSM_CUDA(cudaMemcpyAsync(a.st, h + o_st, sizeof(CloudState) * nc, cudaMemcpyHostToDevice, s));
    CSM_CUDA(cudaMemcpyAsync(a.max_range, h + o_mr, sizeof(float) * nc, cudaMemcpyHostToDevice, s));
  }
  CSM_CUDA(cudaMemcpyAsync(a.table_off, h + o_to, sizeof(long long) * (nc + 1),
                           cudaMemcpyHostToDevice, s));
  const int nb = std::max(1, DivUp(n, kThreads));
  const int cb = std::max(1, DivUp(nc, kThreads));

  if (adaptive && nc > 0) {
    CSM_CUDA(cudaMemsetAsync(a.num_active, 0, sizeof(int) * nc, s));
    CSM_CUDA(cudaMemsetAsync(a.distinct, 0, sizeof(int) * nc, s));
    CSM_CUDA(cudaMemsetAsync(a.empty_seen, 0, sizeof(int) * nc, s));
    if (n > 0) {
      k_vf_range<<<nb, kThreads, 0, s>>>(pts, a.off, nc, a.max_range, d_pre_active, n, a.active,
                                         a.num_active);
      CSM_LAUNCH_CHECK();
    }
    k_vf_start<<<cb, kThreads, 0, s>>>(a.st, a.num_active, nc);
    CSM_LAUNCH_CHECK();
    // first length, 7 halvings, the bisection steps: a cloud that is done skips its points
    for (int trial = 0; trial < 1 + kHalvingSteps + kBisectionSteps; ++trial) {
      if (n > 0) {
        CSM_CUDA(cudaMemsetAsync(a.table, 0xff, sizeof(unsigned long long) * table_slots, s));
        k_vf_count<<<nb, kThreads, 0, s>>>(pts, a.off, nc, a.active, n, a.st, a.table,
                                           a.table_off, a.empty_seen, a.distinct);
        CSM_LAUNCH_CHECK();
      }
      k_vf_decide<<<cb, kThreads, 0, s>>>(a.st, a.distinct, a.empty_seen, nc);
      CSM_LAUNCH_CHECK();
    }
  }

  if (n > 0) {
    const unsigned char* active = adaptive ? a.active : nullptr;
    k_vf_keys<<<nb, kThreads, 0, s>>>(pts, a.off, nc, active, n, a.st, a.keys, a.vals, a.kept);
    CSM_LAUNCH_CHECK();
    size_t tb = temp_bytes;
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(a.temp, tb, a.keys, a.keys_s, a.vals, a.vals_s, n,
                                             0, 64, s));
    k_vf_cloud_ids<<<nb, kThreads, 0, s>>>(a.off, nc, active, a.st, a.vals_s, n, a.cid);
    CSM_LAUNCH_CHECK();
    int cloud_bits = 1;
    while (cloud_bits < 32 && (static_cast<unsigned>(nc) >> cloud_bits) != 0) ++cloud_bits;
    tb = temp_bytes;
    CSM_CUDA(cub::DeviceRadixSort::SortPairs(a.temp, tb, a.cid, a.cid_s, a.vals_s, a.vals2, n, 0,
                                             cloud_bits, s));
    k_vf_starts<<<nb, kThreads, 0, s>>>(a.cid_s, a.vals2, a.keys, nc, n, a.start);
    CSM_LAUNCH_CHECK();
    tb = temp_bytes;
    CSM_CUDA(cub::DeviceScan::InclusiveSum(a.temp, tb, a.start, a.group, n, s));
    k_vf_group_starts<<<nb, kThreads, 0, s>>>(a.start, a.group, n, a.group_start);
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cudaMemsetAsync(a.rank_in, 0, sizeof(int) * un, s));
    CSM_CUDA(cudaMemsetAsync(a.is_call, 0, sizeof(int) * un, s));
    k_vf_ranks<<<nb, kThreads, 0, s>>>(a.cid_s, a.vals2, a.group, a.group_start, nc, n, a.rank_in,
                                       a.group_in, a.is_call);
    CSM_LAUNCH_CHECK();
    tb = temp_bytes;
    CSM_CUDA(cub::DeviceScan::ExclusiveSum(a.temp, tb, a.is_call, a.call, n + 1, s));
    // slots past the call count stay out of the candidates
    CSM_CUDA(cudaMemsetAsync(a.call_flag, 0, un, s));
    k_vf_calls<<<nb, kThreads, 0, s>>>(a.off, nc, a.rank_in, a.call, n, a.call_k,
                                       a.call_mask, a.call_flag, a.ecode);
    CSM_LAUNCH_CHECK();
    CSM_CUDA(cudaMemsetAsync(a.best, 0, sizeof(int) * un, s));
    tb = temp_bytes;
    CSM_CUDA(cub::DeviceSelect::Flagged(a.temp, tb, cub::CountingInputIterator<int>(0),
                                        a.call_flag, a.cand, a.num_cand, n, s));
    k_vf_walk<<<cb, kThreads, 0, s>>>(a.off, nc, a.call, a.cand, a.num_cand, a.call_k,
                                      a.call_mask, a.ecode);
    CSM_LAUNCH_CHECK();
    tb = temp_bytes;
    CSM_CUDA(cub::DeviceScan::InclusiveScan(a.temp, tb, a.ecode, a.eincl, MaxOp(), n, s));
    k_vf_hits<<<nb, kThreads, 0, s>>>(a.off, nc, a.rank_in, a.group_in, a.call, a.eincl, n,
                                      a.best);
    CSM_LAUNCH_CHECK();
    k_vf_keep<<<nb, kThreads, 0, s>>>(a.cid_s, a.vals2, a.rank_in, a.group_in, a.best, nc, n,
                                      a.kept);
    CSM_LAUNCH_CHECK();
    tb = temp_bytes;
    CSM_CUDA(cub::DeviceSelect::Flagged(a.temp, tb, cub::CountingInputIterator<int>(0), a.kept,
                                        a.out, a.num_out, n, s));
    k_vf_counts<<<cb, kThreads, 0, s>>>(a.off, nc, a.out, a.num_out, a.counts);
    CSM_LAUNCH_CHECK();
    k_vf_localize<<<nb, kThreads, 0, s>>>(a.off, nc, a.num_out, n, a.out);
    CSM_LAUNCH_CHECK();
  } else if (nc > 0) {
    CSM_CUDA(cudaMemsetAsync(a.counts, 0, sizeof(int) * nc, s));
  }
  result->kept_indices = a.out;
  result->num_kept = a.counts;
  result->kept = a.kept;
  result->states = a.st;
  return CSM_OK;
}

namespace {

// The whole batch from host clouds to host outputs, with one stream synchronisation.
csm_status Run(const float* const* xyz, const std::vector<int>& off, const float* resolution,
               const csm_adaptive_voxel_filter_options* options, int32_t device,
               int32_t* kept_indices, int32_t* num_kept, csm_stats* stats) {
  const int nc = static_cast<int>(off.size()) - 1;
  const int n = off.back();
  LaneGuard guard;
  CSM_TRY(AcquireLane(device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  VoxelFilterDeviceOut a;
  CSM_TRY(VoxelFilterEnqueue(ctx, "voxel_filter", xyz, nullptr, off, resolution, options,
                             nullptr, ctx->ev0, &a));
  // ---- read-back: indices, counts, states (error flags) ----
  const size_t o_cnt = Align(sizeof(int) * std::max(n, 1));
  const size_t o_rst = o_cnt + Align(sizeof(int) * std::max(nc, 1));
  PinnedBuf& down = ctx->P("voxel_filter_down");
  CSM_TRY(down.Reserve(o_rst + sizeof(CloudState) * std::max(nc, 1)));
  char* d = down.as<char>();
  if (n > 0)
    CSM_CUDA(cudaMemcpyAsync(d, a.kept_indices, sizeof(int) * n, cudaMemcpyDeviceToHost, s));
  if (nc > 0) {
    CSM_CUDA(cudaMemcpyAsync(d + o_cnt, a.num_kept, sizeof(int) * nc, cudaMemcpyDeviceToHost, s));
    CSM_CUDA(cudaMemcpyAsync(d + o_rst, a.states, sizeof(CloudState) * nc, cudaMemcpyDeviceToHost,
                             s));
  }
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  CSM_TRY(VoxelFilterCheckStates(d + o_rst, nc));
  const int* counts = reinterpret_cast<const int*>(d + o_cnt);
  long long total = 0;
  for (int c = 0; c < nc; ++c) total += counts[c];
  if (total > 0) std::memcpy(kept_indices, d, sizeof(int) * total);
  if (nc > 0) std::memcpy(num_kept, counts, sizeof(int) * nc);
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->host_syncs = 1;
    cudaEventElapsedTime(&stats->device_ms, ctx->ev0, ctx->ev1);
  }
  return CSM_OK;
}

}  // namespace
}  // namespace csm

using namespace csm;

extern "C" {

csm_status csm_voxel_filter_batch(const float* const* xyz, const int32_t* num_points,
                                  const float* resolution, int32_t num_clouds, int32_t device,
                                  int32_t* kept_indices, int32_t* num_kept, csm_stats* stats) {
  std::vector<int> off;
  CSM_TRY(ValidateClouds(xyz, num_points, num_clouds, kept_indices, num_kept, &off));
  CSM_REQUIRE(num_clouds == 0 || resolution, "null resolution");
  for (int c = 0; c < num_clouds; ++c)
    CSM_REQUIRE(std::isfinite(resolution[c]) && resolution[c] > 0.f, "resolution");
  return Run(xyz, off, resolution, nullptr, device, kept_indices, num_kept, stats);
}

csm_status csm_adaptive_voxel_filter_batch(const float* const* xyz, const int32_t* num_points,
                                           const csm_adaptive_voxel_filter_options* options,
                                           int32_t num_clouds, int32_t device,
                                           int32_t* kept_indices, int32_t* num_kept,
                                           csm_stats* stats) {
  std::vector<int> off;
  CSM_TRY(ValidateClouds(xyz, num_points, num_clouds, kept_indices, num_kept, &off));
  CSM_REQUIRE(num_clouds == 0 || options, "null options");
  for (int c = 0; c < num_clouds; ++c) {
    CSM_REQUIRE(std::isfinite(options[c].max_length) && options[c].max_length > 0.f,
                "max_length");
    CSM_REQUIRE(!std::isnan(options[c].min_num_points) && !std::isnan(options[c].max_range),
                "min_num_points / max_range");
  }
  return Run(xyz, off, nullptr, options, device, kept_indices, num_kept, stats);
}

}  // extern "C"
