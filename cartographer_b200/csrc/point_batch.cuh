// Pieces shared by the entry points that take many point batches in one call (voxel_filter.cu,
// outlier3d.cu, xray.cu): the reference's float -> int voxel rounding, the batch of a flat point
// index, a 64-bit hash finaliser, the open-addressing tables of packed voxel keys, and the carving
// of one workspace.
#ifndef CSM_POINT_BATCH_CUH_
#define CSM_POINT_BATCH_CUH_

#include <algorithm>
#include <cstdint>
#include <type_traits>

namespace csm {

// DynamicGrid (mapping/3d/hybrid_grid.h) can only grow to the cell indices [-8192, 8192)^3.
constexpr int kCubeHalf = 8192;
constexpr unsigned long long kEmptyKey = ~0ull;     // no packed key has bits above 41 set

__host__ __device__ inline bool InCube(int v) { return v >= -kCubeHalf && v < kCubeHalf; }

// A voxel of the cube as a 42-bit key: 14 bits each of z, y, x offset by kCubeHalf, so that
// ascending keys are ascending (z, y, x).
__host__ __device__ inline unsigned long long Pack(int x, int y, int z) {
  return (static_cast<unsigned long long>(z + kCubeHalf) << 28) |
         (static_cast<unsigned long long>(y + kCubeHalf) << 14) |
         static_cast<unsigned long long>(x + kCubeHalf);
}

// common::RoundToInt = std::lround narrowed to int: half away from zero; an integer at or
// beyond 2^63 in magnitude (and NaN) is LONG_MIN on x86-64, whose low 32 bits are 0.
__device__ inline int RoundToInt(float v) {
  if (!(fabsf(roundf(v)) < 9.223372036854775808e18f)) return 0;
  return static_cast<int>(lroundf(v));
}

// The batch of flat point index i: the last c with off[c] <= i.
__device__ inline int CloudOf(const int* off, int num_clouds, int i) {
  int lo = 0, hi = num_clouds;
  while (hi - lo > 1) {
    const int mid = (lo + hi) / 2;
    if (off[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ inline uint64_t Mix(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  return k ^ (k >> 33);
}

// Open addressing with linear probing over a power-of-two table of packed keys (kEmptyKey when
// free); a table's values, if any, live in a parallel array at the same slot.

// The slot of `key`, or -1 when it is absent.
__device__ inline long long Find(const unsigned long long* __restrict__ keys,
                                 unsigned long long mask, unsigned long long key) {
  unsigned long long h = Mix(key) & mask;
  for (;;) {
    const unsigned long long k = keys[h];
    if (k == key) return static_cast<long long>(h);
    if (k == kEmptyKey) return -1;
    h = (h + 1) & mask;
  }
}

// The slot of `key`, claimed with atomicCAS when it is absent (*inserted says which).
__device__ inline unsigned long long Insert(unsigned long long* keys, unsigned long long mask,
                                            unsigned long long key, bool* inserted) {
  unsigned long long h = Mix(key) & mask;
  for (;;) {
    const unsigned long long old = atomicCAS(&keys[h], kEmptyKey, key);
    if (old == kEmptyKey || old == key) {
      *inserted = old == kEmptyKey;
      return h;
    }
    h = (h + 1) & mask;
  }
}

// The value type of a table that is a set of keys.
struct NoValues {};

// Moves every key of a table (and its value, unless V is NoValues) into a larger, empty one.
template <class V>
__global__ void k_rehash(const unsigned long long* __restrict__ old_keys,
                         const V* __restrict__ old_vals, long long old_slots,
                         unsigned long long* keys, V* vals, unsigned long long mask) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= old_slots || old_keys[i] == kEmptyKey) return;
  bool inserted;
  const unsigned long long h = Insert(keys, mask, old_keys[i], &inserted);
  if constexpr (!std::is_same<V, NoValues>::value) vals[h] = old_vals[i];
}

inline size_t Align(size_t b) { return (b + 255) / 256 * 256; }

// Carves typed arrays out of one workspace.
struct Carver {
  size_t at = 0;
  char* base = nullptr;
  template <typename T>
  T* take(size_t count) {
    T* p = reinterpret_cast<T*>(base + at);
    at += Align(sizeof(T) * std::max<size_t>(count, 1));
    return p;
  }
};

}  // namespace csm

#endif  // CSM_POINT_BATCH_CUH_
