// Pieces shared by the entry points that take many point batches in one call (voxel_filter.cu,
// outlier3d.cu): the reference's float -> int voxel rounding, the batch of a flat point index,
// a 64-bit hash finaliser for open addressing, and the carving of one workspace.
#ifndef CSM_POINT_BATCH_CUH_
#define CSM_POINT_BATCH_CUH_

#include <algorithm>
#include <cstdint>

namespace csm {

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
