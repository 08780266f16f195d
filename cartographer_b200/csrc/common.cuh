// Shared plumbing of libcsm_b200.so: error reporting, per-device context
// (stream + growable device workspace + pinned staging), launch counting.
#ifndef CSM_COMMON_CUH_
#define CSM_COMMON_CUH_

#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/csm_abi.h"

namespace csm {

void SetError(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

#define CSM_CUDA(expr)                                                              \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
      ::csm::SetError("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,            \
                      cudaGetErrorString(_e));                                      \
      return CSM_E_CUDA;                                                            \
    }                                                                               \
  } while (0)

#define CSM_REQUIRE(cond, msg)                                                      \
  do {                                                                              \
    if (!(cond)) {                                                                  \
      ::csm::SetError("%s:%d: invalid argument: %s (%s)", __FILE__, __LINE__, msg,  \
                      #cond);                                                       \
      return CSM_E_INVALID;                                                         \
    }                                                                               \
  } while (0)

#define CSM_TRY(expr)                     \
  do {                                    \
    csm_status _s = (expr);               \
    if (_s != CSM_OK) return _s;          \
  } while (0)

inline int DivUp(long long a, long long b) { return static_cast<int>((a + b - 1) / b); }

// The engines' order-preserving float <-> unsigned map (bounds are kept as unsigned so that
// atomicMax on them orders like the float scores).
__host__ __device__ __forceinline__ unsigned FloatToOrdered(float f) {
#ifdef __CUDA_ARCH__
  const unsigned u = __float_as_uint(f);
#else
  unsigned u;
  std::memcpy(&u, &f, 4);
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float OrderedToFloat(unsigned u) {
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  std::memcpy(&f, &u, 4);
  return f;
#endif
}

#define CSM_LAUNCH_CHECK()                                                          \
  do {                                                                              \
    ::csm::g_launches.fetch_add(1, std::memory_order_relaxed);                      \
    CSM_CUDA(cudaGetLastError());                                                   \
  } while (0)

// A device buffer that only ever grows; reused across calls so the steady state
// performs no cudaMalloc.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaStream_t stream = nullptr;   // set by Ctx::D: the workspace lives on that lane's stream
  csm_status Reserve(size_t bytes) {
    if (bytes <= cap) return CSM_OK;
    // 50 % headroom: batches of a queue differ widely in their scan counts.  Workspaces of a
    // lane are (re)allocated from the stream-ordered pool: a regrowth is then a pair of
    // stream operations, not a cudaFree + cudaMalloc pair that synchronises the whole device
    // (which shows up as outlier steps when several GPUs wait for each other every step).
    const size_t want = bytes + bytes / 2 + 256;
    if (stream) {
      if (p) CSM_CUDA(cudaFreeAsync(p, stream));
      p = nullptr;
      cap = 0;
      CSM_CUDA(cudaMallocAsync(&p, want, stream));
    } else {
      if (p) CSM_CUDA(cudaFree(p));
      p = nullptr;
      cap = 0;
      CSM_CUDA(cudaMalloc(&p, want));
    }
    cap = want;
    return CSM_OK;
  }
  template <typename T>
  T* as() const { return static_cast<T*>(p); }
};

struct PinnedBuf {
  void* p = nullptr;
  size_t cap = 0;
  csm_status Reserve(size_t bytes) {
    if (bytes <= cap) return CSM_OK;
    if (p) CSM_CUDA(cudaFreeHost(p));
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    CSM_CUDA(cudaMallocHost(&p, want));
    cap = want;
    return CSM_OK;
  }
  template <typename T>
  T* as() const { return static_cast<T*>(p); }
};

// One per CUDA device, created on first use.  `mu` serialises engine calls on
// the device (handle-level locking, SURVEY §8b).
struct Ctx {
  int device = -1;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::mutex mu;
  std::map<std::string, DevBuf> dev;      // named workspaces
  std::map<std::string, PinnedBuf> pin;
  DevBuf& D(const char* name) {
    DevBuf& b = dev[name];
    b.stream = stream;
    return b;
  }
  // Workspace `name` with at least `bytes`, in *out.
  csm_status Reserve(const char* name, size_t bytes, DevBuf** out) {
    *out = &D(name);
    return (*out)->Reserve(bytes);
  }
  PinnedBuf& P(const char* name) { return pin[name]; }
  // Recycled device buffers of destroyed point clouds (guarded by `mu`): node scans
  // come and go at sensor rate, and cudaMalloc / cudaFree serialise the whole device.
  std::vector<std::pair<void*, size_t>> cloud_pool;
  size_t cloud_pool_bytes = 0;
};

csm_status GetCtx(int device, Ctx** out);

// Match calls do not serialise on the device-wide context: each call borrows a
// "lane" — a Ctx of the same device with its own stream, events and workspace —
// so that several host threads (the reference's pool threads,
// constraints/constraint_builder_2d.cc:102-111) keep the GPU busy with concurrent
// matches.  Handles (stacks, clouds, matchers) are read-only during matches and are
// shared by all lanes.
struct LaneGuard {
  Ctx* lane = nullptr;
  std::unique_lock<std::mutex> lock;
};
csm_status AcquireLane(int device, LaneGuard* out);

// Optional per-kernel timing (csm_profile_enable): CUDA events on the engine's
// own stream around every launch of a named kernel; bench.py reads the totals
// to compute the roofline numbers of the dominant kernel.
extern std::atomic<int> g_profile_on;
void ProfBegin(Ctx* ctx);  // per-lane events
void ProfStop(Ctx* ctx);                                   // records the end event
void ProfCommit(Ctx* ctx, const char* name, double units);  // waits for it and accumulates
inline void ProfEnd(Ctx* ctx, const char* name, double units) {
  ProfStop(ctx);
  ProfCommit(ctx, name, units);
}

}  // namespace csm

#endif  // CSM_COMMON_CUH_
