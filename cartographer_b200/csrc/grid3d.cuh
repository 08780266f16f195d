// The dense device copies of a HybridGrid (csm_grid3d) and an IntensityHybridGrid
// (csm_intensity_grid3d).  grid3d.cu makes, reads, grows and enumerates them; the real-time
// 3D matcher (rt3d.cu), the fast matcher (engine3d.cu), the 3D refinement (refine3d.cu), the
// range-data inserter (insert3d.cu) and the submap textures (submap_texture.cu) use them.
#ifndef CSM_GRID3D_CUH_
#define CSM_GRID3D_CUH_

#include "common.cuh"

namespace csm {

// HybridGrid indices lie in the 2^14 cube, -kCube .. kCube - 1 on each axis (hybrid_grid.h:387).
constexpr int kCube = 8192;
// The dense volumes' size guards, in voxels.  An intensity volume's insert sorts 32-bit voxel
// keys, so its guard is lower.
constexpr size_t kMaxVoxels3 = size_t(8) << 30;
constexpr size_t kMaxIntensityVoxels3 = size_t(4) << 30;

// A dense box: n[a] voxels from lo[a] on each axis, x fastest, z slowest.
struct Box3 {
  int lo[3];
  int n[3];
  __host__ __device__ __forceinline__ unsigned long long Index(int x, int y, int z) const {
    return (static_cast<unsigned long long>(z - lo[2]) * n[1] + (y - lo[1])) * n[0] + (x - lo[0]);
  }
  __host__ __device__ __forceinline__ size_t Volume() const {
    return static_cast<size_t>(n[0]) * n[1] * n[2];
  }
};

// The smallest box holding a set of voxels, empty until the first of them.  A handle's tight
// box holds every voxel it was made from and every origin / hit cell inserted since; its dense
// box always contains it, and an insert sizes a grown box from it.
struct TightBox3 {
  bool empty = true;
  int lo[3] = {0, 0, 0};
  int hi[3] = {0, 0, 0};
  void Include(const int* c) {
    for (int a = 0; a < 3; ++a) {
      if (empty || c[a] < lo[a]) lo[a] = c[a];
      if (empty || c[a] > hi[a]) hi[a] = c[a];
    }
    empty = false;
  }
  bool InCube() const {
    for (int a = 0; a < 3; ++a)
      if (lo[a] < -kCube || hi[a] >= kCube) return false;
    return true;
  }
  // The dense box of exactly this box; one voxel at the origin when empty.
  Box3 Dense() const {
    return Box3{{lo[0], lo[1], lo[2]}, {hi[0] - lo[0] + 1, hi[1] - lo[1] + 1, hi[2] - lo[2] + 1}};
  }
};

// The tight box of the voxel list idx[3 n] ({x, y, z} each).
TightBox3 ListBox3(const int32_t* idx, int64_t n);

// A HybridGrid volume as the matchers read it: values at box {lo, n}, 0 outside, and
// GetProbability's conversion.
struct Grid3Dev {
  const uint16_t* p;
  int lo[3];
  int n[3];
  float resolution, k_scale, bias, min_probability;
};

Grid3Dev MakeGrid3Dev(const uint16_t* p, const Box3& box, float resolution);

inline Box3 BoxOf(const Grid3Dev& g) {
  return Box3{{g.lo[0], g.lo[1], g.lo[2]}, {g.n[0], g.n[1], g.n[2]}};
}

}  // namespace csm

struct csm_grid3d {
  csm::Ctx* ctx = nullptr;
  csm::Grid3Dev g;
  uint16_t* d_vol = nullptr;
  csm::TightBox3 tight;
  ~csm_grid3d() { cudaFree(d_vol); }
};

// GetIntensity per voxel of `box`, 0 elsewhere.  The first insert adds the AverageIntensityData
// volumes d_sum / d_count, filled from the voxel list the handle was made from (kept on the host
// until then), so a handle that is never inserted into keeps only the means on the device.
struct csm_intensity_grid3d {
  csm::Ctx* ctx = nullptr;
  float* d_vol = nullptr;
  csm::Box3 box{};
  float resolution = 0.f;
  csm::TightBox3 tight;
  float* d_sum = nullptr;
  int32_t* d_count = nullptr;
  std::vector<int32_t> made_idx, made_count;
  std::vector<float> made_sum;
  ~csm_intensity_grid3d() {
    cudaFree(d_vol);
    cudaFree(d_sum);
    cudaFree(d_count);
  }
};

namespace csm {

// A handle's dense volume as the kernels that walk it read it.
struct Box16 {
  const uint16_t* p;
  int lo[3];
  int n[3];
};

inline Box16 HandleBox(const csm_grid3d* g) {
  return Box16{g->g.p, {g->g.lo[0], g->g.lo[1], g->g.lo[2]}, {g->g.n[0], g->g.n[1], g->g.n[2]}};
}

// The value of cell (x, y, z) of the source box, 0 outside it.
__device__ __forceinline__ uint16_t Val16(const Box16& b, int x, int y, int z) {
  const int lx = x - b.lo[0], ly = y - b.lo[1], lz = z - b.lo[2];
  if (static_cast<unsigned>(lx) >= static_cast<unsigned>(b.n[0]) ||
      static_cast<unsigned>(ly) >= static_cast<unsigned>(b.n[1]) ||
      static_cast<unsigned>(lz) >= static_cast<unsigned>(b.n[2]))
    return 0;
  return __ldg(b.p + (static_cast<size_t>(lz) * b.n[1] + ly) * b.n[0] + lx);
}

// Launch shape of the kernels that walk a box row by row: x along the rows of a box of
// nx x rows cells (coalesced), blockIdx.y over the rows, at most `max_blocks` blocks in all.
inline dim3 RowGrid(int nx, long long rows, int max_blocks) {
  const int bx = DivUp(nx, 256);
  const long long by = std::max<long long>(1, std::min<long long>(rows, max_blocks / bx));
  return dim3(bx, static_cast<unsigned>(std::min<long long>(by, 65535)));
}

// Scatters the voxel list idx[3 n] / values[n], in host memory, into `vol`, a zero-filled volume
// of `box` holding every listed voxel, on the context's stream.  Caller holds ctx->mu.
template <typename T>
csm_status ScatterVoxels3(Ctx* ctx, const int32_t* idx, const T* values, long long n,
                          const Box3& box, T* vol);

// Queues on the context's stream the bounding box of the non-zero voxels of `g`'s dense volume,
// as offsets from its lo, into the device words mn[0..2] (the min) and mx[0..2] (the max + 1;
// mx[0] == 0: no non-zero voxel).  Caller holds ctx->mu.
csm_status QueueNonZeroBox3(const csm_grid3d* g, unsigned* mn, unsigned* mx);

// The number *n of non-zero voxels of `g` and, when it is at most list_capacity, the voxels in
// HybridGrid's iteration order in device workspaces: *d_idx ({x, y, z} each) and *d_val, ready on
// the context's stream (what csm_grid3d_voxels returns).  Caller holds ctx->mu.
csm_status DeviceVoxels3D(const csm_grid3d* g, long long list_capacity, long long* n,
                          const int** d_idx, const uint16_t** d_val);

// The part of one 3D insert that changes the handles (caller holds ctx->mu; intensity_grid is
// null when the insert adds no intensities):
//   1. Grow: from the tight boxes the insert needs, the box each handle's volumes grow to;
//   2. Begin: queues on the context's stream the grown volumes, with the old ones copied in,
//      and, on the first insert into the intensity handle, its sum / count volumes at their
//      final box with the voxel list it was made from scattered in;
//   3. the caller's kernels write vol at `box` and mean / sum / count at `ibox`; the caller
//      records ctx->ev1 (ctx->ev0 before its first device work) and synchronises the stream;
//   4. Commit: installs the volumes, boxes and tight boxes, frees the volumes they replace,
//      drops the voxel list the intensity handle was made from and fills stats (may be NULL).
// No handle field changes before Commit.  Volumes not committed are freed when the transaction
// ends: the handles keep their volumes, boxes and contents.  Several transactions make one when
// the caller grows all of them before it begins any, and commits all of them or none.
class GridInsert3 {
 public:
  GridInsert3(csm_grid3d* grid, csm_intensity_grid3d* intensity_grid);
  ~GridInsert3();
  GridInsert3(const GridInsert3&) = delete;
  GridInsert3& operator=(const GridInsert3&) = delete;
  // CSM_E_INVALID if a grown volume would pass its size guard.
  csm_status Grow(const TightBox3& need, const TightBox3& intensity_need);
  csm_status Begin();
  void Commit(csm_stats* stats);

  Box3 box, ibox{};   // the boxes the insert writes at
  // what it writes: the handles' own volumes, or ones Begin allocated
  uint16_t* vol;
  float* mean = nullptr;
  float* sum = nullptr;
  int32_t* count = nullptr;

 private:
  csm_grid3d* grid_;
  csm_intensity_grid3d* igrid_;
  TightBox3 need_, ineed_;
  bool grow_ = false, igrow_ = false;
};

}  // namespace csm

#endif  // CSM_GRID3D_CUH_
