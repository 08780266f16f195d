// Device-side records of the 2D fast correlative scan matcher.
#ifndef CSM_ENGINE2D_CUH_
#define CSM_ENGINE2D_CUH_

#include <cmath>

#include "common.cuh"
#include "rigid3f.h"

namespace csm {

constexpr int kMaxDepth = 12;

// PrecomputationGridStack2D on the device.  Level h has width w = 2^h, wide
// limits (nx + w - 1, ny + w - 1), offset (-w+1, -w+1) and is stored row-major
// (x + y * wx), exactly the reference's PrecomputationGrid2D::cells_
// (fast_correlative_scan_matcher_2d.h:56-71).
struct StackDev {
  const uint8_t* level[kMaxDepth];
  // Decimated ("phase-major") layout of the lowest-resolution level h = depth-1
  // for the dense passes.  With s = 2^h the flat array
  //   D[((ay * s + ax) * jd + J) * ids + I] = level[h][(s*J + ay) * wx + s*I + ax]
  // (zero outside the wide grid; every row is followed by >= 4 zero bytes) puts
  // the cells that the candidates of one scan lattice need for one scan point
  // into consecutive bytes.  dec4 holds FOUR copies of D, copy k shifted left by
  // k bytes (copy_k[t] = D[t + k]), each dec_lpad bytes long with index 0 at byte
  // 16, so that any 4 consecutive bytes of D can be fetched with one aligned
  // 32-bit load: word(a) = *(u32*)(dec4 + (a & 3) * dec_lpad + 16 + (a & ~3)).
  // Only entry depth-1 is populated.
  const uint8_t* dec4[kMaxDepth];
  int dec_lpad[kMaxDepth], dec_id[kMaxDepth], dec_jd[kMaxDepth], dec_ids[kMaxDepth];
  // Branch layout ("child windows") for parent levels h = 1 .. depth-1.  A node of
  // level h sits on its scan's lattice of stride S = 2^h; its four children are the
  // cells of level h-1 at the node's position and s = S/2 further along x and/or y.
  // With b = (scan point + node offset + s - 1), Q = b >> h and A = b & (S-1) per
  // axis, ONE aligned 32-bit word holds all four children values:
  //   win[h][((Ay*S + Ax) * win_jd + Qy + 1) * win_ids + Qx + 1] =
  //     { L(x, y), L(x+s, y), L(x, y+s), L(x+s, y+s) }   (bytes 0..3, L = level h-1,
  //       x = S*Qx + Ax, y = S*Qy + Ay, zero outside the wide grid)
  // for Qx in [-1, win_ids-1), Qy in [-1, win_jd-1); cells outside that range are all
  // zero.  Lattice neighbours (Qx+1) of the same scan point are neighbouring words.
  const unsigned* win[kMaxDepth];
  int win_jd[kMaxDepth], win_ids[kMaxDepth];
  int wx[kMaxDepth], wy[kMaxDepth];
  int nx, ny, depth;
  double resolution, max_x, max_y;
  float min_score, max_score, k255;  // k255 = (max_score - min_score) / 255.f
};

struct JobDev {
  const StackDev* stack;
  const float* xyz;      // cloud, n x 3
  const float2* trig;    // per scan: (cos(ha), sin(ha)) of the rotation quaternion
  int n;
  int num_scans;
  int scan_base;         // global index of this job's scan 0
  int lin;               // num_linear_perturbations (pre-shrink window)
  int cap;               // top-level slots reserved per scan
  int cap_y;             // max candidates along y (slot = i * nyc + j uses the scan's own nyc)
  Quatf q0;              // initial rotation as Quaternionf(AngleAxisf(yaw, UnitZ))
  float tx, ty;          // initial translation (float casts)
  float min_score;
  // Discrete scans: scan k of the job owns n slots from dscan_off + k * n of the point
  // buffer (short2 cells per point), of `ent` and of `wt`.  When the tile form of the
  // lowest-resolution pass runs, the first ScanInfo::entries slots of `ent` / `wt` hold the
  // runs of equal consecutive cells in beam order, one entry per run of at most kMaxWeight
  // points, with the run length as weight, and the tile pass walks those.
  short2* ent;
  uint8_t* wt;
  long long dscan_off;   // first slot of this job in the discrete-scan buffers
  long long top_off;     // first slot of this job in the top-level sum buffer
};

// Largest weight of one entry (the tile pass flushes its packed u16 sums by weight).
constexpr int kMaxWeight = 4;

struct ScanInfo {
  int job;
  int min_x, max_x, min_y, max_y;  // LinearBounds after ShrinkToFit
  int nxc, nyc;                    // lowest-resolution candidates per axis
  int entries;                     // entries of the discrete scan (0 unless merged)
};

struct Node {  // 16 B
  int scan;    // global scan index
  int xo, yo;  // x/y_index_offset
  float score;
};

// SearchParameters(linear, angular, point cloud, resolution) of both 2D matchers
// (correlative_scan_matcher_2d.cc:27-55).  `max_scan_range` is the caller's fold over its
// points, which starts from 3 * resolution.
struct SearchParameters2D {
  int num_angular;
  int num_scans;
  int lin;
  double step;
};

inline SearchParameters2D MakeSearchParameters2D(double linear_window, double angular_window,
                                                 float max_scan_range, double resolution) {
  const double kSafetyMargin = 1. - 1e-3;
  SearchParameters2D s;
  s.step = kSafetyMargin *
           std::acos(1. - (resolution * resolution) / (2. * (max_scan_range * max_scan_range)));
  s.num_angular = static_cast<int>(std::ceil(angular_window / s.step));
  s.num_scans = 2 * s.num_angular + 1;
  s.lin = static_cast<int>(std::ceil(linear_window / resolution));
  return s;
}

// The rotations of GenerateRotatedScans (correlative_scan_matcher_2d.cc:93-109) as num_scans
// (cos, sin) pairs into `out`: delta_theta accumulates in double and is cast to float for
// AngleAxisf, and Quaternionf takes cos / sin of the float half angle (QuatFromCosSinZ).
inline void FillRotationTable(const SearchParameters2D& sp, float* out) {
  double delta_theta = -sp.num_angular * sp.step;
  for (int k = 0; k < sp.num_scans; ++k, delta_theta += sp.step) {
    const float ha = 0.5f * static_cast<float>(delta_theta);
    out[2 * k] = std::cos(ha);
    out[2 * k + 1] = std::sin(ha);
  }
}

}  // namespace csm

struct csm_stack2d {
  csm::Ctx* ctx = nullptr;
  csm::StackDev h;             // host copy of the descriptor (device pointers inside)
  csm::StackDev* d = nullptr;  // device copy
  uint8_t* d_levels = nullptr;
  uint8_t* d_dec = nullptr;
  unsigned* d_win = nullptr;
  size_t level_off[csm::kMaxDepth];
  size_t win_off[csm::kMaxDepth] = {};   // first word of every child-window level in d_win
  float min_cost = 0.f, max_cost = 0.f;
  // also runs when csm_stack2d_create fails half-way (cudaFree(nullptr) is a no-op)
  ~csm_stack2d() {
    cudaFree(d_levels);
    cudaFree(d_dec);
    cudaFree(d_win);
    cudaFree(d);
  }
};

struct csm_cloud {
  csm::Ctx* ctx = nullptr;
  int n = 0;
  float* d_xyz = nullptr;
  size_t d_bytes = 0;   // capacity of d_xyz (buffers are recycled through Ctx::cloud_pool)
  float max_norm = 0.f;  // max_i sqrt(x*x + y*y) in float (correlative_scan_matcher_2d.cc:35-38)
  std::vector<float> h_xyz;
  ~csm_cloud() { cudaFree(d_xyz); }  // nullptr once the buffer went back to the pool
};

#endif  // CSM_ENGINE2D_CUH_
