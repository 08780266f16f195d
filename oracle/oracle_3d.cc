// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_common.h, oracle_3d.h).
// Restates mapping/3d/hybrid_grid.h and mapping/internal/3d/scan_matching/
// {precomputation_grid_3d,rotational_scan_matcher,low_resolution_matcher,
//  fast_correlative_scan_matcher_3d}.cc.
#include "oracle_3d.h"

#include <algorithm>
#include <cmath>
#include <limits>

namespace oracle {

static thread_local MatchStats3D* stats3_ = nullptr;

// ---- Eigen quaternion / rigid helpers ----------------------------------------
Quatf QuatMul(const Quatf& a, const Quatf& b) {
  Quatf r;
  r.x = (a.x * b.w - a.z * b.y) + (a.y * b.z + a.w * b.x);
  r.y = (a.y * b.w - a.x * b.z) + (a.z * b.x + a.w * b.y);
  r.z = (a.z * b.w - a.y * b.x) + (a.x * b.y + a.w * b.z);
  r.w = (a.w * b.w - a.x * b.x) + (-(a.z * b.z + a.y * b.y));
  return r;
}
float QuatSquaredNorm(const Quatf& q) { return (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w); }
Quatf QuatNormalized(const Quatf& q) {
  const float z = QuatSquaredNorm(q);
  if (z > 0.f) {
    const float n = std::sqrt(z);
    return Quatf{q.w / n, q.x / n, q.y / n, q.z / n};
  }
  return q;
}
Quatf QuatConjugate(const Quatf& q) { return Quatf{q.w, -q.x, -q.y, -q.z}; }
Quatf QuatInverse(const Quatf& q) {
  const float n2 = QuatSquaredNorm(q);
  if (n2 > 0.f) return Quatf{q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
  return Quatf{0.f, 0.f, 0.f, 0.f};
}
Quatf QuatCastInverseD(const Quatd& q) {
  const double n2 = (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w);
  Quatd inv{0., 0., 0., 0.};
  if (n2 > 0.) inv = Quatd{q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
  return Quatf{static_cast<float>(inv.w), static_cast<float>(inv.x), static_cast<float>(inv.y),
               static_cast<float>(inv.z)};
}
Vec3f Rigid3Apply(const Rigid3f& r, const Vec3f& p) {
  const Vec3f v = Rotate(r.q, p);
  return Vec3f{v.x + r.t.x, v.y + r.t.y, v.z + r.t.z};
}
Rigid3f Rigid3Inverse(const Rigid3f& r) {
  const Quatf rot = QuatConjugate(r.q);
  const Vec3f v = Rotate(rot, r.t);
  return Rigid3f{Vec3f{-v.x, -v.y, -v.z}, rot};
}
Rigid3f Rigid3Mul(const Rigid3f& a, const Rigid3f& b) {
  const Vec3f v = Rotate(a.q, b.t);
  return Rigid3f{Vec3f{v.x + a.t.x, v.y + a.t.y, v.z + a.t.z}, QuatNormalized(QuatMul(a.q, b.q))};
}
float GetYaw(const Quatf& q) {
  const Vec3f d = Rotate(q, Vec3f{1.f, 0.f, 0.f});
  return std::atan2(d.y, d.x);
}
Quatf AngleAxisVectorToRotationQuaternion(const Vec3f& aa) {
  float scale = 0.5f;
  float w = 1.f;
  constexpr double kCutoffAngle = 1e-8;
  const float squared_norm = aa.x * aa.x + aa.y * aa.y + aa.z * aa.z;
  if (squared_norm > kCutoffAngle) {
    const float norm = std::sqrt(squared_norm);
    scale = static_cast<float>(std::sin(norm / 2.) / norm);
    w = static_cast<float>(std::cos(norm / 2.));
  }
  return Quatf{w, scale * aa.x, scale * aa.y, scale * aa.z};
}

// ---- HybridGridBase ------------------------------------------------------------
namespace {
inline int Flat3(int x, int y, int z, int bits) { return (((z << bits) + y) << bits) + x; }
}  // namespace

template <typename T>
T HybridGridBase<T>::value(const Array3i& index) const {
  const int gs = grid_size();
  const int sx = index.x + (gs >> 1), sy = index.y + (gs >> 1), sz = index.z + (gs >> 1);
  if (static_cast<unsigned>(sx) >= static_cast<unsigned>(gs) ||
      static_cast<unsigned>(sy) >= static_cast<unsigned>(gs) ||
      static_cast<unsigned>(sz) >= static_cast<unsigned>(gs)) {
    return T();
  }
  const int mx = sx / 64, my = sy / 64, mz = sz / 64;
  const Nested* nested = meta_[Flat3(mx, my, mz, bits_)].get();
  if (nested == nullptr) return T();
  const int ix = sx - mx * 64, iy = sy - my * 64, iz = sz - mz * 64;
  const int fx = ix / 8, fy = iy / 8, fz = iz / 8;
  const Flat* flat = nested->cells[Flat3(fx, fy, fz, 3)].get();
  if (flat == nullptr) return T();
  return flat->cells[Flat3(ix - fx * 8, iy - fy * 8, iz - fz * 8, 3)];
}

template <typename T>
T* HybridGridBase<T>::mutable_value(const Array3i& index) {
  for (;;) {
    const int gs = grid_size();
    const int sx = index.x + (gs >> 1), sy = index.y + (gs >> 1), sz = index.z + (gs >> 1);
    if (static_cast<unsigned>(sx) >= static_cast<unsigned>(gs) ||
        static_cast<unsigned>(sy) >= static_cast<unsigned>(gs) ||
        static_cast<unsigned>(sz) >= static_cast<unsigned>(gs)) {
      Grow();
      continue;
    }
    const int mx = sx / 64, my = sy / 64, mz = sz / 64;
    std::unique_ptr<Nested>& nested = meta_[Flat3(mx, my, mz, bits_)];
    if (nested == nullptr) nested.reset(new Nested);
    const int ix = sx - mx * 64, iy = sy - my * 64, iz = sz - mz * 64;
    const int fx = ix / 8, fy = iy / 8, fz = iz / 8;
    std::unique_ptr<Flat>& flat = nested->cells[Flat3(fx, fy, fz, 3)];
    if (flat == nullptr) flat.reset(new Flat);
    return &flat->cells[Flat3(ix - fx * 8, iy - fy * 8, iz - fz * 8, 3)];
  }
}

template <typename T>
void HybridGridBase<T>::Grow() {
  const int new_bits = bits_ + 1;
  std::vector<std::unique_ptr<Nested>> grown(8 * meta_.size());
  for (int z = 0; z != (1 << bits_); ++z)
    for (int y = 0; y != (1 << bits_); ++y)
      for (int x = 0; x != (1 << bits_); ++x) {
        const int o = 1 << (bits_ - 1);
        grown[Flat3(x + o, y + o, z + o, new_bits)] = std::move(meta_[Flat3(x, y, z, bits_)]);
      }
  meta_ = std::move(grown);
  bits_ = new_bits;
}

template <typename T>
void HybridGridBase<T>::ForEach(const std::function<void(const Array3i&, T)>& fn) const {
  const int half = (1 << (bits_ - 1)) * 64;
  const int mask = (1 << bits_) - 1;
  for (size_t m = 0; m < meta_.size(); ++m) {
    const Nested* nested = meta_[m].get();
    if (!nested) continue;
    const int mx = m & mask, my = (m >> bits_) & mask, mz = (m >> bits_) >> bits_;
    for (int f = 0; f < 512; ++f) {
      const Flat* flat = nested->cells[f].get();
      if (!flat) continue;
      const int fx = f & 7, fy = (f >> 3) & 7, fz = f >> 6;
      for (int c = 0; c < 512; ++c) {
        const T v = flat->cells[c];
        if (v == T()) continue;
        fn(Array3i{mx * 64 + fx * 8 + (c & 7) - half, my * 64 + fy * 8 + ((c >> 3) & 7) - half,
                   mz * 64 + fz * 8 + (c >> 6) - half},
           v);
      }
    }
  }
}

template class HybridGridBase<uint16_t>;
template class HybridGridBase<uint8_t>;

HybridGrid::HybridGrid(float resolution)
    : HybridGridBase<uint16_t>(resolution),
      value_to_probability_(std::make_shared<const std::vector<float>>(
          PrecomputeValueToBoundedFloat(kUnknownProbabilityValue, kMinProbability,
                                        kMinProbability, kMaxProbability))) {}

// ---- precomputation_grid_3d.cc -----------------------------------------------------
PrecomputationGrid3D ConvertToPrecomputationGrid(const HybridGrid& hybrid_grid) {
  PrecomputationGrid3D result(hybrid_grid.resolution());
  const std::vector<float> table = PrecomputeValueToBoundedFloat(
      kUnknownProbabilityValue, kMinProbability, kMinProbability, kMaxProbability);
  hybrid_grid.ForEach([&](const Array3i& index, uint16_t value) {
    const int cell_value = RoundToInt((table[value] - kMinProbability) *
                                      (255.f / (kMaxProbability - kMinProbability)));
    *result.mutable_value(index) = static_cast<uint8_t>(cell_value);
  });
  return result;
}

PrecomputationGrid3D PrecomputeGrid(const PrecomputationGrid3D& grid, const bool half_resolution,
                                    const Array3i& shift) {
  PrecomputationGrid3D result(grid.resolution());
  grid.ForEach([&](const Array3i& index, uint8_t value) {
    for (int i = 0; i != 8; ++i) {
      Array3i c{index.x - shift.x * ((i & 1) ? 1 : 0), index.y - shift.y * ((i & 2) ? 1 : 0),
                index.z - shift.z * ((i & 4) ? 1 : 0)};
      if (half_resolution) c = Array3i{c.x >> 1, c.y >> 1, c.z >> 1};
      uint8_t* const cell = result.mutable_value(c);
      *cell = std::max(value, *cell);
    }
  });
  return result;
}

// fast_correlative_scan_matcher_3d.cc:57-77
PrecomputationGridStack3D::PrecomputationGridStack3D(const HybridGrid& hybrid_grid,
                                                     const FastOptions3D& options) {
  grids_.reserve(options.branch_and_bound_depth);
  grids_.push_back(ConvertToPrecomputationGrid(hybrid_grid));
  int last_width = 1;
  for (int depth = 1; depth != options.branch_and_bound_depth; ++depth) {
    const bool half_resolution = depth >= options.full_resolution_depth;
    const int next_width = 1 << depth;
    const int full_voxels_per_high_resolution_voxel =
        1 << std::max(0, depth - options.full_resolution_depth);
    const int shift = (next_width - last_width + (full_voxels_per_high_resolution_voxel - 1)) /
                      full_voxels_per_high_resolution_voxel;
    grids_.push_back(PrecomputeGrid(grids_.back(), half_resolution, Array3i{shift, shift, shift}));
    last_width = next_width;
  }
}

// ---- rotational_scan_matcher.cc ---------------------------------------------------
std::vector<float> RotateHistogram(const std::vector<float>& histogram, const float angle) {
  if (histogram.empty()) return histogram;
  const int size = static_cast<int>(histogram.size());
  const float rotate_by_buckets =
      static_cast<float>((-angle * static_cast<float>(histogram.size())) / M_PI);
  int full_buckets = RoundToInt(rotate_by_buckets - 0.5f);
  const float fraction = rotate_by_buckets - full_buckets;
  while (full_buckets < 0) full_buckets += size;
  std::vector<float> out(size);
  for (int i = 0; i != size; ++i) {
    const float r0 = histogram[(i + full_buckets) % size];
    const float r1 = histogram[(i + 1 + full_buckets) % size];
    out[i] = fraction * r1 + (1.f - fraction) * r0;
  }
  return out;
}

float MatchHistograms(const std::vector<float>& submap_histogram,
                      const std::vector<float>& scan_histogram) {
  float scan_sq = 0.f, submap_sq = 0.f, dot = 0.f;
  for (size_t i = 0; i < scan_histogram.size(); ++i) {
    scan_sq += scan_histogram[i] * scan_histogram[i];
    submap_sq += submap_histogram[i] * submap_histogram[i];
    dot += submap_histogram[i] * scan_histogram[i];
  }
  const float normalization = std::sqrt(scan_sq) * std::sqrt(submap_sq);
  if (normalization < 1e-3f) return 1.f;
  return dot / normalization;
}

std::vector<float> RotationalMatch(const std::vector<float>& submap_histogram,
                                   const std::vector<float>& histogram, const float initial_angle,
                                   const std::vector<float>& angles) {
  std::vector<float> result;
  result.reserve(angles.size());
  for (const float angle : angles) {
    result.push_back(
        MatchHistograms(submap_histogram, RotateHistogram(histogram, initial_angle + angle)));
  }
  return result;
}

// ---- low_resolution_matcher.cc:23-35 -----------------------------------------------
std::function<float(const Rigid3f&)> CreateLowResolutionMatcher(const HybridGrid* grid,
                                                                const PointCloud* points) {
  return [=](const Rigid3f& pose) {
    float score = 0.f;
    for (const Vec3f& point : *points) {
      score += grid->GetProbability(grid->GetCellIndex(Rigid3Apply(pose, point)));
    }
    if (stats3_) stats3_->low_resolution_evaluations += 1;
    return score / static_cast<float>(points->size());
  };
}

// ---- fast_correlative_scan_matcher_3d.cc -------------------------------------------
struct FastCorrelativeScanMatcher3D::Candidate3D {  // :86-110
  Candidate3D(int scan_index, const Array3i& offset) : scan_index(scan_index), offset(offset) {}
  static Candidate3D Unsuccessful() { return Candidate3D(0, Array3i{0, 0, 0}); }
  int scan_index;
  Array3i offset;
  float score = -std::numeric_limits<float>::infinity();
  float low_resolution_score = 0.f;
  bool operator<(const Candidate3D& other) const { return score < other.score; }
  bool operator>(const Candidate3D& other) const { return score > other.score; }
};

FastCorrelativeScanMatcher3D::FastCorrelativeScanMatcher3D(
    const HybridGrid& hybrid_grid, const HybridGrid* const low_resolution_hybrid_grid,
    const std::vector<float>* rotational_scan_matcher_histogram, const FastOptions3D& options)
    : options_(options),
      resolution_(hybrid_grid.resolution()),
      width_in_voxels_(hybrid_grid.grid_size()),
      stack_(new PrecomputationGridStack3D(hybrid_grid, options)),
      low_resolution_hybrid_grid_(low_resolution_hybrid_grid),
      rotational_histogram_(rotational_scan_matcher_histogram) {}

FastCorrelativeScanMatcher3D::~FastCorrelativeScanMatcher3D() {}

namespace {
Rigid3f CastRigid(const Rigid3d& r) {
  return Rigid3f{Vec3f{static_cast<float>(r.t.x), static_cast<float>(r.t.y),
                       static_cast<float>(r.t.z)},
                 Quatf{static_cast<float>(r.q.w), static_cast<float>(r.q.x),
                       static_cast<float>(r.q.y), static_cast<float>(r.q.z)}};
}
float Norm3(const Vec3f& p) { return std::sqrt(p.x * p.x + p.y * p.y + p.z * p.z); }
}  // namespace

// :127-144
std::unique_ptr<Result3D> FastCorrelativeScanMatcher3D::Match(
    const Rigid3d& global_node_pose, const Rigid3d& global_submap_pose, const NodeData3D& data,
    const float min_score, MatchStats3D* stats) const {
  const auto low_resolution_matcher =
      CreateLowResolutionMatcher(low_resolution_hybrid_grid_, &data.low_resolution_point_cloud);
  const SearchParameters sp{RoundToInt(options_.linear_xy_search_window / resolution_),
                            RoundToInt(options_.linear_z_search_window / resolution_),
                            options_.angular_search_window, &low_resolution_matcher};
  return MatchWithSearchParameters(sp, CastRigid(global_node_pose), CastRigid(global_submap_pose),
                                   data.high_resolution_point_cloud,
                                   data.rotational_scan_matcher_histogram, data.gravity_alignment,
                                   min_score, stats);
}

// :146-170
std::unique_ptr<Result3D> FastCorrelativeScanMatcher3D::MatchFullSubmap(
    const Quatd& global_node_rotation, const Quatd& global_submap_rotation,
    const NodeData3D& data, const float min_score, MatchStats3D* stats) const {
  float max_point_distance = 0.f;
  for (const Vec3f& point : data.high_resolution_point_cloud) {
    max_point_distance = std::max(max_point_distance, Norm3(point));
  }
  const int linear_window_size =
      (width_in_voxels_ + 1) / 2 + RoundToInt(max_point_distance / resolution_ + 0.5f);
  const auto low_resolution_matcher =
      CreateLowResolutionMatcher(low_resolution_hybrid_grid_, &data.low_resolution_point_cloud);
  const SearchParameters sp{linear_window_size, linear_window_size, M_PI, &low_resolution_matcher};
  const Rigid3f node{Vec3f{0.f, 0.f, 0.f},
                     Quatf{static_cast<float>(global_node_rotation.w),
                           static_cast<float>(global_node_rotation.x),
                           static_cast<float>(global_node_rotation.y),
                           static_cast<float>(global_node_rotation.z)}};
  const Rigid3f submap{Vec3f{0.f, 0.f, 0.f},
                       Quatf{static_cast<float>(global_submap_rotation.w),
                             static_cast<float>(global_submap_rotation.x),
                             static_cast<float>(global_submap_rotation.y),
                             static_cast<float>(global_submap_rotation.z)}};
  return MatchWithSearchParameters(sp, node, submap, data.high_resolution_point_cloud,
                                   data.rotational_scan_matcher_histogram, data.gravity_alignment,
                                   min_score, stats);
}

// :172-198
std::unique_ptr<Result3D> FastCorrelativeScanMatcher3D::MatchWithSearchParameters(
    const SearchParameters& sp, const Rigid3f& global_node_pose, const Rigid3f& global_submap_pose,
    const PointCloud& point_cloud, const std::vector<float>& rotational_scan_matcher_histogram,
    const Quatd& gravity_alignment, const float min_score, MatchStats3D* stats) const {
  stats3_ = stats;
  const std::vector<DiscreteScan3D> discrete_scans =
      GenerateDiscreteScans(sp, point_cloud, rotational_scan_matcher_histogram, gravity_alignment,
                            global_node_pose, global_submap_pose, stats);
  const std::vector<Candidate3D> lowest_resolution_candidates =
      ComputeLowestResolutionCandidates(sp, discrete_scans);
  if (stats) {
    stats->lowest_resolution_candidates = lowest_resolution_candidates.size();
    stats->num_scans = static_cast<int>(discrete_scans.size());
  }
  const Candidate3D best_candidate = BranchAndBound(sp, discrete_scans,
                                                    lowest_resolution_candidates,
                                                    stack_->max_depth(), min_score);
  stats3_ = nullptr;
  if (best_candidate.score > min_score) {
    const Rigid3f pose = GetPoseFromCandidate(discrete_scans, best_candidate);
    if (stats) {
      stats->best_scan_index = best_candidate.scan_index;
      stats->best_x = best_candidate.offset.x;
      stats->best_y = best_candidate.offset.y;
      stats->best_z = best_candidate.offset.z;
    }
    return std::unique_ptr<Result3D>(new Result3D{
        best_candidate.score,
        Rigid3d{Vec3d{pose.t.x, pose.t.y, pose.t.z}, Quatd{pose.q.w, pose.q.x, pose.q.y, pose.q.z}},
        discrete_scans[best_candidate.scan_index].rotational_score,
        best_candidate.low_resolution_score});
  }
  return nullptr;
}

// :200-244
FastCorrelativeScanMatcher3D::DiscreteScan3D FastCorrelativeScanMatcher3D::DiscretizeScan(
    const SearchParameters& sp, const PointCloud& point_cloud, const Rigid3f& pose,
    const float rotational_score) const {
  std::vector<std::vector<Array3i>> cell_indices_per_depth;
  const PrecomputationGrid3D& original_grid = stack_->Get(0);
  std::vector<Array3i> full_resolution_cell_indices;
  full_resolution_cell_indices.reserve(point_cloud.size());
  for (const Vec3f& point : point_cloud) {
    full_resolution_cell_indices.push_back(original_grid.GetCellIndex(Rigid3Apply(pose, point)));
  }
  const int full_resolution_depth =
      std::min(options_.full_resolution_depth, options_.branch_and_bound_depth);
  for (int i = 0; i != full_resolution_depth; ++i) {
    cell_indices_per_depth.push_back(full_resolution_cell_indices);
  }
  const int low_resolution_depth = options_.branch_and_bound_depth - full_resolution_depth;
  const Array3i start{-sp.linear_xy_window_size, -sp.linear_xy_window_size,
                      -sp.linear_z_window_size};
  for (int i = 0; i != low_resolution_depth; ++i) {
    const int e = i + 1;
    const Array3i low_start{start.x >> e, start.y >> e, start.z >> e};
    cell_indices_per_depth.emplace_back();
    cell_indices_per_depth.back().reserve(full_resolution_cell_indices.size());
    for (const Array3i& c : full_resolution_cell_indices) {
      cell_indices_per_depth.back().push_back(
          Array3i{((c.x + start.x) >> e) - low_start.x, ((c.y + start.y) >> e) - low_start.y,
                  ((c.z + start.z) >> e) - low_start.z});
    }
  }
  return DiscreteScan3D{pose, std::move(cell_indices_per_depth), rotational_score};
}

// :246-295
std::vector<FastCorrelativeScanMatcher3D::DiscreteScan3D>
FastCorrelativeScanMatcher3D::GenerateDiscreteScans(
    const SearchParameters& sp, const PointCloud& point_cloud,
    const std::vector<float>& rotational_scan_matcher_histogram, const Quatd& gravity_alignment,
    const Rigid3f& global_node_pose, const Rigid3f& global_submap_pose,
    MatchStats3D* stats) const {
  std::vector<DiscreteScan3D> result;
  float max_scan_range = 3.f * resolution_;
  for (const Vec3f& point : point_cloud) {
    max_scan_range = std::max(Norm3(point), max_scan_range);
  }
  const float kSafetyMargin = 1.f - 1e-2f;
  const float angular_step_size =
      kSafetyMargin *
      std::acos(1.f - Pow2(resolution_) / (2.f * Pow2(max_scan_range)));
  const int angular_window_size = RoundToInt(sp.angular_search_window / angular_step_size);
  std::vector<float> angles;
  for (int rz = -angular_window_size; rz <= angular_window_size; ++rz) {
    angles.push_back(rz * angular_step_size);
  }
  if (stats) stats->num_angles = static_cast<int>(angles.size());
  const Rigid3f node_to_submap = Rigid3Mul(Rigid3Inverse(global_submap_pose), global_node_pose);
  const std::vector<float> scores = RotationalMatch(
      *rotational_histogram_, rotational_scan_matcher_histogram,
      GetYaw(QuatMul(node_to_submap.q, QuatCastInverseD(gravity_alignment))), angles);
  for (size_t i = 0; i != angles.size(); ++i) {
    if (scores[i] < options_.min_rotational_score) continue;
    const Vec3f angle_axis{0.f, 0.f, angles[i]};
    const Rigid3f pose{node_to_submap.t,
                       QuatMul(QuatMul(QuatInverse(global_submap_pose.q),
                                       AngleAxisVectorToRotationQuaternion(angle_axis)),
                               global_node_pose.q)};
    result.push_back(DiscretizeScan(sp, point_cloud, pose, scores[i]));
  }
  return result;
}

// :297-330
std::vector<FastCorrelativeScanMatcher3D::Candidate3D>
FastCorrelativeScanMatcher3D::GenerateLowestResolutionCandidates(
    const SearchParameters& sp, const int num_discrete_scans) const {
  const int linear_step_size = 1 << stack_->max_depth();
  std::vector<Candidate3D> candidates;
  for (int scan_index = 0; scan_index != num_discrete_scans; ++scan_index) {
    for (int z = -sp.linear_z_window_size; z <= sp.linear_z_window_size; z += linear_step_size) {
      for (int y = -sp.linear_xy_window_size; y <= sp.linear_xy_window_size;
           y += linear_step_size) {
        for (int x = -sp.linear_xy_window_size; x <= sp.linear_xy_window_size;
             x += linear_step_size) {
          candidates.emplace_back(scan_index, Array3i{x, y, z});
        }
      }
    }
  }
  return candidates;
}

// :338-346, the sum of one candidate (shared by ScoreCandidates and ScoreCandidatesForTest)
int FastCorrelativeScanMatcher3D::CandidateSum(const int depth,
                                               const DiscreteScan3D& discrete_scan,
                                               const Array3i& candidate_offset) const {
  const int reduction_exponent = std::max(0, depth - options_.full_resolution_depth + 1);
  const PrecomputationGrid3D& grid = stack_->Get(depth);
  int sum = 0;
  const Array3i offset{candidate_offset.x >> reduction_exponent,
                       candidate_offset.y >> reduction_exponent,
                       candidate_offset.z >> reduction_exponent};
  for (const Array3i& cell_index : discrete_scan.cell_indices_per_depth[depth]) {
    sum += grid.value(
        Array3i{cell_index.x + offset.x, cell_index.y + offset.y, cell_index.z + offset.z});
  }
  return sum;
}

// :332-355
void FastCorrelativeScanMatcher3D::ScoreCandidates(
    const int depth, const std::vector<DiscreteScan3D>& discrete_scans,
    std::vector<Candidate3D>* const candidates) const {
  for (Candidate3D& candidate : *candidates) {
    const DiscreteScan3D& discrete_scan = discrete_scans[candidate.scan_index];
    const int sum = CandidateSum(depth, discrete_scan, candidate.offset);
    candidate.score = ToProbability3D(
        sum / static_cast<float>(discrete_scan.cell_indices_per_depth[depth].size()));
  }
  if (stats3_) stats3_->candidates_scored += candidates->size();
  std::sort(candidates->begin(), candidates->end(), std::greater<Candidate3D>());
}

// :357-367
std::vector<FastCorrelativeScanMatcher3D::Candidate3D>
FastCorrelativeScanMatcher3D::ComputeLowestResolutionCandidates(
    const SearchParameters& sp, const std::vector<DiscreteScan3D>& discrete_scans) const {
  std::vector<Candidate3D> lowest_resolution_candidates =
      GenerateLowestResolutionCandidates(sp, static_cast<int>(discrete_scans.size()));
  ScoreCandidates(stack_->max_depth(), discrete_scans, &lowest_resolution_candidates);
  return lowest_resolution_candidates;
}

// :369-375
Rigid3f FastCorrelativeScanMatcher3D::GetPoseFromCandidate(
    const std::vector<DiscreteScan3D>& discrete_scans, const Candidate3D& candidate) const {
  const Rigid3f translation{
      Vec3f{resolution_ * static_cast<float>(candidate.offset.x),
            resolution_ * static_cast<float>(candidate.offset.y),
            resolution_ * static_cast<float>(candidate.offset.z)},
      Quatf{1.f, 0.f, 0.f, 0.f}};
  return Rigid3Mul(translation, discrete_scans[candidate.scan_index].pose);
}

// :377-440
FastCorrelativeScanMatcher3D::Candidate3D FastCorrelativeScanMatcher3D::BranchAndBound(
    const SearchParameters& sp, const std::vector<DiscreteScan3D>& discrete_scans,
    const std::vector<Candidate3D>& candidates, const int candidate_depth,
    float min_score) const {
  if (candidate_depth == 0) {
    for (const Candidate3D& candidate : candidates) {
      if (candidate.score <= min_score) return Candidate3D::Unsuccessful();
      const float low_resolution_score =
          (*sp.low_resolution_matcher)(GetPoseFromCandidate(discrete_scans, candidate));
      if (low_resolution_score >= options_.min_low_resolution_score) {
        Candidate3D best_candidate = candidate;
        best_candidate.low_resolution_score = low_resolution_score;
        return best_candidate;
      }
    }
    return Candidate3D::Unsuccessful();
  }
  Candidate3D best_high_resolution_candidate = Candidate3D::Unsuccessful();
  best_high_resolution_candidate.score = min_score;
  for (const Candidate3D& candidate : candidates) {
    if (candidate.score <= min_score) break;
    std::vector<Candidate3D> higher_resolution_candidates;
    const int half_width = 1 << (candidate_depth - 1);
    for (int z : {0, half_width}) {
      if (candidate.offset.z + z > sp.linear_z_window_size) break;
      for (int y : {0, half_width}) {
        if (candidate.offset.y + y > sp.linear_xy_window_size) break;
        for (int x : {0, half_width}) {
          if (candidate.offset.x + x > sp.linear_xy_window_size) break;
          higher_resolution_candidates.emplace_back(
              candidate.scan_index,
              Array3i{candidate.offset.x + x, candidate.offset.y + y, candidate.offset.z + z});
        }
      }
    }
    if (stats3_) stats3_->nodes_expanded += 1;
    ScoreCandidates(candidate_depth - 1, discrete_scans, &higher_resolution_candidates);
    best_high_resolution_candidate = std::max(
        best_high_resolution_candidate,
        BranchAndBound(sp, discrete_scans, higher_resolution_candidates, candidate_depth - 1,
                       best_high_resolution_candidate.score));
  }
  return best_high_resolution_candidate;
}

std::vector<FastCorrelativeScanMatcher3D::DiscreteScan3D>
FastCorrelativeScanMatcher3D::GenerateDiscreteScansForTest(bool full,
                                                           const Rigid3d& global_node_pose,
                                                           const Rigid3d& global_submap_pose,
                                                           const NodeData3D& data) const {
  SearchParameters sp{RoundToInt(options_.linear_xy_search_window / resolution_),
                      RoundToInt(options_.linear_z_search_window / resolution_),
                      options_.angular_search_window, nullptr};
  Rigid3f node = CastRigid(global_node_pose), submap = CastRigid(global_submap_pose);
  if (full) {
    float max_point_distance = 0.f;
    for (const Vec3f& p : data.high_resolution_point_cloud)
      max_point_distance = std::max(max_point_distance, Norm3(p));
    const int w = (width_in_voxels_ + 1) / 2 + RoundToInt(max_point_distance / resolution_ + 0.5f);
    sp = SearchParameters{w, w, M_PI, nullptr};
    node.t = Vec3f{0.f, 0.f, 0.f};
    submap.t = Vec3f{0.f, 0.f, 0.f};
  }
  return GenerateDiscreteScans(sp, data.high_resolution_point_cloud,
                               data.rotational_scan_matcher_histogram, data.gravity_alignment,
                               node, submap, nullptr);
}

void FastCorrelativeScanMatcher3D::ScoreCandidatesForTest(
    bool full, const Rigid3d& global_node_pose, const Rigid3d& global_submap_pose,
    const NodeData3D& data, int depth, const std::vector<std::array<int, 4>>& candidates,
    int* sums, float* scores, float* low_resolution_scores) const {
  const std::vector<DiscreteScan3D> discrete_scans =
      GenerateDiscreteScansForTest(full, global_node_pose, global_submap_pose, data);
  const auto low_resolution_matcher =
      CreateLowResolutionMatcher(low_resolution_hybrid_grid_, &data.low_resolution_point_cloud);
  for (size_t i = 0; i < candidates.size(); ++i) {
    const std::array<int, 4>& c = candidates[i];
    Candidate3D candidate(c[0], Array3i{c[1], c[2], c[3]});
    const DiscreteScan3D& discrete_scan = discrete_scans.at(candidate.scan_index);
    sums[i] = CandidateSum(depth, discrete_scan, candidate.offset);
    scores[i] = ToProbability3D(
        sums[i] / static_cast<float>(discrete_scan.cell_indices_per_depth[depth].size()));
    if (depth == 0 && low_resolution_scores)
      low_resolution_scores[i] =
          low_resolution_matcher(GetPoseFromCandidate(discrete_scans, candidate));
  }
}

// ---- real_time_correlative_scan_matcher_3d.cc ---------------------------------------
// transform/transform.h:34-37: 2 * atan2(rotation.vec().norm(), |rotation.w()|)
float GetAngle(const Rigid3f& transform) {
  const float vec_norm = std::sqrt(transform.q.x * transform.q.x + transform.q.y * transform.q.y +
                                   transform.q.z * transform.q.z);
  return 2.f * std::atan2(vec_norm, std::abs(transform.q.w));
}

// .cc:55-98
std::vector<Rigid3f> RealTimeCorrelativeScanMatcher3D::GenerateExhaustiveSearchTransforms(
    const float resolution, const PointCloud& point_cloud) const {
  std::vector<Rigid3f> result;
  const int linear_window_size = RoundToInt(options_.linear_search_window / resolution);
  // "something on the order of resolution to make sure that the std::acos() below is defined"
  float max_scan_range = 3.f * resolution;
  for (const Vec3f& point : point_cloud) {
    const float range = std::sqrt(point.x * point.x + point.y * point.y + point.z * point.z);
    max_scan_range = std::max(range, max_scan_range);
  }
  const float kSafetyMargin = 1.f - 1e-3f;
  const float angular_step_size =
      kSafetyMargin * std::acos(1.f - (resolution * resolution) /
                                          (2.f * (max_scan_range * max_scan_range)));
  const int angular_window_size = RoundToInt(options_.angular_search_window / angular_step_size);
  for (int z = -linear_window_size; z <= linear_window_size; ++z) {
    for (int y = -linear_window_size; y <= linear_window_size; ++y) {
      for (int x = -linear_window_size; x <= linear_window_size; ++x) {
        for (int rz = -angular_window_size; rz <= angular_window_size; ++rz) {
          for (int ry = -angular_window_size; ry <= angular_window_size; ++ry) {
            for (int rx = -angular_window_size; rx <= angular_window_size; ++rx) {
              const Vec3f angle_axis{rx * angular_step_size, ry * angular_step_size,
                                     rz * angular_step_size};
              result.push_back(Rigid3f{Vec3f{x * resolution, y * resolution, z * resolution},
                                       AngleAxisVectorToRotationQuaternion(angle_axis)});
            }
          }
        }
      }
    }
  }
  return result;
}

// .cc:100-117
float RealTimeCorrelativeScanMatcher3D::ScoreCandidate(const HybridGrid& hybrid_grid,
                                                       const PointCloud& transformed_point_cloud,
                                                       const Rigid3f& transform) const {
  float score = 0.f;
  for (const Vec3f& point : transformed_point_cloud) {
    score += hybrid_grid.GetProbability(hybrid_grid.GetCellIndex(point));
  }
  score /= static_cast<float>(transformed_point_cloud.size());
  const float angle = GetAngle(transform);
  const float t_norm = std::sqrt(transform.t.x * transform.t.x + transform.t.y * transform.t.y +
                                 transform.t.z * transform.t.z);
  const double e = t_norm * options_.translation_delta_cost_weight +
                   angle * options_.rotation_delta_cost_weight;
  score *= std::exp(-(e * e));   // float *= double
  return score;                  // (CHECK_GT(score, 0.f) in the reference)
}

// .cc:34-53
float RealTimeCorrelativeScanMatcher3D::Match(const Rigid3d& initial_pose_estimate,
                                              const PointCloud& point_cloud,
                                              const HybridGrid& hybrid_grid,
                                              Rigid3d* pose_estimate, int64_t* num_candidates,
                                              int64_t* best_index,
                                              std::vector<float>* scores) const {
  float best_score = -1.f;
  // initial_pose_estimate.cast<float>()
  const Rigid3f initial{
      Vec3f{static_cast<float>(initial_pose_estimate.t.x),
            static_cast<float>(initial_pose_estimate.t.y),
            static_cast<float>(initial_pose_estimate.t.z)},
      Quatf{static_cast<float>(initial_pose_estimate.q.w),
            static_cast<float>(initial_pose_estimate.q.x),
            static_cast<float>(initial_pose_estimate.q.y),
            static_cast<float>(initial_pose_estimate.q.z)}};
  const std::vector<Rigid3f> transforms =
      GenerateExhaustiveSearchTransforms(hybrid_grid.resolution(), point_cloud);
  int64_t index = 0;
  PointCloud transformed(point_cloud.size());
  for (const Rigid3f& transform : transforms) {
    const Rigid3f candidate = Rigid3Mul(initial, transform);
    for (size_t i = 0; i < point_cloud.size(); ++i)   // sensor::TransformPointCloud
      transformed[i] = Rigid3Apply(candidate, point_cloud[i]);
    const float score = ScoreCandidate(hybrid_grid, transformed, transform);
    if (scores) scores->push_back(score);
    if (score > best_score) {
      best_score = score;
      *pose_estimate = Rigid3d{Vec3d{candidate.t.x, candidate.t.y, candidate.t.z},
                               Quatd{candidate.q.w, candidate.q.x, candidate.q.y, candidate.q.z}};
      if (best_index) *best_index = index;
    }
    ++index;
  }
  if (num_candidates) *num_candidates = static_cast<int64_t>(transforms.size());
  return best_score;
}

}  // namespace oracle
