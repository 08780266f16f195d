// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_common.h).
// 3D path: HybridGrid, PrecomputationGrid3D stack, RotationalScanMatcher,
// low-resolution matcher, FastCorrelativeScanMatcher3D.
//
// Eigen semantics restated from Eigen 3.3 (not present in this image, so these
// cannot be re-read here — SURVEY.md Appendix B): on x86-64 Eigen uses its SSE
// specialisation of Quaternionf * Quaternionf and 4-lane packet reductions for
// squaredNorm(); both are written out below in that operation order.  Reductions
// over VectorXf (rotational histograms) are restated sequentially; Eigen's SIMD
// order differs in the last ulp, which is inside the reference's own 1e-6 test
// tolerance (rotational_scan_matcher_test.cc:34,53) — "parity unpinned" for the
// last bit of rotational scores only.
#ifndef ORACLE_3D_H_
#define ORACLE_3D_H_

#include <array>
#include <cstdint>
#include <functional>
#include <memory>
#include <vector>

#include "oracle_common.h"

namespace oracle {

struct Array3i { int x, y, z; };
struct Quatd { double w, x, y, z; };
struct Vec3d { double x, y, z; };
struct Rigid3f { Vec3f t; Quatf q; };
struct Rigid3d { Vec3d t; Quatd q; };

// Eigen 3.3 Geometry/arch/Geometry_SSE.h quat_product<SSE, float>.
Quatf QuatMul(const Quatf& a, const Quatf& b);
// coeffs().squaredNorm() with the Packet4f predux order (x²+z²)+(y²+w²).
float QuatSquaredNorm(const Quatf& q);
Quatf QuatNormalized(const Quatf& q);      // q / sqrt(squaredNorm) if > 0
Quatf QuatInverse(const Quatf& q);         // conjugate / squaredNorm
Quatf QuatConjugate(const Quatf& q);
Quatf QuatCastInverseD(const Quatd& q);    // q.inverse().cast<float>()
// transform/rigid_transform.h:148-152 (inverse) and :181-189 (operator*).
Rigid3f Rigid3Inverse(const Rigid3f& r);
Rigid3f Rigid3Mul(const Rigid3f& a, const Rigid3f& b);
Vec3f Rigid3Apply(const Rigid3f& r, const Vec3f& p);   // :192-196
float GetYaw(const Quatf& q);                          // transform/transform.h:42-47
Quatf AngleAxisVectorToRotationQuaternion(const Vec3f& aa);  // transform/transform.h:85-99

// ---- mapping/3d/hybrid_grid.h ------------------------------------------------
// DynamicGrid<NestedGrid<FlatGrid<T,3>,3>>: 8^3 flat cells inside 8^3 nested
// cells inside a 2^bits cube that doubles as needed (:250-407).
template <typename T>
class HybridGridBase {
 public:
  explicit HybridGridBase(float resolution) : resolution_(resolution), bits_(1), meta_(8) {}
  HybridGridBase(HybridGridBase&&) = default;
  float resolution() const { return resolution_; }
  int grid_size() const { return 64 << bits_; }                       // :258

  // hybrid_grid.h:428-433
  Array3i GetCellIndex(const Vec3f& p) const {
    return Array3i{RoundToInt(p.x / resolution_), RoundToInt(p.y / resolution_),
                   RoundToInt(p.z / resolution_)};
  }
  T value(const Array3i& index) const;                                // :263-279
  T* mutable_value(const Array3i& index);                             // :283-299
  // visits every non-default cell (iteration order is irrelevant to all users)
  void ForEach(const std::function<void(const Array3i&, T)>& fn) const;

 private:
  struct Flat { std::array<T, 512> cells{}; };
  struct Nested { std::array<std::unique_ptr<Flat>, 512> cells; };
  void Grow();                                                        // :387-405
  float resolution_;
  int bits_;
  std::vector<std::unique_ptr<Nested>> meta_;
};

class HybridGrid : public HybridGridBase<uint16_t> {                  // :468-526
 public:
  explicit HybridGrid(float resolution);
  void SetProbability(const Array3i& index, float probability) {
    *mutable_value(index) = ProbabilityToValue(probability);
  }
  float GetProbability(const Array3i& index) const {                  // :521-523
    return (*value_to_probability_)[value(index)];
  }
 private:
  std::shared_ptr<const std::vector<float>> value_to_probability_;    // probability_values.cc:56-60
};

using PrecomputationGrid3D = HybridGridBase<uint8_t>;                 // precomputation_grid_3d.h:26-36
inline float ToProbability3D(float value) {                           // :32-35
  return kMinProbability + value * ((kMaxProbability - kMinProbability) / 255.f);
}
PrecomputationGrid3D ConvertToPrecomputationGrid(const HybridGrid& grid);   // .cc:49-61
PrecomputationGrid3D PrecomputeGrid(const PrecomputationGrid3D& grid, bool half_resolution,
                                    const Array3i& shift);                  // .cc:63-81

struct FastOptions3D {  // proto/scan_matching/fast_correlative_scan_matcher_options_3d.proto
  int branch_and_bound_depth;
  int full_resolution_depth;
  double min_rotational_score;
  double min_low_resolution_score;
  double linear_xy_search_window;
  double linear_z_search_window;
  double angular_search_window;
};

class PrecomputationGridStack3D {  // fast_correlative_scan_matcher_3d.cc:57-77
 public:
  PrecomputationGridStack3D(const HybridGrid& grid, const FastOptions3D& options);
  const PrecomputationGrid3D& Get(int depth) const { return grids_.at(depth); }
  int max_depth() const { return static_cast<int>(grids_.size()) - 1; }
 private:
  std::vector<PrecomputationGrid3D> grids_;
};

// rotational_scan_matcher.{h,cc}
std::vector<float> RotateHistogram(const std::vector<float>& histogram, float angle);  // :141-162
float MatchHistograms(const std::vector<float>& submap, const std::vector<float>& scan);  // :121-132
std::vector<float> RotationalMatch(const std::vector<float>& submap_histogram,
                                   const std::vector<float>& histogram, float initial_angle,
                                   const std::vector<float>& angles);                  // :178-189

// mapping/trajectory_node.h:45-63 (the fields the 3D matcher reads)
struct NodeData3D {
  Quatd gravity_alignment{1., 0., 0., 0.};
  PointCloud high_resolution_point_cloud;
  PointCloud low_resolution_point_cloud;
  std::vector<float> rotational_scan_matcher_histogram;
};

struct Result3D {  // fast_correlative_scan_matcher_3d.h:68-73
  float score;
  Rigid3d pose_estimate;
  float rotational_score;
  float low_resolution_score;
};

struct MatchStats3D {
  int64_t candidates_scored = 0;
  int64_t lowest_resolution_candidates = 0;
  int64_t nodes_expanded = 0;
  int64_t low_resolution_evaluations = 0;
  int num_scans = 0;           // discrete scans that survived the rotational filter
  int num_angles = 0;          // before the filter
  int best_scan_index = 0, best_x = 0, best_y = 0, best_z = 0;
};

class FastCorrelativeScanMatcher3D {  // fast_correlative_scan_matcher_3d.{h,cc}
 public:
  FastCorrelativeScanMatcher3D(const HybridGrid& hybrid_grid,
                               const HybridGrid* low_resolution_hybrid_grid,
                               const std::vector<float>* rotational_scan_matcher_histogram,
                               const FastOptions3D& options);
  ~FastCorrelativeScanMatcher3D();
  std::unique_ptr<Result3D> Match(const Rigid3d& global_node_pose,
                                  const Rigid3d& global_submap_pose, const NodeData3D& data,
                                  float min_score, MatchStats3D* stats = nullptr) const;
  std::unique_ptr<Result3D> MatchFullSubmap(const Quatd& global_node_rotation,
                                            const Quatd& global_submap_rotation,
                                            const NodeData3D& data, float min_score,
                                            MatchStats3D* stats = nullptr) const;
  const PrecomputationGridStack3D& stack() const { return *stack_; }

  struct DiscreteScan3D;
  struct Candidate3D;
  struct SearchParameters {
    int linear_xy_window_size;
    int linear_z_window_size;
    double angular_search_window;
    const std::function<float(const Rigid3f&)>* low_resolution_matcher;
  };
  // test hook: the discrete scans (full-resolution cell indices + poses) of a match
  std::vector<DiscreteScan3D> GenerateDiscreteScansForTest(
      bool full, const Rigid3d& global_node_pose, const Rigid3d& global_submap_pose,
      const NodeData3D& data) const;
  // test hook: the sums and scores of caller-given candidates {scan_index, x, y, z} at
  // `depth` on those discrete scans (no sort); at depth 0 also the low-resolution
  // matcher's score of GetPoseFromCandidate (low_resolution_scores may be null)
  void ScoreCandidatesForTest(bool full, const Rigid3d& global_node_pose,
                              const Rigid3d& global_submap_pose, const NodeData3D& data,
                              int depth, const std::vector<std::array<int, 4>>& candidates,
                              int* sums, float* scores, float* low_resolution_scores) const;

 private:
  int CandidateSum(int depth, const DiscreteScan3D& discrete_scan, const Array3i& offset) const;
  std::unique_ptr<Result3D> MatchWithSearchParameters(
      const SearchParameters& sp, const Rigid3f& global_node_pose,
      const Rigid3f& global_submap_pose, const PointCloud& point_cloud,
      const std::vector<float>& rotational_scan_matcher_histogram,
      const Quatd& gravity_alignment, float min_score, MatchStats3D* stats) const;
  DiscreteScan3D DiscretizeScan(const SearchParameters& sp, const PointCloud& point_cloud,
                                const Rigid3f& pose, float rotational_score) const;
  std::vector<DiscreteScan3D> GenerateDiscreteScans(
      const SearchParameters& sp, const PointCloud& point_cloud,
      const std::vector<float>& rotational_scan_matcher_histogram,
      const Quatd& gravity_alignment, const Rigid3f& global_node_pose,
      const Rigid3f& global_submap_pose, MatchStats3D* stats) const;
  std::vector<Candidate3D> GenerateLowestResolutionCandidates(const SearchParameters& sp,
                                                              int num_discrete_scans) const;
  void ScoreCandidates(int depth, const std::vector<DiscreteScan3D>& discrete_scans,
                       std::vector<Candidate3D>* candidates) const;
  std::vector<Candidate3D> ComputeLowestResolutionCandidates(
      const SearchParameters& sp, const std::vector<DiscreteScan3D>& discrete_scans) const;
  Candidate3D BranchAndBound(const SearchParameters& sp,
                             const std::vector<DiscreteScan3D>& discrete_scans,
                             const std::vector<Candidate3D>& candidates, int candidate_depth,
                             float min_score) const;
  Rigid3f GetPoseFromCandidate(const std::vector<DiscreteScan3D>& discrete_scans,
                               const Candidate3D& candidate) const;

  const FastOptions3D options_;
  const float resolution_;
  const int width_in_voxels_;
  std::unique_ptr<PrecomputationGridStack3D> stack_;
  const HybridGrid* const low_resolution_hybrid_grid_;
  const std::vector<float>* const rotational_histogram_;
};

struct FastCorrelativeScanMatcher3D::DiscreteScan3D {  // .cc:79-84
  Rigid3f pose;
  std::vector<std::vector<Array3i>> cell_indices_per_depth;
  float rotational_score;
};

// low_resolution_matcher.cc:23-35
std::function<float(const Rigid3f&)> CreateLowResolutionMatcher(const HybridGrid* grid,
                                                                const PointCloud* points);

// ---- real_time_correlative_scan_matcher_3d.{h,cc} -----------------------------------
struct RealTimeOptions3D {  // proto/scan_matching/real_time_correlative_scan_matcher_options.proto
  double linear_search_window;
  double angular_search_window;
  double translation_delta_cost_weight;
  double rotation_delta_cost_weight;
};
float GetAngle(const Rigid3f& transform);  // transform/transform.h:34-37

class RealTimeCorrelativeScanMatcher3D {  // real_time_correlative_scan_matcher_3d.h:41-67
 public:
  explicit RealTimeCorrelativeScanMatcher3D(const RealTimeOptions3D& options)
      : options_(options) {}
  // .cc:34-53; num_candidates / best_index (generation order) and every candidate's score in
  // generation order are reported for the tests
  float Match(const Rigid3d& initial_pose_estimate, const PointCloud& point_cloud,
              const HybridGrid& hybrid_grid, Rigid3d* pose_estimate,
              int64_t* num_candidates = nullptr, int64_t* best_index = nullptr,
              std::vector<float>* scores = nullptr) const;
  std::vector<Rigid3f> GenerateExhaustiveSearchTransforms(float resolution,
                                                          const PointCloud& point_cloud) const;
  float ScoreCandidate(const HybridGrid& hybrid_grid, const PointCloud& transformed_point_cloud,
                       const Rigid3f& transform) const;

 private:
  const RealTimeOptions3D options_;
};

}  // namespace oracle

#endif  // ORACLE_3D_H_
