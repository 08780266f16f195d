// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_common.h).
// 2D path: SearchParameters / rotated + discretised scans / precomputation grid
// stack / FastCorrelativeScanMatcher2D / RealTimeCorrelativeScanMatcher2D.
#ifndef ORACLE_2D_H_
#define ORACLE_2D_H_

#include <cstdint>
#include <memory>
#include <utility>
#include <vector>

#include "oracle_common.h"

namespace oracle {

// mapping/2d/xy_index.h:34-45
struct CellLimits {
  int num_x_cells = 0;
  int num_y_cells = 0;
};

struct Array2i { int x, y; };

// mapping/2d/map_limits.h:40-95
struct MapLimits {
  double resolution;
  double max_x, max_y;  // Eigen::Vector2d max_
  CellLimits cell_limits;

  // map_limits.h:69-76 — note index.x <- world y, index.y <- world x.
  Array2i GetCellIndex(const float px, const float py) const {
    return Array2i{RoundToInt((max_y - py) / resolution - 0.5),
                   RoundToInt((max_x - px) / resolution - 0.5)};
  }
  // map_limits.h:85-90
  bool Contains(const Array2i& c) const {
    return 0 <= c.x && 0 <= c.y && c.x < cell_limits.num_x_cells &&
           c.y < cell_limits.num_y_cells;
  }
};

// mapping/2d/grid_2d.h:37-141 + probability_grid.{h,cc}; read-only subset.
struct ProbabilityGrid {
  MapLimits limits;
  float min_correspondence_cost = kMinCorrespondenceCost;
  float max_correspondence_cost = kMaxCorrespondenceCost;
  std::vector<uint16_t> cells;                // num_x * y + x  (grid_2d.h:113-116)
  std::vector<float> value_to_cost_table;     // value_conversion_tables.cc:54-67

  ProbabilityGrid(const MapLimits& limits, float min_cost, float max_cost);
  explicit ProbabilityGrid(const MapLimits& limits)
      : ProbabilityGrid(limits, kMinCorrespondenceCost, kMaxCorrespondenceCost) {}

  int ToFlatIndex(const Array2i& c) const {
    return limits.cell_limits.num_x_cells * c.y + c.x;
  }
  // grid_2d.h:53-57
  float GetCorrespondenceCost(const Array2i& c) const {
    if (!limits.Contains(c)) return max_correspondence_cost;
    return value_to_cost_table[cells[ToFlatIndex(c)]];
  }
  // probability_grid.cc:78-82 (kValueToCorrespondenceCost has the same values
  // as the per-grid table for a ProbabilityGrid, probability_values.cc:56-74).
  float GetProbability(const Array2i& c) const {
    if (!limits.Contains(c)) return kMinProbability;
    return CorrespondenceCostToProbability(value_to_cost_table[cells[ToFlatIndex(c)]]);
  }
  // probability_grid.cc:41-49
  void SetProbability(const Array2i& c, const float probability) {
    cells[ToFlatIndex(c)] =
        CorrespondenceCostToValue(ProbabilityToCorrespondenceCost(probability));
  }
};

// mapping/internal/2d/tsdf_2d.{h,cc} + tsd_value_converter.{h,cc}; read-only subset.
struct TSDF2D {
  MapLimits limits;
  float truncation_distance, max_weight;
  std::vector<uint16_t> tsd_cells;      // Grid2D::correspondence_cost_cells_
  std::vector<uint16_t> weight_cells;   // tsdf_2d.h weight_cells_
  std::vector<float> value_to_tsd, value_to_weight;  // tsd_value_converter.cc:24-34

  TSDF2D(const MapLimits& limits, float truncation_distance, float max_weight);
  float GetMaxCorrespondenceCost() const { return truncation_distance; }  // tsdf_2d.cc:26-27
  // tsdf_2d.cc:86-96
  std::pair<float, float> GetTSDAndWeight(const Array2i& c) const {
    if (limits.Contains(c)) {
      const int flat = limits.cell_limits.num_x_cells * c.y + c.x;
      return std::make_pair(value_to_tsd[tsd_cells[flat]], value_to_weight[weight_cells[flat]]);
    }
    return std::make_pair(-truncation_distance, 0.f);
  }
  // tsd_value_converter.h:35-52
  uint16_t TSDToValue(float tsd) const {
    return static_cast<uint16_t>(
        RoundToInt((Clamp(tsd, -truncation_distance, truncation_distance) + truncation_distance) *
                   (32766.f / (truncation_distance - (-truncation_distance)))) + 1);
  }
  uint16_t WeightToValue(float w) const {
    return static_cast<uint16_t>(
        RoundToInt((Clamp(w, 0.f, max_weight) - 0.f) * (32766.f / (max_weight - 0.f))) + 1);
  }
};

typedef std::vector<Array2i> DiscreteScan2D;  // correlative_scan_matcher_2d.h:32

// correlative_scan_matcher_2d.h:35-60, .cc:27-91
struct SearchParameters {
  struct LinearBounds { int min_x, max_x, min_y, max_y; };

  SearchParameters(double linear_search_window, double angular_search_window,
                   const PointCloud& point_cloud, double resolution);
  SearchParameters(int num_linear_perturbations, int num_angular_perturbations,
                   double angular_perturbation_step_size, double resolution);
  void ShrinkToFit(const std::vector<DiscreteScan2D>& scans,
                   const CellLimits& cell_limits);

  int num_angular_perturbations;
  double angular_perturbation_step_size;
  double resolution;
  int num_scans;
  std::vector<LinearBounds> linear_bounds;
};

std::vector<PointCloud> GenerateRotatedScans(const PointCloud& point_cloud,
                                             const SearchParameters& sp);
std::vector<DiscreteScan2D> DiscretizeScans(const MapLimits& map_limits,
                                            const std::vector<PointCloud>& scans,
                                            float tx, float ty);

// correlative_scan_matcher_2d.h:74-103
struct Candidate2D {
  Candidate2D(const int init_scan_index, const int init_x_index_offset,
              const int init_y_index_offset, const SearchParameters& sp)
      : scan_index(init_scan_index),
        x_index_offset(init_x_index_offset),
        y_index_offset(init_y_index_offset),
        x(-y_index_offset * sp.resolution),
        y(-x_index_offset * sp.resolution),
        orientation((scan_index - sp.num_angular_perturbations) *
                    sp.angular_perturbation_step_size) {}
  int scan_index = 0;
  int x_index_offset = 0;
  int y_index_offset = 0;
  double x = 0.;
  double y = 0.;
  double orientation = 0.;
  float score = 0.f;
  bool operator<(const Candidate2D& other) const { return score < other.score; }
  bool operator>(const Candidate2D& other) const { return score > other.score; }
};

// fast_correlative_scan_matcher_2d.h:49-93, .cc:91-169
class PrecomputationGrid2D {
 public:
  PrecomputationGrid2D(const ProbabilityGrid& grid, const CellLimits& limits,
                       int width, std::vector<float>* reusable_intermediate_grid);
  int GetValue(const Array2i& xy_index) const {
    const int lx = xy_index.x - offset_.x;
    const int ly = xy_index.y - offset_.y;
    if (static_cast<unsigned>(lx) >= static_cast<unsigned>(wide_limits_.num_x_cells) ||
        static_cast<unsigned>(ly) >= static_cast<unsigned>(wide_limits_.num_y_cells)) {
      return 0;
    }
    const int stride = wide_limits_.num_x_cells;
    return cells_[lx + ly * stride];
  }
  float ToScore(float value) const {
    return min_score_ + value * ((max_score_ - min_score_) / 255.f);
  }
  const std::vector<uint8_t>& cells() const { return cells_; }
  const CellLimits& wide_limits() const { return wide_limits_; }
  float min_score() const { return min_score_; }
  float max_score() const { return max_score_; }

 private:
  uint8_t ComputeCellValue(float probability) const;
  const Array2i offset_;
  const CellLimits wide_limits_;
  const float min_score_;
  const float max_score_;
  std::vector<uint8_t> cells_;
};

struct FastOptions2D {  // proto/scan_matching/fast_correlative_scan_matcher_options_2d.proto
  double linear_search_window;
  double angular_search_window;
  int branch_and_bound_depth;
};

class PrecomputationGridStack2D {  // fast...2d.cc:171-186
 public:
  PrecomputationGridStack2D(const ProbabilityGrid& grid, const FastOptions2D& options);
  const PrecomputationGrid2D& Get(int index) const { return grids_[index]; }
  int max_depth() const { return static_cast<int>(grids_.size()) - 1; }
 private:
  std::vector<PrecomputationGrid2D> grids_;
};

struct Rigid2d { double x, y, theta; };

struct MatchStats {
  int64_t candidates_scored = 0;     // one per candidate.score assignment
  int64_t lowest_resolution_candidates = 0;
  int64_t nodes_expanded = 0;        // B&B inner ScoreCandidates calls
  int num_scans = 0;
  // winning candidate (integer identity, for bit-exact parity)
  int best_scan_index = 0, best_x_offset = 0, best_y_offset = 0;
};

class FastCorrelativeScanMatcher2D {  // fast...2d.h:112-164, .cc:188-378
 public:
  FastCorrelativeScanMatcher2D(const ProbabilityGrid& grid, const FastOptions2D& options);
  bool Match(const Rigid2d& initial_pose_estimate, const PointCloud& point_cloud,
             float min_score, float* score, Rigid2d* pose_estimate,
             MatchStats* stats = nullptr) const;
  bool MatchFullSubmap(const PointCloud& point_cloud, float min_score,
                       float* score, Rigid2d* pose_estimate,
                       MatchStats* stats = nullptr) const;
  const PrecomputationGridStack2D& stack() const { return *stack_; }
  const MapLimits& limits() const { return limits_; }

  // "visible for testing" hook mirroring ScoreCandidates (no sort when
  // sort == false so the caller can compare per-candidate).
  void ScoreCandidates(const PrecomputationGrid2D& precomputation_grid,
                       const std::vector<DiscreteScan2D>& discrete_scans,
                       const SearchParameters& search_parameters,
                       std::vector<Candidate2D>* candidates, bool sort = true) const;

 private:
  bool MatchWithSearchParameters(SearchParameters search_parameters,
                                 const Rigid2d& initial_pose_estimate,
                                 const PointCloud& point_cloud, float min_score,
                                 float* score, Rigid2d* pose_estimate,
                                 MatchStats* stats) const;
  std::vector<Candidate2D> ComputeLowestResolutionCandidates(
      const std::vector<DiscreteScan2D>& discrete_scans,
      const SearchParameters& search_parameters) const;
  std::vector<Candidate2D> GenerateLowestResolutionCandidates(
      const SearchParameters& search_parameters) const;
  Candidate2D BranchAndBound(const std::vector<DiscreteScan2D>& discrete_scans,
                             const SearchParameters& search_parameters,
                             const std::vector<Candidate2D>& candidates,
                             int candidate_depth, float min_score) const;
  const FastOptions2D options_;
  MapLimits limits_;
  std::unique_ptr<PrecomputationGridStack2D> stack_;
};

struct RealTimeOptions {  // proto/scan_matching/real_time_correlative_scan_matcher_options.proto
  double linear_search_window;
  double angular_search_window;
  double translation_delta_cost_weight;
  double rotation_delta_cost_weight;
};

class RealTimeCorrelativeScanMatcher2D {  // real_time...2d.h:53-85, .cc:77-176
 public:
  explicit RealTimeCorrelativeScanMatcher2D(const RealTimeOptions& options)
      : options_(options) {}
  // `scores` (for the tests) receives every candidate's score in generation order, as
  // max_element sees them
  double Match(const Rigid2d& initial_pose_estimate, const PointCloud& point_cloud,
               const ProbabilityGrid& grid, Rigid2d* pose_estimate,
               MatchStats* stats = nullptr, std::vector<float>* scores = nullptr) const;
  void ScoreCandidates(const ProbabilityGrid& grid,
                       const std::vector<DiscreteScan2D>& discrete_scans,
                       const SearchParameters& search_parameters,
                       std::vector<Candidate2D>* candidates) const;
  // TSDF grid type (real_time_correlative_scan_matcher_2d.cc:38-59, 160-166)
  double Match(const Rigid2d& initial_pose_estimate, const PointCloud& point_cloud,
               const TSDF2D& grid, Rigid2d* pose_estimate, MatchStats* stats = nullptr,
               std::vector<float>* scores = nullptr) const;
  void ScoreCandidates(const TSDF2D& grid, const std::vector<DiscreteScan2D>& discrete_scans,
                       const SearchParameters& search_parameters,
                       std::vector<Candidate2D>* candidates) const;
  std::vector<Candidate2D> GenerateExhaustiveSearchCandidates(
      const SearchParameters& search_parameters) const;
 private:
  const RealTimeOptions options_;
};

}  // namespace oracle

#endif  // ORACLE_2D_H_
