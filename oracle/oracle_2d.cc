// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_common.h).
// Restates mapping/internal/2d/scan_matching/{correlative_scan_matcher_2d,
// fast_correlative_scan_matcher_2d,real_time_correlative_scan_matcher_2d}.cc.
#include "oracle_2d.h"

#include <algorithm>
#include <cmath>
#include <deque>
#include <functional>

namespace oracle {

// oracle-only instrumentation; thread-local so that one matcher can be shared by
// the CPU-baseline worker threads like the reference's pool threads share theirs.
static thread_local MatchStats* stats_ = nullptr;

ProbabilityGrid::ProbabilityGrid(const MapLimits& l, float min_cost, float max_cost)
    : limits(l),
      min_correspondence_cost(min_cost),
      max_correspondence_cost(max_cost),
      cells(static_cast<size_t>(l.cell_limits.num_x_cells) * l.cell_limits.num_y_cells,
            kUnknownCorrespondenceValue),
      // grid_2d.cc:66-71: GetConversionTable(max_cost, min_cost, max_cost)
      value_to_cost_table(PrecomputeValueToBoundedFloat(0, max_cost, min_cost, max_cost)) {}

// ---------------------------------------------------------------------------
// correlative_scan_matcher_2d.cc:27-55
SearchParameters::SearchParameters(const double linear_search_window,
                                   const double angular_search_window,
                                   const PointCloud& point_cloud,
                                   const double resolution)
    : resolution(resolution) {
  float max_scan_range = 3.f * resolution;  // :34 (float = float * double -> float)
  for (const Vec3f& point : point_cloud) {
    // position.head<2>().norm(): sqrt(x*x + y*y) in float  (:36)
    const float range = std::sqrt(point.x * point.x + point.y * point.y);
    max_scan_range = std::max(range, max_scan_range);
  }
  const double kSafetyMargin = 1. - 1e-3;
  angular_perturbation_step_size =
      kSafetyMargin *
      // Pow2(max_scan_range) is Pow2<float>: squared in float, then promoted (:42)
      std::acos(1. - Pow2(resolution) / (2. * Pow2(max_scan_range)));
  num_angular_perturbations =
      static_cast<int>(std::ceil(angular_search_window / angular_perturbation_step_size));
  num_scans = 2 * num_angular_perturbations + 1;
  const int num_linear_perturbations =
      static_cast<int>(std::ceil(linear_search_window / resolution));
  linear_bounds.reserve(num_scans);
  for (int i = 0; i != num_scans; ++i) {
    linear_bounds.push_back(LinearBounds{-num_linear_perturbations, num_linear_perturbations,
                                         -num_linear_perturbations, num_linear_perturbations});
  }
}

// correlative_scan_matcher_2d.cc:57-71 ("for testing" ctor)
SearchParameters::SearchParameters(const int num_linear_perturbations,
                                   const int num_angular_perturbations,
                                   const double angular_perturbation_step_size,
                                   const double resolution)
    : num_angular_perturbations(num_angular_perturbations),
      angular_perturbation_step_size(angular_perturbation_step_size),
      resolution(resolution),
      num_scans(2 * num_angular_perturbations + 1) {
  linear_bounds.reserve(num_scans);
  for (int i = 0; i != num_scans; ++i) {
    linear_bounds.push_back(LinearBounds{-num_linear_perturbations, num_linear_perturbations,
                                         -num_linear_perturbations, num_linear_perturbations});
  }
}

// correlative_scan_matcher_2d.cc:73-91
void SearchParameters::ShrinkToFit(const std::vector<DiscreteScan2D>& scans,
                                   const CellLimits& cell_limits) {
  for (int i = 0; i != num_scans; ++i) {
    int min_bx = 0, min_by = 0, max_bx = 0, max_by = 0;
    for (const Array2i& xy : scans[i]) {
      min_bx = std::min(min_bx, -xy.x);
      min_by = std::min(min_by, -xy.y);
      max_bx = std::max(max_bx, cell_limits.num_x_cells - 1 - xy.x);
      max_by = std::max(max_by, cell_limits.num_y_cells - 1 - xy.y);
    }
    linear_bounds[i].min_x = std::max(linear_bounds[i].min_x, min_bx);
    linear_bounds[i].max_x = std::min(linear_bounds[i].max_x, max_bx);
    linear_bounds[i].min_y = std::max(linear_bounds[i].min_y, min_by);
    linear_bounds[i].max_y = std::min(linear_bounds[i].max_y, max_by);
  }
}

// correlative_scan_matcher_2d.cc:93-109
std::vector<PointCloud> GenerateRotatedScans(const PointCloud& point_cloud,
                                             const SearchParameters& sp) {
  std::vector<PointCloud> rotated_scans;
  rotated_scans.reserve(sp.num_scans);
  double delta_theta = -sp.num_angular_perturbations * sp.angular_perturbation_step_size;
  for (int scan_index = 0; scan_index < sp.num_scans;
       ++scan_index, delta_theta += sp.angular_perturbation_step_size) {
    // AngleAxisf(delta_theta, UnitZ): double -> float cast of the angle (:105)
    rotated_scans.push_back(
        TransformPointCloudRotZ(point_cloud, static_cast<float>(delta_theta)));
  }
  return rotated_scans;
}

// correlative_scan_matcher_2d.cc:111-127
std::vector<DiscreteScan2D> DiscretizeScans(const MapLimits& map_limits,
                                            const std::vector<PointCloud>& scans,
                                            const float tx, const float ty) {
  std::vector<DiscreteScan2D> discrete_scans;
  discrete_scans.reserve(scans.size());
  for (const PointCloud& scan : scans) {
    discrete_scans.emplace_back();
    discrete_scans.back().reserve(scan.size());
    for (const Vec3f& point : scan) {
      // Affine2f(Translation2f) * v == I*v + t; 1*x + 0*y is exact (:120-121)
      const float px = (1.f * point.x + 0.f * point.y) + tx;
      const float py = (0.f * point.x + 1.f * point.y) + ty;
      discrete_scans.back().push_back(map_limits.GetCellIndex(px, py));
    }
  }
  return discrete_scans;
}

// ---------------------------------------------------------------------------
namespace {

// fast_correlative_scan_matcher_2d.cc:41-74 (SlidingWindowMaximum) used the way
// the ctor :108-160 uses it: out[k] = max(in[max(0,k-w+1) .. min(n-1,k)]),
// k in [0, n+w-1).  Same deque discipline (AddValue / RemoveValue / GetMaximum).
class SlidingWindowMaximum {
 public:
  void AddValue(const float value) {
    while (!maxima_.empty() && value > maxima_.back()) maxima_.pop_back();
    maxima_.push_back(value);
  }
  void RemoveValue(const float value) {
    if (value == maxima_.front()) maxima_.pop_front();
  }
  float GetMaximum() const { return maxima_.front(); }
 private:
  std::deque<float> maxima_;
};

template <typename In, typename Out>
void ClippedWindowMax(const int n, const int w, In in, Out out) {
  SlidingWindowMaximum window;
  window.AddValue(in(0));
  for (int s = -w + 1; s != 0; ++s) {          // window start s < 0   (:113-118)
    out(s + w - 1, window.GetMaximum());
    if (s + w < n) window.AddValue(in(s + w));
  }
  for (int s = 0; s < n - w; ++s) {            // fully inside          (:119-125)
    out(s + w - 1, window.GetMaximum());
    window.RemoveValue(in(s));
    window.AddValue(in(s + w));
  }
  for (int s = std::max(n - w, 0); s != n; ++s) {  // running off the end (:126-131)
    out(s + w - 1, window.GetMaximum());
    window.RemoveValue(in(s));
  }
}

}  // namespace

// fast_correlative_scan_matcher_2d.cc:91-161
PrecomputationGrid2D::PrecomputationGrid2D(const ProbabilityGrid& grid,
                                           const CellLimits& limits, const int width,
                                           std::vector<float>* reusable_intermediate_grid)
    : offset_{-width + 1, -width + 1},
      wide_limits_{limits.num_x_cells + width - 1, limits.num_y_cells + width - 1},
      min_score_(1.f - grid.max_correspondence_cost),
      max_score_(1.f - grid.min_correspondence_cost),
      cells_(static_cast<size_t>(wide_limits_.num_x_cells) * wide_limits_.num_y_cells) {
  const int stride = wide_limits_.num_x_cells;
  std::vector<float>& intermediate = *reusable_intermediate_grid;
  intermediate.resize(static_cast<size_t>(wide_limits_.num_x_cells) * limits.num_y_cells);
  for (int y = 0; y != limits.num_y_cells; ++y) {
    ClippedWindowMax(
        limits.num_x_cells, width,
        [&](int x) { return 1.f - std::abs(grid.GetCorrespondenceCost(Array2i{x, y})); },
        [&](int k, float v) { intermediate[k + y * stride] = v; });
  }
  for (int x = 0; x != wide_limits_.num_x_cells; ++x) {
    ClippedWindowMax(
        limits.num_y_cells, width,
        [&](int y) { return intermediate[x + y * stride]; },
        [&](int k, float v) { cells_[x + k * stride] = ComputeCellValue(v); });
  }
}

// fast_correlative_scan_matcher_2d.cc:163-169
uint8_t PrecomputationGrid2D::ComputeCellValue(const float probability) const {
  const int cell_value =
      RoundToInt((probability - min_score_) * (255.f / (max_score_ - min_score_)));
  return static_cast<uint8_t>(cell_value);
}

// fast_correlative_scan_matcher_2d.cc:171-186
PrecomputationGridStack2D::PrecomputationGridStack2D(const ProbabilityGrid& grid,
                                                     const FastOptions2D& options) {
  const int max_width = 1 << (options.branch_and_bound_depth - 1);
  grids_.reserve(options.branch_and_bound_depth);
  std::vector<float> reusable_intermediate_grid;
  const CellLimits limits = grid.limits.cell_limits;
  reusable_intermediate_grid.reserve(
      static_cast<size_t>(limits.num_x_cells + max_width - 1) * limits.num_y_cells);
  for (int i = 0; i != options.branch_and_bound_depth; ++i) {
    const int width = 1 << i;
    grids_.emplace_back(grid, limits, width, &reusable_intermediate_grid);
  }
}

// fast_correlative_scan_matcher_2d.cc:188-194
FastCorrelativeScanMatcher2D::FastCorrelativeScanMatcher2D(const ProbabilityGrid& grid,
                                                           const FastOptions2D& options)
    : options_(options),
      limits_(grid.limits),
      stack_(new PrecomputationGridStack2D(grid, options)) {}

// :198-208
bool FastCorrelativeScanMatcher2D::Match(const Rigid2d& initial_pose_estimate,
                                         const PointCloud& point_cloud,
                                         const float min_score, float* score,
                                         Rigid2d* pose_estimate, MatchStats* stats) const {
  const SearchParameters search_parameters(options_.linear_search_window,
                                           options_.angular_search_window, point_cloud,
                                           limits_.resolution);
  return MatchWithSearchParameters(search_parameters, initial_pose_estimate, point_cloud,
                                   min_score, score, pose_estimate, stats);
}

// :210-225
bool FastCorrelativeScanMatcher2D::MatchFullSubmap(const PointCloud& point_cloud,
                                                   float min_score, float* score,
                                                   Rigid2d* pose_estimate,
                                                   MatchStats* stats) const {
  const SearchParameters search_parameters(1e6 * limits_.resolution, M_PI, point_cloud,
                                           limits_.resolution);
  // center = max - 0.5 * resolution * (num_y_cells, num_x_cells)   (:219-222)
  const Rigid2d center{
      limits_.max_x - 0.5 * limits_.resolution * limits_.cell_limits.num_y_cells,
      limits_.max_y - 0.5 * limits_.resolution * limits_.cell_limits.num_x_cells, 0.};
  return MatchWithSearchParameters(search_parameters, center, point_cloud, min_score,
                                   score, pose_estimate, stats);
}

// :227-262
bool FastCorrelativeScanMatcher2D::MatchWithSearchParameters(
    SearchParameters search_parameters, const Rigid2d& initial_pose_estimate,
    const PointCloud& point_cloud, float min_score, float* score,
    Rigid2d* pose_estimate, MatchStats* stats) const {
  stats_ = stats;
  const double initial_rotation = initial_pose_estimate.theta;
  // Rotation2Dd::cast<float>().angle() is a plain double->float cast (:239)
  const PointCloud rotated_point_cloud =
      TransformPointCloudRotZ(point_cloud, static_cast<float>(initial_rotation));
  const std::vector<PointCloud> rotated_scans =
      GenerateRotatedScans(rotated_point_cloud, search_parameters);
  // Translation2f(double, double): double -> float casts (:242-244)
  const std::vector<DiscreteScan2D> discrete_scans =
      DiscretizeScans(limits_, rotated_scans, static_cast<float>(initial_pose_estimate.x),
                      static_cast<float>(initial_pose_estimate.y));
  search_parameters.ShrinkToFit(discrete_scans, limits_.cell_limits);

  const std::vector<Candidate2D> lowest_resolution_candidates =
      ComputeLowestResolutionCandidates(discrete_scans, search_parameters);
  if (stats) {
    stats->lowest_resolution_candidates = lowest_resolution_candidates.size();
    stats->num_scans = search_parameters.num_scans;
  }
  const Candidate2D best_candidate =
      BranchAndBound(discrete_scans, search_parameters, lowest_resolution_candidates,
                     stack_->max_depth(), min_score);
  stats_ = nullptr;
  if (best_candidate.score > min_score) {
    *score = best_candidate.score;
    // Rotation2Dd * Rotation2Dd adds the angles (:258)
    *pose_estimate = Rigid2d{initial_pose_estimate.x + best_candidate.x,
                             initial_pose_estimate.y + best_candidate.y,
                             initial_rotation + best_candidate.orientation};
    if (stats) {
      stats->best_scan_index = best_candidate.scan_index;
      stats->best_x_offset = best_candidate.x_index_offset;
      stats->best_y_offset = best_candidate.y_index_offset;
    }
    return true;
  }
  return false;
}

// :264-274
std::vector<Candidate2D> FastCorrelativeScanMatcher2D::ComputeLowestResolutionCandidates(
    const std::vector<DiscreteScan2D>& discrete_scans,
    const SearchParameters& search_parameters) const {
  std::vector<Candidate2D> lowest_resolution_candidates =
      GenerateLowestResolutionCandidates(search_parameters);
  ScoreCandidates(stack_->Get(stack_->max_depth()), discrete_scans, search_parameters,
                  &lowest_resolution_candidates);
  return lowest_resolution_candidates;
}

// :276-312
std::vector<Candidate2D> FastCorrelativeScanMatcher2D::GenerateLowestResolutionCandidates(
    const SearchParameters& sp) const {
  const int linear_step_size = 1 << stack_->max_depth();
  int num_candidates = 0;
  for (int scan_index = 0; scan_index != sp.num_scans; ++scan_index) {
    const SearchParameters::LinearBounds& b = sp.linear_bounds[scan_index];
    const int nx = (b.max_x - b.min_x + linear_step_size) / linear_step_size;
    const int ny = (b.max_y - b.min_y + linear_step_size) / linear_step_size;
    num_candidates += nx * ny;
  }
  std::vector<Candidate2D> candidates;
  candidates.reserve(num_candidates);
  for (int scan_index = 0; scan_index != sp.num_scans; ++scan_index) {
    const SearchParameters::LinearBounds& b = sp.linear_bounds[scan_index];
    for (int xo = b.min_x; xo <= b.max_x; xo += linear_step_size) {
      for (int yo = b.min_y; yo <= b.max_y; yo += linear_step_size) {
        candidates.emplace_back(scan_index, xo, yo, sp);
      }
    }
  }
  return candidates;
}

// :314-333
void FastCorrelativeScanMatcher2D::ScoreCandidates(
    const PrecomputationGrid2D& precomputation_grid,
    const std::vector<DiscreteScan2D>& discrete_scans,
    const SearchParameters& /*search_parameters*/,
    std::vector<Candidate2D>* const candidates, bool sort) const {
  for (Candidate2D& candidate : *candidates) {
    int sum = 0;
    for (const Array2i& xy_index : discrete_scans[candidate.scan_index]) {
      const Array2i proposed{xy_index.x + candidate.x_index_offset,
                             xy_index.y + candidate.y_index_offset};
      sum += precomputation_grid.GetValue(proposed);
    }
    candidate.score = precomputation_grid.ToScore(
        sum / static_cast<float>(discrete_scans[candidate.scan_index].size()));
  }
  if (stats_) stats_->candidates_scored += candidates->size();
  if (sort) std::sort(candidates->begin(), candidates->end(), std::greater<Candidate2D>());
}

// :335-378
Candidate2D FastCorrelativeScanMatcher2D::BranchAndBound(
    const std::vector<DiscreteScan2D>& discrete_scans,
    const SearchParameters& search_parameters, const std::vector<Candidate2D>& candidates,
    const int candidate_depth, float min_score) const {
  if (candidate_depth == 0) {
    return *candidates.begin();
  }
  Candidate2D best_high_resolution_candidate(0, 0, 0, search_parameters);
  best_high_resolution_candidate.score = min_score;
  for (const Candidate2D& candidate : candidates) {
    if (candidate.score <= min_score) break;
    std::vector<Candidate2D> higher_resolution_candidates;
    const int half_width = 1 << (candidate_depth - 1);
    for (int x_offset : {0, half_width}) {
      if (candidate.x_index_offset + x_offset >
          search_parameters.linear_bounds[candidate.scan_index].max_x) {
        break;
      }
      for (int y_offset : {0, half_width}) {
        if (candidate.y_index_offset + y_offset >
            search_parameters.linear_bounds[candidate.scan_index].max_y) {
          break;
        }
        higher_resolution_candidates.emplace_back(candidate.scan_index,
                                                  candidate.x_index_offset + x_offset,
                                                  candidate.y_index_offset + y_offset,
                                                  search_parameters);
      }
    }
    if (stats_) stats_->nodes_expanded += 1;
    ScoreCandidates(stack_->Get(candidate_depth - 1), discrete_scans, search_parameters,
                    &higher_resolution_candidates);
    best_high_resolution_candidate =
        std::max(best_high_resolution_candidate,
                 BranchAndBound(discrete_scans, search_parameters,
                                higher_resolution_candidates, candidate_depth - 1,
                                best_high_resolution_candidate.score));
  }
  return best_high_resolution_candidate;
}

// ---------------------------------------------------------------------------
// real_time_correlative_scan_matcher_2d.cc:83-115
std::vector<Candidate2D> RealTimeCorrelativeScanMatcher2D::GenerateExhaustiveSearchCandidates(
    const SearchParameters& sp) const {
  int num_candidates = 0;
  for (int s = 0; s != sp.num_scans; ++s) {
    const SearchParameters::LinearBounds& b = sp.linear_bounds[s];
    num_candidates += (b.max_x - b.min_x + 1) * (b.max_y - b.min_y + 1);
  }
  std::vector<Candidate2D> candidates;
  candidates.reserve(num_candidates);
  for (int s = 0; s != sp.num_scans; ++s) {
    const SearchParameters::LinearBounds& b = sp.linear_bounds[s];
    for (int xo = b.min_x; xo <= b.max_x; ++xo) {
      for (int yo = b.min_y; yo <= b.max_y; ++yo) {
        candidates.emplace_back(s, xo, yo, sp);
      }
    }
  }
  return candidates;
}

// real_time_correlative_scan_matcher_2d.cc:117-149
double RealTimeCorrelativeScanMatcher2D::Match(const Rigid2d& initial_pose_estimate,
                                               const PointCloud& point_cloud,
                                               const ProbabilityGrid& grid,
                                               Rigid2d* pose_estimate,
                                               MatchStats* stats,
                                               std::vector<float>* scores) const {
  const double initial_rotation = initial_pose_estimate.theta;
  const PointCloud rotated_point_cloud =
      TransformPointCloudRotZ(point_cloud, static_cast<float>(initial_rotation));
  const SearchParameters search_parameters(options_.linear_search_window,
                                           options_.angular_search_window,
                                           rotated_point_cloud, grid.limits.resolution);
  const std::vector<PointCloud> rotated_scans =
      GenerateRotatedScans(rotated_point_cloud, search_parameters);
  const std::vector<DiscreteScan2D> discrete_scans =
      DiscretizeScans(grid.limits, rotated_scans,
                      static_cast<float>(initial_pose_estimate.x),
                      static_cast<float>(initial_pose_estimate.y));
  std::vector<Candidate2D> candidates = GenerateExhaustiveSearchCandidates(search_parameters);
  ScoreCandidates(grid, discrete_scans, search_parameters, &candidates);
  if (scores)
    for (const Candidate2D& c : candidates) scores->push_back(c.score);
  const Candidate2D& best_candidate =
      *std::max_element(candidates.begin(), candidates.end());
  *pose_estimate = Rigid2d{initial_pose_estimate.x + best_candidate.x,
                           initial_pose_estimate.y + best_candidate.y,
                           initial_rotation + best_candidate.orientation};
  if (stats) {
    stats->candidates_scored += candidates.size();
    stats->num_scans = search_parameters.num_scans;
    stats->best_scan_index = best_candidate.scan_index;
    stats->best_x_offset = best_candidate.x_index_offset;
    stats->best_y_offset = best_candidate.y_index_offset;
  }
  return best_candidate.score;
}

// real_time_correlative_scan_matcher_2d.cc:151-176 (+ :61-75 probability variant)
void RealTimeCorrelativeScanMatcher2D::ScoreCandidates(
    const ProbabilityGrid& grid, const std::vector<DiscreteScan2D>& discrete_scans,
    const SearchParameters& /*search_parameters*/,
    std::vector<Candidate2D>* const candidates) const {
  for (Candidate2D& candidate : *candidates) {
    float candidate_score = 0.f;
    const DiscreteScan2D& discrete_scan = discrete_scans[candidate.scan_index];
    for (const Array2i& xy_index : discrete_scan) {
      const Array2i proposed{xy_index.x + candidate.x_index_offset,
                             xy_index.y + candidate.y_index_offset};
      candidate_score += grid.GetProbability(proposed);
    }
    candidate_score /= static_cast<float>(discrete_scan.size());
    candidate.score = candidate_score;
    // float *= double: promoted to double, product rounded back to float (:170-174)
    candidate.score *= std::exp(-Pow2(std::hypot(candidate.x, candidate.y) *
                                          options_.translation_delta_cost_weight +
                                      std::abs(candidate.orientation) *
                                          options_.rotation_delta_cost_weight));
  }
}

// ---- TSDF variant ---------------------------------------------------------------
TSDF2D::TSDF2D(const MapLimits& l, float truncation, float max_w)
    : limits(l),
      truncation_distance(truncation),
      max_weight(max_w),
      tsd_cells(static_cast<size_t>(l.cell_limits.num_x_cells) * l.cell_limits.num_y_cells, 0),
      weight_cells(tsd_cells.size(), 0),
      // tsd_value_converter.cc:31-34: GetConversionTable(min_tsd, min_tsd, max_tsd) and
      // GetConversionTable(min_weight, min_weight, max_weight)
      value_to_tsd(PrecomputeValueToBoundedFloat(0, -truncation, -truncation, truncation)),
      value_to_weight(PrecomputeValueToBoundedFloat(0, 0.f, 0.f, max_w)) {}

// real_time_correlative_scan_matcher_2d.cc:38-59 + :170-174
void RealTimeCorrelativeScanMatcher2D::ScoreCandidates(
    const TSDF2D& tsdf, const std::vector<DiscreteScan2D>& discrete_scans,
    const SearchParameters& /*search_parameters*/,
    std::vector<Candidate2D>* const candidates) const {
  for (Candidate2D& candidate : *candidates) {
    float candidate_score = 0.f;
    float summed_weight = 0.f;
    for (const Array2i& xy_index : discrete_scans[candidate.scan_index]) {
      const Array2i proposed{xy_index.x + candidate.x_index_offset,
                             xy_index.y + candidate.y_index_offset};
      const std::pair<float, float> tsd_and_weight = tsdf.GetTSDAndWeight(proposed);
      const float normalized_tsd_score =
          (tsdf.GetMaxCorrespondenceCost() - std::abs(tsd_and_weight.first)) /
          tsdf.GetMaxCorrespondenceCost();
      const float weight = tsd_and_weight.second;
      candidate_score += normalized_tsd_score * weight;
      summed_weight += weight;
    }
    if (summed_weight == 0.f) {
      candidate_score = 0.f;
    } else {
      candidate_score /= summed_weight;
    }
    candidate.score = candidate_score;
    candidate.score *= std::exp(-Pow2(std::hypot(candidate.x, candidate.y) *
                                          options_.translation_delta_cost_weight +
                                      std::abs(candidate.orientation) *
                                          options_.rotation_delta_cost_weight));
  }
}

double RealTimeCorrelativeScanMatcher2D::Match(const Rigid2d& initial_pose_estimate,
                                               const PointCloud& point_cloud, const TSDF2D& grid,
                                               Rigid2d* pose_estimate, MatchStats* stats,
                                               std::vector<float>* scores) const {
  const double initial_rotation = initial_pose_estimate.theta;
  const PointCloud rotated_point_cloud =
      TransformPointCloudRotZ(point_cloud, static_cast<float>(initial_rotation));
  const SearchParameters search_parameters(options_.linear_search_window,
                                           options_.angular_search_window,
                                           rotated_point_cloud, grid.limits.resolution);
  const std::vector<PointCloud> rotated_scans =
      GenerateRotatedScans(rotated_point_cloud, search_parameters);
  const std::vector<DiscreteScan2D> discrete_scans =
      DiscretizeScans(grid.limits, rotated_scans, static_cast<float>(initial_pose_estimate.x),
                      static_cast<float>(initial_pose_estimate.y));
  std::vector<Candidate2D> candidates = GenerateExhaustiveSearchCandidates(search_parameters);
  ScoreCandidates(grid, discrete_scans, search_parameters, &candidates);
  if (scores)
    for (const Candidate2D& c : candidates) scores->push_back(c.score);
  const Candidate2D& best_candidate = *std::max_element(candidates.begin(), candidates.end());
  *pose_estimate = Rigid2d{initial_pose_estimate.x + best_candidate.x,
                           initial_pose_estimate.y + best_candidate.y,
                           initial_rotation + best_candidate.orientation};
  if (stats) {
    stats->candidates_scored += candidates.size();
    stats->num_scans = search_parameters.num_scans;
    stats->best_scan_index = best_candidate.scan_index;
    stats->best_x_offset = best_candidate.x_index_offset;
    stats->best_y_offset = best_candidate.y_index_offset;
  }
  return best_candidate.score;
}

}  // namespace oracle
