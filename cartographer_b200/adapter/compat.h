// Layout-compatible stand-ins for the handful of Cartographer types that appear
// in the signatures of the scan matchers.  Used ONLY when the real headers are
// not on the include path (this image has no Eigen/glog/abseil/protobuf, so the
// reference cannot be compiled here); inside a Cartographer checkout the
// adapter includes the real headers instead (see the __has_include switch in
// scan_matchers_b200.h and INTEGRATION.md).
//
// Only the members the adapter touches are provided.
#ifndef CSM_ADAPTER_COMPAT_H_
#define CSM_ADAPTER_COMPAT_H_

#include <cmath>
#include <cstdint>
#include <functional>
#include <memory>
#include <utility>
#include <vector>

namespace cartographer {

namespace transform {
// transform/rigid_transform.h:34-103 (Rigid2<double>): translation + Rotation2D angle.
class Rigid2d {
 public:
  struct Vector {
    double x_, y_;
    double x() const { return x_; }
    double y() const { return y_; }
    double norm() const { return std::sqrt(x_ * x_ + y_ * y_); }
  };
  struct Rotation2D { double angle_; double angle() const { return angle_; } };
  Rigid2d() : t_{0., 0.}, r_{0.} {}
  Rigid2d(const Vector& t, double rotation) : t_(t), r_{rotation} {}
  static Rigid2d Identity() { return Rigid2d(); }
  const Vector& translation() const { return t_; }
  Rotation2D rotation() const { return r_; }
  // rigid_transform.h:76-80 and :93-99
  Rigid2d inverse() const {
    const double c = std::cos(-r_.angle_), s = std::sin(-r_.angle_);
    return Rigid2d({-(c * t_.x_ - s * t_.y_), -(s * t_.x_ + c * t_.y_)}, -r_.angle_);
  }
  friend Rigid2d operator*(const Rigid2d& a, const Rigid2d& b) {
    const double c = std::cos(a.r_.angle_), s = std::sin(a.r_.angle_);
    return Rigid2d({c * b.t_.x_ - s * b.t_.y_ + a.t_.x_, s * b.t_.x_ + c * b.t_.y_ + a.t_.y_},
                   a.r_.angle_ + b.r_.angle_);
  }
 private:
  Vector t_;
  Rotation2D r_;
};
}  // namespace transform

namespace sensor {
// sensor/rangefinder_point.h:31-33 and sensor/point_cloud.h:33-92.
struct RangefinderPoint { struct { float v[3]; float x() const { return v[0]; } float y() const { return v[1]; } float z() const { return v[2]; } } position; };
class PointCloud {
 public:
  PointCloud() = default;
  PointCloud(std::vector<RangefinderPoint> points, std::vector<float> intensities)
      : points_(std::move(points)), intensities_(std::move(intensities)) {}
  void push_back(const RangefinderPoint& p) { points_.push_back(p); }
  size_t size() const { return points_.size(); }
  const std::vector<RangefinderPoint>& points() const { return points_; }
  const std::vector<float>& intensities() const { return intensities_; }
 private:
  std::vector<RangefinderPoint> points_;
  std::vector<float> intensities_;
};
// sensor/range_data.h:28-35 (origin is an Eigen::Vector3f there).
struct RangeData {
  struct { float v[3]; float x() const { return v[0]; } float y() const { return v[1]; } float z() const { return v[2]; } } origin;
  PointCloud returns;
  PointCloud misses;
};
}  // namespace sensor

namespace mapping {
namespace proto {
// mapping/proto/range_data_inserter_options_3d.proto
class RangeDataInserterOptions3D {
 public:
  double hit_probability() const { return hit_; }
  double miss_probability() const { return miss_; }
  int num_free_space_voxels() const { return nfsv_; }
  float intensity_threshold() const { return threshold_; }
  void set_hit_probability(double v) { hit_ = v; }
  void set_miss_probability(double v) { miss_ = v; }
  void set_num_free_space_voxels(int v) { nfsv_ = v; }
  void set_intensity_threshold(float v) { threshold_ = v; }
 private:
  double hit_ = 0., miss_ = 0.;
  int nfsv_ = 0;
  float threshold_ = 0.f;
};
// mapping/proto/probability_grid_range_data_inserter_options_2d.proto
class ProbabilityGridRangeDataInserterOptions2D {
 public:
  double hit_probability() const { return hit_; }
  double miss_probability() const { return miss_; }
  bool insert_free_space() const { return insert_free_space_; }
  void set_hit_probability(double v) { hit_ = v; }
  void set_miss_probability(double v) { miss_ = v; }
  void set_insert_free_space(bool v) { insert_free_space_ = v; }
 private:
  double hit_ = 0., miss_ = 0.;
  bool insert_free_space_ = true;
};
// mapping/proto/normal_estimation_options_2d.proto
class NormalEstimationOptions2D {
 public:
  int32_t num_normal_samples() const { return num_normal_samples_; }
  double sample_radius() const { return sample_radius_; }
  void set_num_normal_samples(int32_t v) { num_normal_samples_ = v; }
  void set_sample_radius(double v) { sample_radius_ = v; }
 private:
  int32_t num_normal_samples_ = 0;
  double sample_radius_ = 0.;
};
// mapping/proto/tsdf_range_data_inserter_options_2d.proto
class TSDFRangeDataInserterOptions2D {
 public:
  double truncation_distance() const { return truncation_distance_; }
  double maximum_weight() const { return maximum_weight_; }
  bool update_free_space() const { return update_free_space_; }
  const NormalEstimationOptions2D& normal_estimation_options() const { return normal_; }
  NormalEstimationOptions2D* mutable_normal_estimation_options() { return &normal_; }
  bool project_sdf_distance_to_scan_normal() const { return project_; }
  int32_t update_weight_range_exponent() const { return range_exponent_; }
  double update_weight_angle_scan_normal_to_ray_kernel_bandwidth() const { return angle_bw_; }
  double update_weight_distance_cell_to_hit_kernel_bandwidth() const { return distance_bw_; }
  void set_truncation_distance(double v) { truncation_distance_ = v; }
  void set_maximum_weight(double v) { maximum_weight_ = v; }
  void set_update_free_space(bool v) { update_free_space_ = v; }
  void set_project_sdf_distance_to_scan_normal(bool v) { project_ = v; }
  void set_update_weight_range_exponent(int32_t v) { range_exponent_ = v; }
  void set_update_weight_angle_scan_normal_to_ray_kernel_bandwidth(double v) { angle_bw_ = v; }
  void set_update_weight_distance_cell_to_hit_kernel_bandwidth(double v) { distance_bw_ = v; }
 private:
  double truncation_distance_ = 0., maximum_weight_ = 0.;
  bool update_free_space_ = false;
  NormalEstimationOptions2D normal_;
  bool project_ = false;
  int32_t range_exponent_ = 0;
  double angle_bw_ = 0., distance_bw_ = 0.;
};
}  // namespace proto
}  // namespace mapping

namespace transform {
// transform/rigid_transform.h:116-196 (Rigid3<double>) and Eigen::Quaterniond as used
// in the 3D matcher's signatures.
struct Quaterniond {
  double w_, x_, y_, z_;
  double w() const { return w_; } double x() const { return x_; }
  double y() const { return y_; } double z() const { return z_; }
};
class Rigid3d {
 public:
  struct Vector { double v[3]; double x() const { return v[0]; } double y() const { return v[1]; } double z() const { return v[2]; } };
  Rigid3d() : t_{{0., 0., 0.}}, q_{1., 0., 0., 0.} {}
  Rigid3d(const Vector& t, const Quaterniond& q) : t_(t), q_(q) {}
  const Vector& translation() const { return t_; }
  const Quaterniond& rotation() const { return q_; }
 private:
  Vector t_;
  Quaterniond q_;
};
}  // namespace transform

namespace mapping {
// mapping/3d/hybrid_grid.h:468-526: what the adapter needs is iteration over the
// non-zero voxels (HybridGrid::Iterator / begin()-end(), :413-460) and resolution().
class HybridGrid {
 public:
  struct Voxel { int x, y, z; uint16_t value; };
  explicit HybridGrid(float resolution) : resolution_(resolution) {}
  float resolution() const { return resolution_; }
  int grid_size() const { return grid_size_; }
  void Set(int x, int y, int z, uint16_t value) {
    voxels_.push_back(Voxel{x, y, z, value});
    while (x < -(grid_size_ >> 1) || x >= (grid_size_ >> 1) || y < -(grid_size_ >> 1) ||
           y >= (grid_size_ >> 1) || z < -(grid_size_ >> 1) || z >= (grid_size_ >> 1))
      grid_size_ <<= 1;
  }
  const std::vector<Voxel>& voxels() const { return voxels_; }
 private:
  float resolution_;
  int grid_size_ = 128;
  std::vector<Voxel> voxels_;
};
// mapping/3d/hybrid_grid.h:547-570: AddIntensity and iteration over the voxels'
// AverageIntensityData {sum, count}.
class IntensityHybridGrid {
 public:
  struct Voxel { int x, y, z; float sum; int count; };
  explicit IntensityHybridGrid(float resolution) : resolution_(resolution) {}
  float resolution() const { return resolution_; }
  void AddIntensity(int x, int y, int z, float intensity) {
    for (Voxel& v : voxels_)
      if (v.x == x && v.y == y && v.z == z) {
        v.count += 1;
        v.sum += intensity;
        return;
      }
    voxels_.push_back(Voxel{x, y, z, intensity, 1});
  }
  const std::vector<Voxel>& voxels() const { return voxels_; }
 private:
  float resolution_;
  std::vector<Voxel> voxels_;
};
// mapping/trajectory_node.h:45-63 (the fields the 3D matcher reads).
struct TrajectoryNodeData {
  transform::Quaterniond gravity_alignment{1., 0., 0., 0.};
  sensor::PointCloud filtered_gravity_aligned_point_cloud;   // 2D
  sensor::PointCloud high_resolution_point_cloud;
  sensor::PointCloud low_resolution_point_cloud;
  std::vector<float> rotational_scan_matcher_histogram;   // Eigen::VectorXf
};
}  // namespace mapping

namespace mapping {
// mapping/2d/xy_index.h:34-45, mapping/2d/map_limits.h:40-95.
struct CellLimits { int num_x_cells = 0; int num_y_cells = 0; };
class MapLimits {
 public:
  struct Vector2d { double x_, y_; double x() const { return x_; } double y() const { return y_; } };
  MapLimits(double resolution, double max_x, double max_y, const CellLimits& c)
      : resolution_(resolution), max_{max_x, max_y}, cell_limits_(c) {}
  double resolution() const { return resolution_; }
  const Vector2d& max() const { return max_; }
  const CellLimits& cell_limits() const { return cell_limits_; }
 private:
  double resolution_;
  Vector2d max_;
  CellLimits cell_limits_;
};
// mapping/2d/grid_2d.h:37-141 — the read-only accessors the matcher ctor uses.
enum class GridType { PROBABILITY_GRID, TSDF };  // mapping/2d/grid_2d.h:35
class Grid2D {
 public:
  Grid2D(const MapLimits& limits, float min_cost, float max_cost, std::vector<uint16_t> cells)
      : limits_(limits), min_(min_cost), max_(max_cost), cells_(std::move(cells)) {}
  virtual ~Grid2D() {}
  virtual GridType GetGridType() const { return GridType::PROBABILITY_GRID; }
  const MapLimits& limits() const { return limits_; }
  float GetMinCorrespondenceCost() const { return min_; }
  float GetMaxCorrespondenceCost() const { return max_; }
  // protected in the reference (grid_2d.h:98-100); the real adapter is a friend or
  // uses ToProto().cells() — see INTEGRATION.md.
  const std::vector<uint16_t>& correspondence_cost_cells() const { return cells_; }
 private:
  MapLimits limits_;
  float min_, max_;
  std::vector<uint16_t> cells_;
};

// mapping/2d/tsdf_2d.h:32-80 — what the real-time matcher's TSDF branch reads: the TSD
// cells (Grid2D::correspondence_cost_cells), the weight cells and the TSDValueConverter
// parameters (mapping/internal/2d/tsd_value_converter.h:32-43).
class TSDF2D : public Grid2D {
 public:
  TSDF2D(const MapLimits& limits, float truncation_distance, float max_weight,
         std::vector<uint16_t> tsd_cells, std::vector<uint16_t> weight_cells)
      : Grid2D(limits, -truncation_distance, truncation_distance, std::move(tsd_cells)),
        truncation_distance_(truncation_distance), max_weight_(max_weight),
        weight_cells_(std::move(weight_cells)) {}
  // the all-unknown TSDF2D ActiveSubmaps2D::CreateGrid makes (tsdf_2d.cc:24-33)
  TSDF2D(const MapLimits& limits, float truncation_distance, float max_weight)
      : TSDF2D(limits, truncation_distance, max_weight, Unknown(limits), Unknown(limits)) {}
  GridType GetGridType() const override { return GridType::TSDF; }
  float truncation_distance() const { return truncation_distance_; }
  float max_weight() const { return max_weight_; }
  const std::vector<uint16_t>& weight_cells() const { return weight_cells_; }
 private:
  static std::vector<uint16_t> Unknown(const MapLimits& l) {
    return std::vector<uint16_t>(
        static_cast<size_t>(l.cell_limits().num_x_cells) * l.cell_limits().num_y_cells, 0);
  }
  float truncation_distance_, max_weight_;
  std::vector<uint16_t> weight_cells_;
};

namespace scan_matching {
// internal/2d/scan_matching/correlative_scan_matcher_2d.h:32-103 — the types in the
// signature of the public RealTimeCorrelativeScanMatcher2D::ScoreCandidates.
struct Array2i { int v[2]; int x() const { return v[0]; } int y() const { return v[1]; } };
typedef std::vector<Array2i> DiscreteScan2D;
struct SearchParameters {
  struct LinearBounds { int min_x, max_x, min_y, max_y; };
  SearchParameters(int num_linear_perturbations, int num_angular_perturbations,
                   double angular_perturbation_step_size, double resolution)
      : num_angular_perturbations(num_angular_perturbations),
        angular_perturbation_step_size(angular_perturbation_step_size), resolution(resolution),
        num_scans(2 * num_angular_perturbations + 1),
        linear_bounds(num_scans, LinearBounds{-num_linear_perturbations, num_linear_perturbations,
                                              -num_linear_perturbations, num_linear_perturbations}) {}
  int num_angular_perturbations;
  double angular_perturbation_step_size;
  double resolution;
  int num_scans;
  std::vector<LinearBounds> linear_bounds;
};
struct Candidate2D {   // :74-103
  Candidate2D(int init_scan_index, int init_x_index_offset, int init_y_index_offset,
              const SearchParameters& sp)
      : scan_index(init_scan_index), x_index_offset(init_x_index_offset),
        y_index_offset(init_y_index_offset), x(-y_index_offset * sp.resolution),
        y(-x_index_offset * sp.resolution),
        orientation((scan_index - sp.num_angular_perturbations) *
                    sp.angular_perturbation_step_size) {}
  int scan_index = 0, x_index_offset = 0, y_index_offset = 0;
  double x = 0., y = 0., orientation = 0.;
  float score = 0.f;
  bool operator<(const Candidate2D& other) const { return score < other.score; }
  bool operator>(const Candidate2D& other) const { return score > other.score; }
};
}  // namespace scan_matching

namespace scan_matching {
namespace proto {
// proto/scan_matching/fast_correlative_scan_matcher_options_2d.proto
class FastCorrelativeScanMatcherOptions2D {
 public:
  double linear_search_window() const { return linear_search_window_; }
  double angular_search_window() const { return angular_search_window_; }
  int branch_and_bound_depth() const { return branch_and_bound_depth_; }
  void set_linear_search_window(double v) { linear_search_window_ = v; }
  void set_angular_search_window(double v) { angular_search_window_ = v; }
  void set_branch_and_bound_depth(int v) { branch_and_bound_depth_ = v; }
 private:
  double linear_search_window_ = 0., angular_search_window_ = 0.;
  int branch_and_bound_depth_ = 1;
};
// proto/scan_matching/real_time_correlative_scan_matcher_options.proto
class RealTimeCorrelativeScanMatcherOptions {
 public:
  double linear_search_window() const { return lin_; }
  double angular_search_window() const { return ang_; }
  double translation_delta_cost_weight() const { return wt_; }
  double rotation_delta_cost_weight() const { return wr_; }
  void set_linear_search_window(double v) { lin_ = v; }
  void set_angular_search_window(double v) { ang_ = v; }
  void set_translation_delta_cost_weight(double v) { wt_ = v; }
  void set_rotation_delta_cost_weight(double v) { wr_ = v; }
 private:
  double lin_ = 0., ang_ = 0., wt_ = 0., wr_ = 0.;
};
// proto/scan_matching/ceres_scan_matcher_options_2d.proto + common/proto/ceres_solver_options.proto
// (defaults: configuration_files/pose_graph.lua:30-39)
class CeresScanMatcherOptions2D {
 public:
  struct CeresSolverOptions {
    bool use_nonmonotonic_steps_ = true;
    int max_num_iterations_ = 10, num_threads_ = 1;
    bool use_nonmonotonic_steps() const { return use_nonmonotonic_steps_; }
    int max_num_iterations() const { return max_num_iterations_; }
    int num_threads() const { return num_threads_; }
  };
  double occupied_space_weight() const { return occupied_; }
  double translation_weight() const { return translation_; }
  double rotation_weight() const { return rotation_; }
  const CeresSolverOptions& ceres_solver_options() const { return solver_; }
  CeresSolverOptions* mutable_ceres_solver_options() { return &solver_; }
  void set_occupied_space_weight(double v) { occupied_ = v; }
  void set_translation_weight(double v) { translation_ = v; }
  void set_rotation_weight(double v) { rotation_ = v; }
 private:
  double occupied_ = 20., translation_ = 10., rotation_ = 1.;
  CeresSolverOptions solver_;
};
// proto/scan_matching/ceres_scan_matcher_options_3d.proto:21-26
class IntensityCostFunctionOptions {
 public:
  double weight() const { return weight_; }
  double huber_scale() const { return huber_scale_; }
  float intensity_threshold() const { return intensity_threshold_; }
  void set_weight(double v) { weight_ = v; }
  void set_huber_scale(double v) { huber_scale_ = v; }
  void set_intensity_threshold(float v) { intensity_threshold_ = v; }
 private:
  double weight_ = 0., huber_scale_ = 0.;
  float intensity_threshold_ = 0.f;
};
// proto/scan_matching/ceres_scan_matcher_options_3d.proto (defaults: pose_graph.lua:49-60)
class CeresScanMatcherOptions3D {
 public:
  int occupied_space_weight_size() const { return 2; }
  const IntensityCostFunctionOptions& intensity_cost_function_options(int i) const {
    return intensity_[i];
  }
  IntensityCostFunctionOptions* mutable_intensity_cost_function_options(int i) {
    return &intensity_[i];
  }
  double occupied_space_weight(int i) const { return occupied_[i]; }
  double translation_weight() const { return translation_; }
  double rotation_weight() const { return rotation_; }
  bool only_optimize_yaw() const { return only_optimize_yaw_; }
  const CeresScanMatcherOptions2D::CeresSolverOptions& ceres_solver_options() const {
    return solver_;
  }
  CeresScanMatcherOptions2D::CeresSolverOptions* mutable_ceres_solver_options() {
    return &solver_;
  }
  void set_occupied_space_weight(int i, double v) { occupied_[i] = v; }
  void set_translation_weight(double v) { translation_ = v; }
  void set_rotation_weight(double v) { rotation_ = v; }
 private:
  double occupied_[2] = {5., 30.};
  IntensityCostFunctionOptions intensity_[2];
  double translation_ = 10., rotation_ = 1.;
  bool only_optimize_yaw_ = false;
  CeresScanMatcherOptions2D::CeresSolverOptions solver_{false, 10, 1};
};
// proto/scan_matching/fast_correlative_scan_matcher_options_3d.proto
class FastCorrelativeScanMatcherOptions3D {
 public:
  int branch_and_bound_depth() const { return o.branch_and_bound_depth; }
  int full_resolution_depth() const { return o.full_resolution_depth; }
  double min_rotational_score() const { return o.min_rotational_score; }
  double min_low_resolution_score() const { return o.min_low_resolution_score; }
  double linear_xy_search_window() const { return o.linear_xy_search_window; }
  double linear_z_search_window() const { return o.linear_z_search_window; }
  double angular_search_window() const { return o.angular_search_window; }
  struct { int branch_and_bound_depth = 8, full_resolution_depth = 3;
           double min_rotational_score = 0.77, min_low_resolution_score = 0.55,
                  linear_xy_search_window = 5., linear_z_search_window = 1.,
                  angular_search_window = 0.2617993877991494; } o;
};
}  // namespace proto
}  // namespace scan_matching
}  // namespace mapping
}  // namespace cartographer

// ---- stand-ins for the ConstraintBuilder's surroundings --------------------------
namespace cartographer {
namespace common {
// common/task.h:36-80 and common/thread_pool.h:35-49, reduced to what the builders use.
class Task {
 public:
  void SetWorkItem(const std::function<void()>& work_item) { work_item_ = work_item; }
  void Execute() { if (work_item_) work_item_(); }
 private:
  std::function<void()> work_item_;
};
class ThreadPoolInterface {
 public:
  virtual ~ThreadPoolInterface() {}
  virtual std::weak_ptr<Task> Schedule(std::unique_ptr<Task> task) = 0;
};
// Runs every task at once on the calling thread (enough for the self-test; a checkout
// uses common::ThreadPool).
class InlineThreadPool : public ThreadPoolInterface {
 public:
  std::weak_ptr<Task> Schedule(std::unique_ptr<Task> task) override {
    std::shared_ptr<Task> shared(std::move(task));
    shared->Execute();
    return shared;
  }
};
// common/fixed_ratio_sampler.cc:23-39
class FixedRatioSampler {
 public:
  explicit FixedRatioSampler(double ratio) : ratio_(ratio) {}
  bool Pulse() {
    ++num_pulses_;
    if (static_cast<double>(num_samples_) / num_pulses_ < ratio_) {
      ++num_samples_;
      return true;
    }
    return false;
  }
 private:
  const double ratio_;
  int64_t num_pulses_ = 0, num_samples_ = 0;
};
}  // namespace common

namespace mapping {
// mapping/id.h:43-82
struct SubmapId {
  int trajectory_id, submap_index;
  bool operator<(const SubmapId& o) const {
    return trajectory_id != o.trajectory_id ? trajectory_id < o.trajectory_id
                                            : submap_index < o.submap_index;
  }
};
struct NodeId {
  int trajectory_id, node_index;
  bool operator<(const NodeId& o) const {
    return trajectory_id != o.trajectory_id ? trajectory_id < o.trajectory_id
                                            : node_index < o.node_index;
  }
};
// mapping/2d/submap_2d.h:43-73 / mapping/3d/submap_3d.h:41-83: what the builders read.
class Submap2D {
 public:
  Submap2D(const Grid2D* grid, const transform::Rigid2d& local_pose_2d)
      : grid_(grid), local_pose_2d_(local_pose_2d) {}
  const Grid2D* grid() const { return grid_; }
  // stands for transform::Project2D(local_pose()) = ComputeSubmapPose (submap_2d.h, constraint_builder_2d.cc:48-50)
  const transform::Rigid2d& local_pose_2d() const { return local_pose_2d_; }
 private:
  const Grid2D* grid_;
  transform::Rigid2d local_pose_2d_;
};
class Submap3D {
 public:
  Submap3D(const HybridGrid* high, const HybridGrid* low, const std::vector<float>* histogram)
      : high_(high), low_(low), histogram_(histogram) {}
  const HybridGrid& high_resolution_hybrid_grid() const { return *high_; }
  const HybridGrid& low_resolution_hybrid_grid() const { return *low_; }
  const std::vector<float>& rotational_scan_matcher_histogram() const { return *histogram_; }
 private:
  const HybridGrid* high_;
  const HybridGrid* low_;
  const std::vector<float>* histogram_;
};
// mapping/pose_graph_interface.h:36-53
struct PoseGraphInterface {
  struct Constraint {
    struct Pose {
      transform::Rigid3d zbar_ij;
      double translation_weight;
      double rotation_weight;
    };
    SubmapId submap_id;
    NodeId node_id;
    Pose pose;
    enum Tag { INTRA_SUBMAP, INTER_SUBMAP } tag;
  };
};
namespace constraints {
namespace proto {
// constraints/proto/constraint_builder_options.proto (fields on the path)
struct ConstraintBuilderOptions {
  double sampling_ratio_ = 0.3, max_constraint_distance_ = 15., min_score_ = 0.55,
         global_localization_min_score_ = 0.6, loop_closure_translation_weight_ = 1.1e4,
         loop_closure_rotation_weight_ = 1e5;
  scan_matching::proto::FastCorrelativeScanMatcherOptions2D fast2d_;
  scan_matching::proto::FastCorrelativeScanMatcherOptions3D fast3d_;
  scan_matching::proto::CeresScanMatcherOptions2D ceres2d_;
  scan_matching::proto::CeresScanMatcherOptions3D ceres3d_;
  const scan_matching::proto::CeresScanMatcherOptions3D& ceres_scan_matcher_options_3d() const {
    return ceres3d_;
  }
  const scan_matching::proto::CeresScanMatcherOptions2D& ceres_scan_matcher_options() const {
    return ceres2d_;
  }
  double sampling_ratio() const { return sampling_ratio_; }
  double max_constraint_distance() const { return max_constraint_distance_; }
  double min_score() const { return min_score_; }
  double global_localization_min_score() const { return global_localization_min_score_; }
  double loop_closure_translation_weight() const { return loop_closure_translation_weight_; }
  double loop_closure_rotation_weight() const { return loop_closure_rotation_weight_; }
  const scan_matching::proto::FastCorrelativeScanMatcherOptions2D&
  fast_correlative_scan_matcher_options() const { return fast2d_; }
  const scan_matching::proto::FastCorrelativeScanMatcherOptions3D&
  fast_correlative_scan_matcher_options_3d() const { return fast3d_; }
};
}  // namespace proto
}  // namespace constraints
}  // namespace mapping
}  // namespace cartographer

#endif  // CSM_ADAPTER_COMPAT_H_
