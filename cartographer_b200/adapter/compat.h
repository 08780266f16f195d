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

#include <array>
#include <cmath>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <unordered_set>
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
// sensor/rangefinder_point.h:36-40 and sensor/point_cloud.h:95 (TimedPointCloud).
struct TimedRangefinderPoint {
  struct { float v[3]; float x() const { return v[0]; } float y() const { return v[1]; } float z() const { return v[2]; } } position;
  float time;
};
using TimedPointCloud = std::vector<TimedRangefinderPoint>;
// sensor/timed_point_cloud_data.h:36-45.
struct TimedPointCloudOriginData {
  struct RangeMeasurement {
    TimedRangefinderPoint point_time;
    float intensity;
    size_t origin_index;
  };
};
namespace proto {
// sensor/proto/adaptive_voxel_filter_options.proto: three float fields.
class AdaptiveVoxelFilterOptions {
 public:
  float max_length() const { return max_length_; }
  float min_num_points() const { return min_num_points_; }
  float max_range() const { return max_range_; }
  void set_max_length(float v) { max_length_ = v; }
  void set_min_num_points(float v) { min_num_points_ = v; }
  void set_max_range(float v) { max_range_ = v; }
 private:
  float max_length_ = 0.f, min_num_points_ = 0.f, max_range_ = 0.f;
};
}  // namespace proto
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
  // :159-163 and :184-189, with Eigen's Quaternion * Vector3 (_transformVector) and
  // quaternion product in their scalar order
  Rigid3d inverse() const {
    const Quaterniond q{q_.w_, -q_.x_, -q_.y_, -q_.z_};
    const Vector t = Rotate(q, t_);
    return Rigid3d({{-t.v[0], -t.v[1], -t.v[2]}}, q);
  }
  friend Rigid3d operator*(const Rigid3d& a, const Rigid3d& b) {
    Vector t = Rotate(a.q_, b.t_);
    for (int k = 0; k < 3; ++k) t.v[k] = t.v[k] + a.t_.v[k];
    const Quaterniond& p = a.q_;
    const Quaterniond& q = b.q_;
    const double w = p.w_ * q.w_ - p.x_ * q.x_ - p.y_ * q.y_ - p.z_ * q.z_;
    const double x = p.w_ * q.x_ + p.x_ * q.w_ + p.y_ * q.z_ - p.z_ * q.y_;
    const double y = p.w_ * q.y_ + p.y_ * q.w_ + p.z_ * q.x_ - p.x_ * q.z_;
    const double z = p.w_ * q.z_ + p.z_ * q.w_ + p.x_ * q.y_ - p.y_ * q.x_;
    const double n = std::sqrt(w * w + x * x + y * y + z * z);
    return Rigid3d(t, Quaterniond{w / n, x / n, y / n, z / n});
  }
  // Eigen's Quaterniond * Vector3d (_transformVector)
  static Vector Rotate(const Quaterniond& q, const Vector& c) {
    const double* v = c.v;
    double uv[3] = {q.y_ * v[2] - q.z_ * v[1], q.z_ * v[0] - q.x_ * v[2], q.x_ * v[1] - q.y_ * v[0]};
    for (double& u : uv) u += u;
    const double x[3] = {q.y_ * uv[2] - q.z_ * uv[1], q.z_ * uv[0] - q.x_ * uv[2],
                         q.x_ * uv[1] - q.y_ * uv[0]};
    return Vector{{v[0] + q.w_ * uv[0] + x[0], v[1] + q.w_ * uv[1] + x[1],
                   v[2] + q.w_ * uv[2] + x[2]}};
  }
  Vector t_;
  Quaterniond q_;
};
// Eigen's Quaterniond product, in its scalar order, without normalisation.
inline Quaterniond operator*(const Quaterniond& p, const Quaterniond& q) {
  return Quaterniond{p.w_ * q.w_ - p.x_ * q.x_ - p.y_ * q.y_ - p.z_ * q.z_,
                     p.w_ * q.x_ + p.x_ * q.w_ + p.y_ * q.z_ - p.z_ * q.y_,
                     p.w_ * q.y_ + p.y_ * q.w_ + p.z_ * q.x_ - p.x_ * q.z_,
                     p.w_ * q.z_ + p.z_ * q.w_ + p.x_ * q.y_ - p.y_ * q.x_};
}
// transform/transform.h:42-47
inline double GetYaw(const Quaterniond& rotation) {
  const Rigid3d::Vector direction = Rigid3d::Rotate(rotation, {{1., 0., 0.}});
  return std::atan2(direction.y(), direction.x());
}
}  // namespace transform

namespace mapping {
namespace proto {
// mapping/proto/submaps_options_3d.proto
class SubmapsOptions3D {
 public:
  double high_resolution() const { return high_resolution_; }
  double high_resolution_max_range() const { return high_resolution_max_range_; }
  double low_resolution() const { return low_resolution_; }
  int32_t num_range_data() const { return num_range_data_; }
  const RangeDataInserterOptions3D& range_data_inserter_options() const { return inserter_; }
  RangeDataInserterOptions3D* mutable_range_data_inserter_options() { return &inserter_; }
  void set_high_resolution(double v) { high_resolution_ = v; }
  void set_high_resolution_max_range(double v) { high_resolution_max_range_ = v; }
  void set_low_resolution(double v) { low_resolution_ = v; }
  void set_num_range_data(int32_t v) { num_range_data_ = v; }
 private:
  double high_resolution_ = 0., high_resolution_max_range_ = 0., low_resolution_ = 0.;
  int32_t num_range_data_ = 0;
  RangeDataInserterOptions3D inserter_;
};
// mapping/proto/grid_2d_options.proto: the grid type and the float resolution
class GridOptions2D {
 public:
  enum GridType { INVALID_GRID = 0, PROBABILITY_GRID = 1, TSDF = 2 };
  GridType grid_type() const { return grid_type_; }
  float resolution() const { return resolution_; }
  void set_grid_type(GridType v) { grid_type_ = v; }
  void set_resolution(float v) { resolution_ = v; }
 private:
  GridType grid_type_ = PROBABILITY_GRID;
  float resolution_ = 0.f;
};
// mapping/proto/range_data_inserter_options.proto
class RangeDataInserterOptions {
 public:
  enum RangeDataInserterType {
    INVALID_INSERTER = 0, PROBABILITY_GRID_INSERTER_2D = 1, TSDF_INSERTER_2D = 2 };
  RangeDataInserterType range_data_inserter_type() const { return type_; }
  void set_range_data_inserter_type(RangeDataInserterType v) { type_ = v; }
  const ProbabilityGridRangeDataInserterOptions2D&
  probability_grid_range_data_inserter_options_2d() const { return probability_; }
  ProbabilityGridRangeDataInserterOptions2D*
  mutable_probability_grid_range_data_inserter_options_2d() { return &probability_; }
 private:
  RangeDataInserterType type_ = PROBABILITY_GRID_INSERTER_2D;
  ProbabilityGridRangeDataInserterOptions2D probability_;
};
// mapping/proto/submaps_options_2d.proto
class SubmapsOptions2D {
 public:
  int32_t num_range_data() const { return num_range_data_; }
  const GridOptions2D& grid_options_2d() const { return grid_; }
  GridOptions2D* mutable_grid_options_2d() { return &grid_; }
  const RangeDataInserterOptions& range_data_inserter_options() const { return inserter_; }
  RangeDataInserterOptions* mutable_range_data_inserter_options() { return &inserter_; }
  void set_num_range_data(int32_t v) { num_range_data_ = v; }
 private:
  int32_t num_range_data_ = 0;
  GridOptions2D grid_;
  RangeDataInserterOptions inserter_;
};
}  // namespace proto
namespace scan_matching {
// mapping/internal/3d/scan_matching/rotational_scan_matcher.cc:141-162, on the std::vector<float>
// that stands in for Eigen::VectorXf.
struct RotationalScanMatcher {
  static std::vector<float> RotateHistogram(const std::vector<float>& histogram,
                                            const float angle) {
    const int size = static_cast<int>(histogram.size());
    if (size == 0) return histogram;
    const float rotate_by_buckets = -angle * size / M_PI;
    int full_buckets = static_cast<int>(std::lround(rotate_by_buckets - 0.5f));
    const float fraction = rotate_by_buckets - full_buckets;
    while (full_buckets < 0) full_buckets += size;
    std::vector<float> rotated(size);
    for (int i = 0; i != size; ++i)
      rotated[i] = fraction * histogram[(i + 1 + full_buckets) % size] +
                   (1.f - fraction) * histogram[(i + full_buckets) % size];
    return rotated;
  }
};
}  // namespace scan_matching
}  // namespace mapping

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
  // what OverlappingSubmapsTrimmer2D reads (mapping/submaps.h:61-80): local_pose() and
  // insertion_finished(); the grid lives on the device
  Submap2D(const transform::Rigid3d& local_pose, bool insertion_finished)
      : grid_(nullptr), local_pose_(local_pose), insertion_finished_(insertion_finished) {}
  const Grid2D* grid() const { return grid_; }
  // stands for transform::Project2D(local_pose()) = ComputeSubmapPose (submap_2d.h, constraint_builder_2d.cc:48-50)
  const transform::Rigid2d& local_pose_2d() const { return local_pose_2d_; }
  const transform::Rigid3d& local_pose() const { return local_pose_; }
  bool insertion_finished() const { return insertion_finished_; }
 private:
  const Grid2D* grid_;
  transform::Rigid2d local_pose_2d_;
  transform::Rigid3d local_pose_;
  bool insertion_finished_ = false;
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
  struct SubmapData {   // :55-58
    std::shared_ptr<const Submap2D> submap;
    transform::Rigid3d pose;
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

// mapping/id.h:194-428: the read-only part of MapById that the trimmer uses (ordered iteration
// with .id and .data, size(), Contains(), at()).
template <typename IdType, typename DataType>
class MapById {
 public:
  struct IdDataReference {
    const IdType& id;
    const DataType& data;
  };
  class ConstIterator {
   public:
    explicit ConstIterator(typename std::map<IdType, DataType>::const_iterator it) : it_(it) {}
    IdDataReference operator*() const { return IdDataReference{it_->first, it_->second}; }
    ConstIterator& operator++() {
      ++it_;
      return *this;
    }
    bool operator!=(const ConstIterator& o) const { return it_ != o.it_; }
   private:
    typename std::map<IdType, DataType>::const_iterator it_;
  };
  void Insert(const IdType& id, const DataType& data) { map_[id] = data; }
  void Trim(const IdType& id) { map_.erase(id); }
  size_t size() const { return map_.size(); }
  bool Contains(const IdType& id) const { return map_.count(id) != 0; }
  const DataType& at(const IdType& id) const { return map_.at(id); }
  ConstIterator begin() const { return ConstIterator(map_.begin()); }
  ConstIterator end() const { return ConstIterator(map_.end()); }
 private:
  std::map<IdType, DataType> map_;
};

// mapping/trajectory_node.h:35-72: the node's time (common::Time, whose ticks the trimmer
// reads through time_since_epoch().count()).
struct TrajectoryNode {
  struct Time {
    struct Ticks {
      int64_t ticks;
      int64_t count() const { return ticks; }
    };
    int64_t ticks;
    Ticks time_since_epoch() const { return Ticks{ticks}; }
  };
  Time time_;
  Time time() const { return time_; }
};

// mapping/pose_graph_trimmer.h:27-61
class Trimmable {
 public:
  virtual ~Trimmable() {}
  virtual MapById<SubmapId, PoseGraphInterface::SubmapData> GetOptimizedSubmapData() const = 0;
  virtual const MapById<NodeId, TrajectoryNode>& GetTrajectoryNodes() const = 0;
  virtual const std::vector<PoseGraphInterface::Constraint>& GetConstraints() const = 0;
  virtual void TrimSubmap(const SubmapId& submap_id) = 0;
};
class PoseGraphTrimmer {
 public:
  virtual ~PoseGraphTrimmer() {}
  virtual void Trim(Trimmable* pose_graph) = 0;
  virtual bool IsFinished() = 0;
};
}  // namespace mapping
}  // namespace cartographer

// ---- points processing (io/points_batch.h, io/points_processor.h) ----
namespace Eigen {
// The Eigen::Array2i DrawProbabilityGrid fills with the offset of the cropped limits.
struct Array2i {
  Array2i() = default;
  Array2i(int x, int y) : v{x, y} {}
  int x() const { return v[0]; }
  int y() const { return v[1]; }
  int v[2] = {0, 0};
};
}  // namespace Eigen

namespace absl {
// The set type io::RemovePoints takes (absl/container/flat_hash_set.h).
template <class T>
using flat_hash_set = std::unordered_set<T>;
}  // namespace absl

namespace cartographer {
namespace common {
using Time = int64_t;   // common/time.h: a std::chrono time point there, compared the same way
}  // namespace common
namespace transform {
// transform/rigid_transform.h:116-196 (Rigid3<float>): the accessors the X-ray adapter reads.
class Rigid3f {
 public:
  struct Vector { float x_, y_, z_; float x() const { return x_; } float y() const { return y_; } float z() const { return z_; } };
  struct Quaternion { float w_, x_, y_, z_; float w() const { return w_; } float x() const { return x_; } float y() const { return y_; } float z() const { return z_; } };
  Rigid3f(const Vector& t, const Quaternion& q) : t_(t), q_(q) {}
  const Vector& translation() const { return t_; }
  const Quaternion& rotation() const { return q_; }
 private:
  Vector t_;
  Quaternion q_;
};
}  // namespace transform
namespace mapping {
// mapping/detect_floors.h:26-39.
struct Timespan {
  common::Time start;
  common::Time end;
};
struct Floor {
  std::vector<Timespan> timespans;
  double z;
};
namespace proto {
struct Trajectory {};   // mapping/proto/trajectory.proto: not drawn outside a checkout
}  // namespace proto
}  // namespace mapping
namespace io {
using FloatColor = std::array<float, 3>;   // io/color.h
using Uint8Color = std::array<uint8_t, 3>;
// io/file_writer.h:28-65.
class FileWriter {
 public:
  virtual ~FileWriter() {}
  virtual bool WriteHeader(const char* data, size_t len) = 0;
  virtual bool Write(const char* data, size_t len) = 0;
  virtual bool Close() = 0;
  virtual std::string GetFilename() = 0;
};
using FileWriterFactory = std::function<std::unique_ptr<FileWriter>(const std::string& filename)>;
// io/image.h:30-61 without cairo: the pixels as cairo ARGB32 words, row-major.  A checkout's
// WritePng encodes a PNG through cairo; this stand-in writes the words themselves
// (little-endian), which is what the self-test compares.
class Image {
 public:
  Image(int width, int height) : width_(width), height_(height), pixels_(width * height, 0) {}
  int width() const { return width_; }
  int height() const { return height_; }
  void SetPixel(int x, int y, const Uint8Color& color) {
    pixels_[y * width_ + x] = static_cast<uint32_t>(255) << 24 |
                              static_cast<uint32_t>(color[0]) << 16 |
                              static_cast<uint32_t>(color[1]) << 8 | color[2];
  }
  void WritePng(FileWriter* const file_writer) {
    file_writer->Write(reinterpret_cast<const char*>(pixels_.data()), 4 * pixels_.size());
  }
 private:
  int width_, height_;
  std::vector<uint32_t> pixels_;
};
// io/points_batch.h:31-66 (origin is an Eigen::Vector3f there, zero by default).
struct PointsBatch {
  struct { float v[3] = {0.f, 0.f, 0.f}; float x() const { return v[0]; } float y() const { return v[1]; } float z() const { return v[2]; } } origin;
  common::Time start_time = 0;
  std::string frame_id;
  int trajectory_id = 0;
  std::vector<sensor::RangefinderPoint> points;
  std::vector<float> intensities;   // empty, or one per point
  std::vector<FloatColor> colors;   // empty, or one per point
};
// io/points_batch.cc:22-49: the points whose indices are not in to_remove, in order, with their
// intensities and colors where the batch has them.
inline void RemovePoints(absl::flat_hash_set<int> to_remove, PointsBatch* batch) {
  PointsBatch kept;
  for (size_t i = 0; i < batch->points.size(); ++i) {
    if (to_remove.count(static_cast<int>(i))) continue;
    kept.points.push_back(batch->points[i]);
    if (!batch->intensities.empty()) kept.intensities.push_back(batch->intensities[i]);
    if (!batch->colors.empty()) kept.colors.push_back(batch->colors[i]);
  }
  batch->points = std::move(kept.points);
  batch->intensities = std::move(kept.intensities);
  batch->colors = std::move(kept.colors);
}
// io/points_processor.h:27-52.
class PointsProcessor {
 public:
  enum class FlushResult { kRestartStream, kFinished };
  PointsProcessor() {}
  virtual ~PointsProcessor() {}
  virtual void Process(std::unique_ptr<PointsBatch> points_batch) = 0;
  virtual FlushResult Flush() = 0;
};
}  // namespace io
}  // namespace cartographer

#endif  // CSM_ADAPTER_COMPAT_H_
