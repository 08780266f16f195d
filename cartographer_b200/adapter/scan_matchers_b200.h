// Drop-in C++ classes with the reference's names, namespaces and signatures that
// forward to the C ABI (include/csm_abi.h).  A Cartographer checkout replaces the
// bodies of
//   mapping/internal/2d/scan_matching/fast_correlative_scan_matcher_2d.{h,cc}
//   mapping/internal/2d/scan_matching/real_time_correlative_scan_matcher_2d.{h,cc}
// with this header (see INTEGRATION.md); callers — ConstraintBuilder2D
// (constraints/constraint_builder_2d.cc:213-215, 226-228) and
// LocalTrajectoryBuilder2D::ScanMatch (internal/2d/local_trajectory_builder_2d.cc:77-82)
// — compile unchanged.
//
// Error convention: the reference CHECK-aborts on programmer errors; the adapter
// keeps that contract by aborting with the C ABI's error string (the ABI itself
// never aborts).  "No pose above min_score" returns false and leaves the outputs
// untouched, exactly like fast_correlative_scan_matcher_2d.cc:253-261.
#ifndef CSM_ADAPTER_SCAN_MATCHERS_B200_H_
#define CSM_ADAPTER_SCAN_MATCHERS_B200_H_

#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "../../include/csm_abi.h"

#if defined(__has_include) && __has_include("cartographer/mapping/2d/grid_2d.h")
#include "cartographer/mapping/2d/grid_2d.h"
#include "cartographer/mapping/internal/2d/scan_matching/correlative_scan_matcher_2d.h"
#include "cartographer/mapping/internal/2d/tsdf_2d.h"
#include "cartographer/mapping/proto/scan_matching/ceres_scan_matcher_options_2d.pb.h"
#include "cartographer/mapping/proto/scan_matching/fast_correlative_scan_matcher_options_2d.pb.h"
#include "cartographer/mapping/proto/scan_matching/real_time_correlative_scan_matcher_options.pb.h"
#include "cartographer/mapping/proto/hybrid_grid.pb.h"
#include "cartographer/mapping/proto/range_data_inserter_options_3d.pb.h"
#include "cartographer/mapping/proto/submap_visualization.pb.h"
#include "cartographer/mapping/proto/probability_grid_range_data_inserter_options_2d.pb.h"
#include "cartographer/sensor/point_cloud.h"
#include "cartographer/sensor/range_data.h"
#include "cartographer/transform/rigid_transform.h"
#define CSM_ADAPTER_REAL_CARTOGRAPHER 1
#else
#include "compat.h"
#endif

namespace cartographer {
namespace mapping {
namespace scan_matching {

namespace b200_internal {
// Programmer errors and CUDA failures keep the reference's CHECK semantics (abort with the
// ABI's message).  CSM_E_CAPACITY — an engine limit the reference does not have (more than
// 2^21 exactly tied optima, a scan point more than 30 000 cells from the grid origin) — is
// logged and reported to the caller, which treats the search as "no match": one
// pathological (submap, node) pair must not take the SLAM process down.
inline bool Check(csm_status s) {
  if (s == CSM_OK) return true;
  std::fprintf(stderr, "libcsm_b200: %s\n", csm_last_error_string());
  if (s == CSM_E_CAPACITY) return false;
  std::abort();  // glog CHECK semantics of the reference
}
inline std::vector<float> Flatten(const sensor::PointCloud& point_cloud) {
  std::vector<float> xyz;
  xyz.reserve(3 * point_cloud.size());
  for (const auto& p : point_cloud.points()) {
    xyz.push_back(p.position.x());
    xyz.push_back(p.position.y());
    xyz.push_back(p.position.z());
  }
  return xyz;
}
// A Rigid3d as the ABI's pose[7] (tx, ty, tz, qw, qx, qy, qz); FromPose7 is the way back.
inline void Pose7(const transform::Rigid3d& p, double out[7]) {
  out[0] = p.translation().x(); out[1] = p.translation().y(); out[2] = p.translation().z();
  out[3] = p.rotation().w(); out[4] = p.rotation().x(); out[5] = p.rotation().y();
  out[6] = p.rotation().z();
}
// The serialised message of one *_to_proto entry point (sized by a first call).  A message
// of 2 GiB or more, which protobuf cannot hold, aborts as the reference's serialiser does.
template <typename Handle>
std::string Serialize(csm_status (*to_proto)(const Handle*, uint8_t*, int64_t, int64_t*),
                      const Handle* handle) {
  int64_t size = 0;
  if (!Check(to_proto(handle, nullptr, 0, &size))) std::abort();
  std::string bytes(static_cast<size_t>(size), '\0');
  if (!Check(to_proto(handle, reinterpret_cast<uint8_t*>(&bytes[0]), size, &size))) std::abort();
  return bytes;
}
// A proto::HybridGrid / proto::Grid2D parsed from those bytes in a Cartographer checkout; the
// bytes themselves in the stand-in build.
#ifdef CSM_ADAPTER_REAL_CARTOGRAPHER
template <typename Message>
Message Parse(const std::string& bytes) {
  Message message;
  if (!message.ParseFromString(bytes)) std::abort();
  return message;
}
using HybridGridProto = ::cartographer::mapping::proto::HybridGrid;
using Grid2DProto = ::cartographer::mapping::proto::Grid2D;
using SubmapTextureProto = ::cartographer::mapping::proto::SubmapQuery::Response::SubmapTexture;
#else
template <typename Message>
Message Parse(const std::string& bytes) {
  return bytes;
}
using HybridGridProto = std::string;
using Grid2DProto = std::string;
using SubmapTextureProto = std::string;
#endif
// The serialised texture one *_to_texture entry point draws with `pose`.  Every call does the
// whole work, so the first goes with a buffer that holds most textures and a second, sized
// exactly, only when that one was too small.
template <typename Handle>
std::string DrawTexture(csm_status (*to_texture)(const Handle*, const double*, uint8_t*, int64_t,
                                                 int64_t*),
                        const Handle* handle, const transform::Rigid3d& pose) {
  double p[7];
  Pose7(pose, p);
  std::string bytes(size_t(1) << 16, '\0');
  int64_t size = 0;
  csm_status st = to_texture(handle, p, reinterpret_cast<uint8_t*>(&bytes[0]),
                             static_cast<int64_t>(bytes.size()), &size);
  if (st == CSM_E_CAPACITY && size > static_cast<int64_t>(bytes.size())) {
    bytes.resize(static_cast<size_t>(size));
    st = to_texture(handle, p, reinterpret_cast<uint8_t*>(&bytes[0]), size, &size);
  }
  if (!Check(st)) std::abort();
  bytes.resize(static_cast<size_t>(size));
  return bytes;
}
}  // namespace b200_internal

class DeviceGrid2D;

// fast_correlative_scan_matcher_2d.h:112-136
class FastCorrelativeScanMatcher2D {
 public:
  // The stack of a submap whose grid lives on the device (a DeviceGrid2D::ComputeCroppedGrid
  // result, as Submap2D::Finish leaves it): built from the device cells.
  FastCorrelativeScanMatcher2D(const DeviceGrid2D& grid,
                               const proto::FastCorrelativeScanMatcherOptions2D& options);
  FastCorrelativeScanMatcher2D(const Grid2D& grid,
                               const proto::FastCorrelativeScanMatcherOptions2D& options,
                               int device = 0)
      : options_(options) {
    const MapLimits& l = grid.limits();
    b200_internal::Check(csm_stack2d_create(
        grid.correspondence_cost_cells().data(), l.cell_limits().num_x_cells,
        l.cell_limits().num_y_cells, l.resolution(), l.max().x(), l.max().y(),
        grid.GetMinCorrespondenceCost(), grid.GetMaxCorrespondenceCost(),
        options.branch_and_bound_depth(), device, &stack_));
  }
  ~FastCorrelativeScanMatcher2D() { csm_stack2d_destroy(stack_); }
  FastCorrelativeScanMatcher2D(const FastCorrelativeScanMatcher2D&) = delete;
  FastCorrelativeScanMatcher2D& operator=(const FastCorrelativeScanMatcher2D&) = delete;

  bool Match(const transform::Rigid2d& initial_pose_estimate,
             const sensor::PointCloud& point_cloud, float min_score, float* score,
             transform::Rigid2d* pose_estimate) const {
    const double init[3] = {initial_pose_estimate.translation().x(),
                            initial_pose_estimate.translation().y(),
                            initial_pose_estimate.rotation().angle()};
    return Run(init, 0, point_cloud, min_score, score, pose_estimate);
  }

  bool MatchFullSubmap(const sensor::PointCloud& point_cloud, float min_score, float* score,
                       transform::Rigid2d* pose_estimate) const {
    const double init[3] = {0., 0., 0.};
    return Run(init, 1, point_cloud, min_score, score, pose_estimate);
  }

  const csm_stack2d* stack() const { return stack_; }  // for the batched ConstraintBuilder

 private:
  bool Run(const double init[3], int full, const sensor::PointCloud& point_cloud,
           float min_score, float* score, transform::Rigid2d* pose_estimate) const {
    if (score == nullptr || pose_estimate == nullptr) std::abort();  // CHECK(:232-233)
    const std::vector<float> xyz = b200_internal::Flatten(point_cloud);
    int32_t found = 0;
    float s = 0.f;
    double pose[3] = {0., 0., 0.};
    if (!b200_internal::Check(csm_match2d(stack_, xyz.data(),
                                          static_cast<int32_t>(point_cloud.size()), init, full,
                                          options_.linear_search_window(),
                                          options_.angular_search_window(), min_score, &found,
                                          &s, pose, nullptr)))
      return false;
    if (!found) return false;
    *score = s;
    *pose_estimate = transform::Rigid2d({pose[0], pose[1]}, pose[2]);
    return true;
  }
  const proto::FastCorrelativeScanMatcherOptions2D options_;
  csm_stack2d* stack_ = nullptr;
};

// real_time_correlative_scan_matcher_2d.h:53-85 (ProbabilityGrid and TSDF grids)
class RealTimeCorrelativeScanMatcher2D {
 public:
  explicit RealTimeCorrelativeScanMatcher2D(
      const proto::RealTimeCorrelativeScanMatcherOptions& options, int device = 0)
      : options_(options), device_(device) {}

  double Match(const transform::Rigid2d& initial_pose_estimate,
               const sensor::PointCloud& point_cloud, const Grid2D& grid,
               transform::Rigid2d* pose_estimate) const {
    if (pose_estimate == nullptr) std::abort();  // CHECK(:121)
    const MapLimits& l = grid.limits();
    const std::vector<float> xyz = b200_internal::Flatten(point_cloud);
    const double init[3] = {initial_pose_estimate.translation().x(),
                            initial_pose_estimate.translation().y(),
                            initial_pose_estimate.rotation().angle()};
    double score = 0., pose[3] = {0., 0., 0.};
    bool ok;
    if (grid.GetGridType() == GridType::TSDF) {  // real_time…2d.cc:160-166
      const TSDF2D& tsdf = static_cast<const TSDF2D&>(grid);
#ifdef CSM_ADAPTER_REAL_CARTOGRAPHER
      // TSDF2D keeps its weight cells and converter private (internal/2d/tsdf_2d.h:57-60);
      // the proto form carries exactly what the kernel needs (grid_2d.proto:23-42).
      const proto::Grid2D p = tsdf.ToProto();
      std::vector<uint16_t> tsd(p.cells().begin(), p.cells().end());
      std::vector<uint16_t> weights(p.tsdf_2d().weight_cells().begin(),
                                    p.tsdf_2d().weight_cells().end());
      const float truncation = p.tsdf_2d().truncation_distance();
      const float max_weight = p.tsdf_2d().max_weight();
      const uint16_t* tsd_cells = tsd.data();
      const uint16_t* weight_cells = weights.data();
#else
      const float truncation = tsdf.truncation_distance(), max_weight = tsdf.max_weight();
      const uint16_t* tsd_cells = tsdf.correspondence_cost_cells().data();
      const uint16_t* weight_cells = tsdf.weight_cells().data();
#endif
      ok = b200_internal::Check(csm_rt_match2d_tsdf(
          tsd_cells, weight_cells, l.cell_limits().num_x_cells, l.cell_limits().num_y_cells,
          l.resolution(), l.max().x(), l.max().y(), truncation, max_weight, xyz.data(),
          static_cast<int32_t>(point_cloud.size()), init, options_.linear_search_window(),
          options_.angular_search_window(), options_.translation_delta_cost_weight(),
          options_.rotation_delta_cost_weight(), device_, &score, pose, nullptr));
    } else {
      ok = b200_internal::Check(csm_rt_match2d(
          grid.correspondence_cost_cells().data(), l.cell_limits().num_x_cells,
          l.cell_limits().num_y_cells, l.resolution(), l.max().x(), l.max().y(), xyz.data(),
          static_cast<int32_t>(point_cloud.size()), init, options_.linear_search_window(),
          options_.angular_search_window(), options_.translation_delta_cost_weight(),
          options_.rotation_delta_cost_weight(), device_, &score, pose, nullptr));
    }
    if (!ok) {  // engine capacity: keep the initial estimate (a zero-offset candidate)
      *pose_estimate = initial_pose_estimate;
      return 0.;
    }
    *pose_estimate = transform::Rigid2d({pose[0], pose[1]}, pose[2]);
    return score;
  }

  // Public in the reference (real_time_correlative_scan_matcher_2d.h:75, .cc:151-176):
  // computes the score of every candidate of `candidates` in place.
  void ScoreCandidates(const Grid2D& grid, const std::vector<DiscreteScan2D>& discrete_scans,
                       const SearchParameters& search_parameters,
                       std::vector<Candidate2D>* const candidates) const {
    if (candidates == nullptr || candidates->empty()) return;
    if (grid.GetGridType() != GridType::PROBABILITY_GRID) {
      std::fprintf(stderr, "ScoreCandidates (b200): only ProbabilityGrid is supported\n");
      std::abort();
    }
    const MapLimits& l = grid.limits();
    const int32_t num_scans = static_cast<int32_t>(discrete_scans.size());
    const int32_t n = num_scans ? static_cast<int32_t>(discrete_scans[0].size()) : 0;
    std::vector<int32_t> ds;
    ds.reserve(2 * static_cast<size_t>(num_scans) * n);
    for (const DiscreteScan2D& scan : discrete_scans) {
      if (static_cast<int32_t>(scan.size()) != n) std::abort();  // one cloud, S rotations
      for (const auto& xy : scan) {
        ds.push_back(xy.x());
        ds.push_back(xy.y());
      }
    }
    std::vector<int32_t> cand;
    cand.reserve(3 * candidates->size());
    for (const Candidate2D& c : *candidates) {
      cand.push_back(c.scan_index);
      cand.push_back(c.x_index_offset);
      cand.push_back(c.y_index_offset);
    }
    std::vector<float> scores(candidates->size());
    if (!b200_internal::Check(csm_rt_score_candidates2d(
            grid.correspondence_cost_cells().data(), l.cell_limits().num_x_cells,
            l.cell_limits().num_y_cells, l.resolution(), l.max().x(), l.max().y(), ds.data(),
            num_scans, n, search_parameters.num_angular_perturbations,
            search_parameters.angular_perturbation_step_size, cand.data(),
            static_cast<int32_t>(candidates->size()), options_.translation_delta_cost_weight(),
            options_.rotation_delta_cost_weight(), device_, scores.data())))
      return;
    for (size_t i = 0; i < scores.size(); ++i) (*candidates)[i].score = scores[i];
  }

 private:
  const proto::RealTimeCorrelativeScanMatcherOptions options_;
  int device_;
};

// A ProbabilityGrid kept on the device (csm_rt_grid2d): the form in which the batched
// real-time matcher and the refinement below take the submap's grid.
class DeviceGrid2D {
 public:
  explicit DeviceGrid2D(const Grid2D& grid, int device = 0) : device_(device) {
    if (grid.GetGridType() != GridType::PROBABILITY_GRID) {
      std::fprintf(stderr, "DeviceGrid2D (b200): only ProbabilityGrid is supported\n");
      std::abort();
    }
    const MapLimits& l = grid.limits();
    b200_internal::Check(csm_rt_grid2d_create(
        grid.correspondence_cost_cells().data(), l.cell_limits().num_x_cells,
        l.cell_limits().num_y_cells, l.resolution(), l.max().x(), l.max().y(), device, &grid_));
  }
  // ProbabilityGrid(limits): the all-unknown grid ActiveSubmaps2D::CreateGrid makes, filled
  // by ProbabilityGridRangeDataInserter2D below.
  DeviceGrid2D(const MapLimits& limits, int device) : device_(device) {
    b200_internal::Check(csm_rt_grid2d_create_empty(
        limits.resolution(), limits.max().x(), limits.max().y(),
        limits.cell_limits().num_x_cells, limits.cell_limits().num_y_cells, device, &grid_));
  }
  // TSDF2D(limits, truncation_distance, max_weight): the all-unknown TSDF2D
  // ActiveSubmaps2D::CreateGrid makes for GridType::TSDF, filled by TSDFRangeDataInserter2D below.
  DeviceGrid2D(const MapLimits& limits, float truncation_distance, float max_weight, int device)
      : device_(device) {
    b200_internal::Check(csm_rt_grid2d_create_empty_tsdf(
        limits.resolution(), limits.max().x(), limits.max().y(),
        limits.cell_limits().num_x_cells, limits.cell_limits().num_y_cells, truncation_distance,
        max_weight, device, &grid_));
  }
  ~DeviceGrid2D() { csm_rt_grid2d_destroy(grid_); }
  DeviceGrid2D(const DeviceGrid2D&) = delete;
  DeviceGrid2D& operator=(const DeviceGrid2D&) = delete;
  const csm_rt_grid2d* handle() const { return grid_; }
  csm_rt_grid2d* mutable_handle() { return grid_; }
  int device() const { return device_; }   // the CUDA device the cells live on

  // ProbabilityGrid::ComputeCroppedGrid (probability_grid.cc:91-107), device to device.
  std::unique_ptr<DeviceGrid2D> ComputeCroppedGrid() const {
    csm_rt_grid2d* cropped = nullptr;
    b200_internal::Check(csm_rt_grid2d_crop(grid_, &cropped));
    return std::unique_ptr<DeviceGrid2D>(new DeviceGrid2D(cropped, device_));
  }
  // limits(), the known-cells box and, with cells != nullptr, the cells (num_y x num_x):
  // what Submap2D::ToProto serialises.
  csm_rt_grid2d_info Read(std::vector<uint16_t>* cells) const {
    csm_rt_grid2d_info info;
    b200_internal::Check(csm_rt_grid2d_read(grid_, &info, nullptr, 0));
    if (cells != nullptr) {
      cells->resize(static_cast<size_t>(info.num_x_cells) * info.num_y_cells);
      b200_internal::Check(csm_rt_grid2d_read(grid_, &info, cells->data(),
                                              static_cast<int64_t>(cells->size())));
    }
    return info;
  }
  // ProbabilityGrid::ToProto / TSDF2D::ToProto (csm_rt_grid2d_to_proto): the grid part of
  // Submap2D::ToProto, byte for byte what the reference serialises.
  b200_internal::Grid2DProto ToProto() const {
    return b200_internal::Parse<b200_internal::Grid2DProto>(
        b200_internal::Serialize(csm_rt_grid2d_to_proto, grid_));
  }
  // ProbabilityGrid::DrawToSubmapTexture / TSDF2D::DrawToSubmapTexture
  // (csm_rt_grid2d_to_texture): the texture Submap2D::ToResponseProto adds with the submap's
  // local pose.
  bool DrawToSubmapTexture(b200_internal::SubmapTextureProto* texture,
                           const transform::Rigid3d& local_pose) const {
    *texture = b200_internal::Parse<b200_internal::SubmapTextureProto>(
        b200_internal::DrawTexture(csm_rt_grid2d_to_texture, grid_, local_pose));
    return true;
  }
  // The weight cells of a TSDF2D (num_y x num_x); Read gives its tsd cells.
  void ReadWeights(std::vector<uint16_t>* weight_cells) const {
    const csm_rt_grid2d_info info = Read(nullptr);
    weight_cells->resize(static_cast<size_t>(info.num_x_cells) * info.num_y_cells);
    b200_internal::Check(csm_rt_grid2d_read_weights(grid_, weight_cells->data(),
                                                    static_cast<int64_t>(weight_cells->size())));
  }

 private:
  DeviceGrid2D(csm_rt_grid2d* grid, int device) : device_(device), grid_(grid) {}
  int device_;
  csm_rt_grid2d* grid_ = nullptr;
};

inline FastCorrelativeScanMatcher2D::FastCorrelativeScanMatcher2D(
    const DeviceGrid2D& grid, const proto::FastCorrelativeScanMatcherOptions2D& options)
    : options_(options) {
  b200_internal::Check(csm_stack2d_create_from_rt_grid2d(
      grid.handle(), options.branch_and_bound_depth(), &stack_));
}

// mapping/2d/probability_grid_range_data_inserter_2d.h:33-52 on device grids: Submap2D
// (submap_2d.cc) keeps its grid as a DeviceGrid2D and inserts every scan in place, so the
// real-time matcher and CeresScanMatcher2D read the updated submap without a re-upload, and
// Submap2D::Finish crops it on the device.
class ProbabilityGridRangeDataInserter2D {
 public:
  explicit ProbabilityGridRangeDataInserter2D(
      const mapping::proto::ProbabilityGridRangeDataInserterOptions2D& options, int device = 0) {
    csm_range_inserter_options2d o{};
    o.hit_probability = options.hit_probability();
    o.miss_probability = options.miss_probability();
    o.insert_free_space = options.insert_free_space() ? 1 : 0;
    b200_internal::Check(csm_range_inserter2d_create(&o, device, &inserter_));
  }
  ~ProbabilityGridRangeDataInserter2D() { csm_range_inserter2d_destroy(inserter_); }
  ProbabilityGridRangeDataInserter2D(const ProbabilityGridRangeDataInserter2D&) = delete;
  ProbabilityGridRangeDataInserter2D& operator=(const ProbabilityGridRangeDataInserter2D&) =
      delete;

  // probability_grid_range_data_inserter_2d.cc:124-133; range_data in the grid's frame.
  void Insert(const sensor::RangeData& range_data, DeviceGrid2D* grid) const {
    if (grid == nullptr) std::abort();  // CHECK(:127)
    const std::vector<float> returns = b200_internal::Flatten(range_data.returns);
    const std::vector<float> misses = b200_internal::Flatten(range_data.misses);
    const float origin[3] = {range_data.origin.x(), range_data.origin.y(), range_data.origin.z()};
    b200_internal::Check(csm_range_inserter2d_insert(
        inserter_, origin, returns.data(), static_cast<int32_t>(range_data.returns.size()),
        misses.data(), static_cast<int32_t>(range_data.misses.size()), grid->mutable_handle(),
        nullptr));
  }
  // Insert(range_data, grid) into every grid of `grids`, in one call
  // (csm_range_inserter2d_insert_submaps): what ActiveSubmaps2D::InsertRangeData
  // (submap_2d.cc:162-175) does to its active submaps.  Each grid ends as grids.size() Insert
  // calls in order would leave it; range_data in the local frame.
  void InsertSubmaps(const sensor::RangeData& range_data,
                     const std::vector<DeviceGrid2D*>& grids) const {
    std::vector<csm_rt_grid2d*> handles;
    for (DeviceGrid2D* grid : grids) {
      if (grid == nullptr) std::abort();  // CHECK(:127)
      handles.push_back(grid->mutable_handle());
    }
    const std::vector<float> returns = b200_internal::Flatten(range_data.returns);
    const std::vector<float> misses = b200_internal::Flatten(range_data.misses);
    const float origin[3] = {range_data.origin.x(), range_data.origin.y(), range_data.origin.z()};
    b200_internal::Check(csm_range_inserter2d_insert_submaps(
        inserter_, origin, returns.data(), static_cast<int32_t>(range_data.returns.size()),
        misses.data(), static_cast<int32_t>(range_data.misses.size()), handles.data(),
        static_cast<int32_t>(handles.size()), nullptr));
  }

 private:
  csm_range_inserter2d* inserter_ = nullptr;
};

// mapping/internal/2d/tsdf_range_data_inserter_2d.h:29-50 on device grids: Submap2D with
// GridType::TSDF keeps its grid as a DeviceGrid2D(limits, truncation, max_weight, device) and
// inserts every scan in place.
class TSDFRangeDataInserter2D {
 public:
  explicit TSDFRangeDataInserter2D(const mapping::proto::TSDFRangeDataInserterOptions2D& options,
                                   int device = 0) {
    csm_tsdf_inserter_options2d o{};
    o.truncation_distance = options.truncation_distance();
    o.maximum_weight = options.maximum_weight();
    o.update_free_space = options.update_free_space() ? 1 : 0;
    o.num_normal_samples = options.normal_estimation_options().num_normal_samples();
    o.sample_radius = options.normal_estimation_options().sample_radius();
    o.project_sdf_distance_to_scan_normal = options.project_sdf_distance_to_scan_normal() ? 1 : 0;
    o.update_weight_range_exponent = options.update_weight_range_exponent();
    o.update_weight_angle_scan_normal_to_ray_kernel_bandwidth =
        options.update_weight_angle_scan_normal_to_ray_kernel_bandwidth();
    o.update_weight_distance_cell_to_hit_kernel_bandwidth =
        options.update_weight_distance_cell_to_hit_kernel_bandwidth();
    b200_internal::Check(csm_tsdf_inserter2d_create(&o, device, &inserter_));
  }
  ~TSDFRangeDataInserter2D() { csm_tsdf_inserter2d_destroy(inserter_); }
  TSDFRangeDataInserter2D(const TSDFRangeDataInserter2D&) = delete;
  TSDFRangeDataInserter2D& operator=(const TSDFRangeDataInserter2D&) = delete;

  // tsdf_range_data_inserter_2d.cc:131-165; range_data in the grid's frame (misses unused).
  void Insert(const sensor::RangeData& range_data, DeviceGrid2D* grid) const {
    if (grid == nullptr) std::abort();
    const std::vector<float> returns = b200_internal::Flatten(range_data.returns);
    const float origin[3] = {range_data.origin.x(), range_data.origin.y(), range_data.origin.z()};
    b200_internal::Check(csm_tsdf_inserter2d_insert(
        inserter_, origin, returns.data(), static_cast<int32_t>(range_data.returns.size()),
        grid->mutable_handle(), nullptr));
  }

 private:
  csm_tsdf_inserter2d* inserter_ = nullptr;
};

// ceres_scan_matcher_2d.h:42-64.  Same constructor and Match signature, except that the
// summary is this struct instead of ceres::Solver::Summary (Ceres is not linked; the
// fields are the ones of the same name there).  MatchBatch is the form the constraint
// builder uses: all found matches of a queue in one launch.
class CeresScanMatcher2D {
 public:
  struct Summary {
    double initial_cost = 0., final_cost = 0.;
    int iterations = 0, num_successful_steps = 0;
    int termination = 0;   // csm_ceres_result2d::termination
  };
  struct Job {
    double target_translation[2];
    transform::Rigid2d initial_pose_estimate;
    const sensor::PointCloud* point_cloud;
    const DeviceGrid2D* grid;
  };

  explicit CeresScanMatcher2D(const proto::CeresScanMatcherOptions2D& options, int device = 0)
      : options_(options), device_(device) {}

  template <typename Vector2>
  void Match(const Vector2& target_translation, const transform::Rigid2d& initial_pose_estimate,
             const sensor::PointCloud& point_cloud, const Grid2D& grid,
             transform::Rigid2d* const pose_estimate, Summary* const summary) const {
    const DeviceGrid2D device_grid(grid, device_);
    std::vector<transform::Rigid2d> poses;
    std::vector<Summary> summaries;
    MatchBatch({Job{{target_translation.x(), target_translation.y()}, initial_pose_estimate,
                    &point_cloud, &device_grid}},
               &poses, &summaries);
    *pose_estimate = poses[0];
    if (summary != nullptr) *summary = summaries[0];
  }

  void MatchBatch(const std::vector<Job>& jobs, std::vector<transform::Rigid2d>* poses,
                  std::vector<Summary>* summaries) const {
    poses->clear();
    if (summaries != nullptr) summaries->clear();
    if (jobs.empty()) return;
    std::vector<std::vector<float>> xyz(jobs.size());
    std::vector<csm_ceres_job2d> cj(jobs.size());
    for (size_t i = 0; i < jobs.size(); ++i) {
      xyz[i] = b200_internal::Flatten(*jobs[i].point_cloud);
      cj[i] = csm_ceres_job2d{};
      cj[i].grid = jobs[i].grid->handle();
      cj[i].xyz = xyz[i].data();
      cj[i].num_points = static_cast<int32_t>(jobs[i].point_cloud->size());
      cj[i].target_translation[0] = jobs[i].target_translation[0];
      cj[i].target_translation[1] = jobs[i].target_translation[1];
      cj[i].initial_pose[0] = jobs[i].initial_pose_estimate.translation().x();
      cj[i].initial_pose[1] = jobs[i].initial_pose_estimate.translation().y();
      cj[i].initial_pose[2] = jobs[i].initial_pose_estimate.rotation().angle();
    }
    csm_ceres_options2d o;
    o.occupied_space_weight = options_.occupied_space_weight();
    o.translation_weight = options_.translation_weight();
    o.rotation_weight = options_.rotation_weight();
    o.use_nonmonotonic_steps = options_.ceres_solver_options().use_nonmonotonic_steps() ? 1 : 0;
    o.max_num_iterations = options_.ceres_solver_options().max_num_iterations();
    std::vector<csm_ceres_result2d> res(jobs.size());
    b200_internal::Check(csm_ceres_match2d_batch(cj.data(), static_cast<int32_t>(cj.size()), &o,
                                                 res.data(), nullptr));
    for (const csm_ceres_result2d& r : res) {
      poses->push_back(
          transform::Rigid2d({r.pose_estimate[0], r.pose_estimate[1]}, r.pose_estimate[2]));
      if (summaries != nullptr) {
        Summary s;
        s.initial_cost = r.initial_cost;
        s.final_cost = r.final_cost;
        s.iterations = r.iterations;
        s.num_successful_steps = r.num_successful_steps;
        s.termination = r.termination;
        summaries->push_back(s);
      }
    }
  }

 private:
  const proto::CeresScanMatcherOptions2D options_;
  int device_;
};

#ifndef CSM_ADAPTER_REAL_CARTOGRAPHER
namespace b200_internal {
inline csm_options3d Options3D(const proto::FastCorrelativeScanMatcherOptions3D& options) {
  csm_options3d o;
  o.branch_and_bound_depth = options.branch_and_bound_depth();
  o.full_resolution_depth = options.full_resolution_depth();
  o.min_rotational_score = options.min_rotational_score();
  o.min_low_resolution_score = options.min_low_resolution_score();
  o.linear_xy_search_window = options.linear_xy_search_window();
  o.linear_z_search_window = options.linear_z_search_window();
  o.angular_search_window = options.angular_search_window();
  return o;
}
inline transform::Rigid3d FromPose7(const double p[7]) {
  return transform::Rigid3d({{p[0], p[1], p[2]}}, transform::Quaterniond{p[3], p[4], p[5], p[6]});
}
// A HybridGrid's voxels as the ABI takes them: (x, y, z) index triples and their values.
inline void Flatten(const HybridGrid& grid, std::vector<int32_t>* idx,
                    std::vector<uint16_t>* val) {
  for (const auto& v : grid.voxels()) {
    idx->push_back(v.x);
    idx->push_back(v.y);
    idx->push_back(v.z);
    val->push_back(v.value);
  }
}
// The csm_node3d of a node's data.  Its clouds are flattened into `high` and `low`, which must
// outlive it.
inline csm_node3d Node3D(const TrajectoryNodeData& data, std::vector<float>* high,
                         std::vector<float>* low) {
  *high = Flatten(data.high_resolution_point_cloud);
  *low = Flatten(data.low_resolution_point_cloud);
  csm_node3d node;
  node.high_resolution_point_cloud = high->data();
  node.num_high = static_cast<int32_t>(data.high_resolution_point_cloud.size());
  node.low_resolution_point_cloud = low->data();
  node.num_low = static_cast<int32_t>(data.low_resolution_point_cloud.size());
  node.rotational_scan_matcher_histogram = data.rotational_scan_matcher_histogram.data();
  node.histogram_size = static_cast<int32_t>(data.rotational_scan_matcher_histogram.size());
  node.gravity_alignment[0] = data.gravity_alignment.w();
  node.gravity_alignment[1] = data.gravity_alignment.x();
  node.gravity_alignment[2] = data.gravity_alignment.y();
  node.gravity_alignment[3] = data.gravity_alignment.z();
  return node;
}
}  // namespace b200_internal

class DeviceHybridGrid;

// fast_correlative_scan_matcher_3d.h:66-101.  (Inside a Cartographer checkout the
// same body is used with HybridGrid::Iterator for the voxel walk, Eigen::VectorXf
// for the histograms and TrajectoryNode::Data — see INTEGRATION.md §3.)
class FastCorrelativeScanMatcher3D {
 public:
  struct Result {  // fast_correlative_scan_matcher_3d.h:68-73
    float score;
    transform::Rigid3d pose_estimate;
    float rotational_score;
    float low_resolution_score;
  };

  // The matcher of a submap whose grids live on the device (Submap3D::InsertData on
  // DeviceHybridGrids): built from the grids' non-zero voxels device to device, on their
  // device.  It owns its copies; grid_size_in_voxels as HybridGrid::grid_size() (0 = derive it
  // from the high-resolution grid's non-zero voxels).
  FastCorrelativeScanMatcher3D(const DeviceHybridGrid& hybrid_grid,
                               const DeviceHybridGrid* low_resolution_hybrid_grid,
                               const std::vector<float>* rotational_scan_matcher_histogram,
                               const proto::FastCorrelativeScanMatcherOptions3D& options,
                               int grid_size_in_voxels = 0);
  FastCorrelativeScanMatcher3D(const HybridGrid& hybrid_grid,
                               const HybridGrid* low_resolution_hybrid_grid,
                               const std::vector<float>* rotational_scan_matcher_histogram,
                               const proto::FastCorrelativeScanMatcherOptions3D& options,
                               int device = 0) {
    std::vector<int32_t> hi_idx, lo_idx;
    std::vector<uint16_t> hi_val, lo_val;
    b200_internal::Flatten(hybrid_grid, &hi_idx, &hi_val);
    b200_internal::Flatten(*low_resolution_hybrid_grid, &lo_idx, &lo_val);
    const csm_options3d o = b200_internal::Options3D(options);
    b200_internal::Check(csm_matcher3d_create(
        hi_idx.data(), hi_val.data(), static_cast<int64_t>(hi_val.size()),
        hybrid_grid.resolution(), hybrid_grid.grid_size(), lo_idx.data(), lo_val.data(),
        static_cast<int64_t>(lo_val.size()), low_resolution_hybrid_grid->resolution(),
        rotational_scan_matcher_histogram->data(),
        static_cast<int32_t>(rotational_scan_matcher_histogram->size()), &o, device, &matcher_));
  }
  ~FastCorrelativeScanMatcher3D() { csm_matcher3d_destroy(matcher_); }
  FastCorrelativeScanMatcher3D(const FastCorrelativeScanMatcher3D&) = delete;
  FastCorrelativeScanMatcher3D& operator=(const FastCorrelativeScanMatcher3D&) = delete;

  std::unique_ptr<Result> Match(const transform::Rigid3d& global_node_pose,
                                const transform::Rigid3d& global_submap_pose,
                                const TrajectoryNodeData& constant_data, float min_score) const {
    return Run(0, global_node_pose, global_submap_pose, constant_data, min_score);
  }
  std::unique_ptr<Result> MatchFullSubmap(const transform::Quaterniond& global_node_rotation,
                                          const transform::Quaterniond& global_submap_rotation,
                                          const TrajectoryNodeData& constant_data,
                                          float min_score) const {
    return Run(1, transform::Rigid3d({{0., 0., 0.}}, global_node_rotation),
               transform::Rigid3d({{0., 0., 0.}}, global_submap_rotation), constant_data,
               min_score);
  }

  const csm_matcher3d* matcher() const { return matcher_; }  // for the batched ConstraintBuilder

 private:
  std::unique_ptr<Result> Run(int full, const transform::Rigid3d& node_pose,
                              const transform::Rigid3d& submap_pose,
                              const TrajectoryNodeData& data, float min_score) const {
    std::vector<float> hi, lo;
    const csm_node3d node = b200_internal::Node3D(data, &hi, &lo);
    double np[7], sp[7];
    b200_internal::Pose7(node_pose, np);
    b200_internal::Pose7(submap_pose, sp);
    csm_result3d r;
    if (!b200_internal::Check(csm_match3d(matcher_, &node, np, sp, full, min_score, &r, nullptr)))
      return nullptr;
    if (!r.found) return nullptr;  // fast_correlative_scan_matcher_3d.cc:197
    return std::unique_ptr<Result>(new Result{r.score, b200_internal::FromPose7(r.pose_estimate),
                                              r.rotational_score, r.low_resolution_score});
  }
  csm_matcher3d* matcher_ = nullptr;
};

// real_time_correlative_scan_matcher_3d.h:41-67.  The reference takes the HybridGrid per
// call; flattening + uploading a whole submap grid for every scan would dominate, so the
// grid lives in a DeviceHybridGrid that the caller refreshes when the submap changed
// (LocalTrajectoryBuilder3D matches against the active submap's high-resolution grid,
// internal/3d/local_trajectory_builder_3d.cc:139-148).
class DeviceHybridGrid {
 public:
  explicit DeviceHybridGrid(const HybridGrid& grid, int device = 0) {
    std::vector<int32_t> idx;
    std::vector<uint16_t> val;
    b200_internal::Flatten(grid, &idx, &val);
    b200_internal::Check(csm_grid3d_create(idx.data(), val.data(),
                                           static_cast<int64_t>(val.size()), grid.resolution(),
                                           device, &grid_));
  }
  // The grid of a fresh submap (HybridGrid(resolution)), filled by RangeDataInserter3D below.
  DeviceHybridGrid(float resolution, int device) {
    b200_internal::Check(csm_grid3d_create(nullptr, nullptr, 0, resolution, device, &grid_));
  }
  ~DeviceHybridGrid() { csm_grid3d_destroy(grid_); }
  DeviceHybridGrid(const DeviceHybridGrid&) = delete;
  DeviceHybridGrid& operator=(const DeviceHybridGrid&) = delete;
  const csm_grid3d* handle() const { return grid_; }
  csm_grid3d* mutable_handle() { return grid_; }
  // HybridGrid::ToProto (hybrid_grid.h:528-540, csm_grid3d_to_proto): what Submap3D::ToProto
  // writes for its high- and low-resolution grids.
  b200_internal::HybridGridProto ToProto() const {
    return b200_internal::Parse<b200_internal::HybridGridProto>(
        b200_internal::Serialize(csm_grid3d_to_proto, grid_));
  }
  // AddToTextureProto (mapping/3d/submap_3d.cc:146-176, csm_grid3d_to_texture): the texture
  // Submap3D::ToResponseProto adds for this grid with the global submap pose, the
  // high-resolution grid's first.
  void AddToTextureProto(const transform::Rigid3d& global_submap_pose,
                         b200_internal::SubmapTextureProto* texture) const {
    *texture = b200_internal::Parse<b200_internal::SubmapTextureProto>(
        b200_internal::DrawTexture(csm_grid3d_to_texture, grid_, global_submap_pose));
  }

 private:
  csm_grid3d* grid_ = nullptr;
};

inline FastCorrelativeScanMatcher3D::FastCorrelativeScanMatcher3D(
    const DeviceHybridGrid& hybrid_grid, const DeviceHybridGrid* low_resolution_hybrid_grid,
    const std::vector<float>* rotational_scan_matcher_histogram,
    const proto::FastCorrelativeScanMatcherOptions3D& options, int grid_size_in_voxels) {
  const csm_options3d o = b200_internal::Options3D(options);
  b200_internal::Check(csm_matcher3d_create_from_grid3d(
      hybrid_grid.handle(), grid_size_in_voxels, low_resolution_hybrid_grid->handle(),
      rotational_scan_matcher_histogram->data(),
      static_cast<int32_t>(rotational_scan_matcher_histogram->size()), &o, &matcher_));
}

// An IntensityHybridGrid resident on the device (csm_intensity_grid3d), for the intensity
// residual blocks of CeresScanMatcher3D (LocalTrajectoryBuilder3D passes the active submap's
// high-resolution intensity grid with use_intensities).
class DeviceIntensityGrid {
 public:
  explicit DeviceIntensityGrid(const IntensityHybridGrid& grid, int device = 0) {
    std::vector<int32_t> idx, count;
    std::vector<float> sum;
    for (const auto& v : grid.voxels()) {
      idx.push_back(v.x);
      idx.push_back(v.y);
      idx.push_back(v.z);
      sum.push_back(v.sum);
      count.push_back(v.count);
    }
    b200_internal::Check(csm_intensity_grid3d_create(idx.data(), sum.data(), count.data(),
                                                     static_cast<int64_t>(sum.size()),
                                                     grid.resolution(), device, &grid_));
  }
  // The intensity grid of a fresh submap (IntensityHybridGrid(resolution)).
  DeviceIntensityGrid(float resolution, int device) {
    b200_internal::Check(
        csm_intensity_grid3d_create(nullptr, nullptr, nullptr, 0, resolution, device, &grid_));
  }
  ~DeviceIntensityGrid() { csm_intensity_grid3d_destroy(grid_); }
  DeviceIntensityGrid(const DeviceIntensityGrid&) = delete;
  DeviceIntensityGrid& operator=(const DeviceIntensityGrid&) = delete;
  const csm_intensity_grid3d* handle() const { return grid_; }
  csm_intensity_grid3d* mutable_handle() { return grid_; }

 private:
  csm_intensity_grid3d* grid_ = nullptr;
};

// mapping/3d/range_data_inserter_3d.h:28-45 on device grids: Submap3D::InsertData
// (submap_3d.cc:271-290) keeps its submap's high-resolution, low-resolution and intensity
// grids as DeviceHybridGrid / DeviceIntensityGrid and inserts every scan in place, so the
// real-time matcher and CeresScanMatcher3D read the updated submap without a re-upload.
class RangeDataInserter3D {
 public:
  explicit RangeDataInserter3D(const mapping::proto::RangeDataInserterOptions3D& options,
                               int device = 0) {
    csm_range_inserter_options3d o;
    o.hit_probability = options.hit_probability();
    o.miss_probability = options.miss_probability();
    o.num_free_space_voxels = options.num_free_space_voxels();
    o.intensity_threshold = options.intensity_threshold();
    b200_internal::Check(csm_range_inserter3d_create(&o, device, &inserter_));
  }
  ~RangeDataInserter3D() { csm_range_inserter3d_destroy(inserter_); }
  RangeDataInserter3D(const RangeDataInserter3D&) = delete;
  RangeDataInserter3D& operator=(const RangeDataInserter3D&) = delete;

  // range_data_inserter_3d.cc:87-114; range_data in the grids' frame.
  void Insert(const sensor::RangeData& range_data, DeviceHybridGrid* hybrid_grid,
              DeviceIntensityGrid* intensity_hybrid_grid) const {
    if (hybrid_grid == nullptr) std::abort();  // CHECK_NOTNULL (:90)
    const std::vector<float> xyz = b200_internal::Flatten(range_data.returns);
    const float origin[3] = {range_data.origin.x(), range_data.origin.y(), range_data.origin.z()};
    const std::vector<float>& intensities = range_data.returns.intensities();
    b200_internal::Check(csm_range_inserter3d_insert(
        inserter_, origin, xyz.data(), intensities.empty() ? nullptr : intensities.data(),
        static_cast<int32_t>(range_data.returns.size()), hybrid_grid->mutable_handle(),
        intensity_hybrid_grid ? intensity_hybrid_grid->mutable_handle() : nullptr, nullptr));
  }

  // The grids of one submap that InsertSubmaps writes, in that submap's frame.
  struct SubmapGrids {
    transform::Rigid3d local_pose;
    DeviceHybridGrid* high_resolution_hybrid_grid;
    DeviceHybridGrid* low_resolution_hybrid_grid;
    DeviceIntensityGrid* high_resolution_intensity_hybrid_grid;   // null once forgotten
  };
  // Submap3D::InsertData's two inserts (submap_3d.cc:276-287) into each of `submaps`, in
  // order, with one call (csm_range_inserter3d_insert_submaps); range_data in the local frame.
  void InsertSubmaps(const sensor::RangeData& range_data, const std::vector<SubmapGrids>& submaps,
                     float high_resolution_max_range) const {
    std::vector<csm_submap_insert3d> entries(submaps.size());
    for (size_t i = 0; i < submaps.size(); ++i) {
      b200_internal::Pose7(submaps[i].local_pose, entries[i].local_pose);
      entries[i].high_resolution = submaps[i].high_resolution_hybrid_grid->mutable_handle();
      entries[i].low_resolution = submaps[i].low_resolution_hybrid_grid->mutable_handle();
      entries[i].intensity = submaps[i].high_resolution_intensity_hybrid_grid
                                 ? submaps[i].high_resolution_intensity_hybrid_grid->mutable_handle()
                                 : nullptr;
    }
    const std::vector<float> xyz = b200_internal::Flatten(range_data.returns);
    const float origin[3] = {range_data.origin.x(), range_data.origin.y(), range_data.origin.z()};
    const std::vector<float>& intensities = range_data.returns.intensities();
    b200_internal::Check(csm_range_inserter3d_insert_submaps(
        inserter_, entries.data(), static_cast<int32_t>(entries.size()), origin, xyz.data(),
        intensities.empty() ? nullptr : intensities.data(),
        static_cast<int32_t>(range_data.returns.size()), high_resolution_max_range, nullptr));
  }

 private:
  csm_range_inserter3d* inserter_ = nullptr;
};

class RealTimeCorrelativeScanMatcher3D {
 public:
  explicit RealTimeCorrelativeScanMatcher3D(
      const proto::RealTimeCorrelativeScanMatcherOptions& options)
      : options_(options) {}
  RealTimeCorrelativeScanMatcher3D(const RealTimeCorrelativeScanMatcher3D&) = delete;
  RealTimeCorrelativeScanMatcher3D& operator=(const RealTimeCorrelativeScanMatcher3D&) = delete;

  // The reference signature (grid per call: one upload per call).
  float Match(const transform::Rigid3d& initial_pose_estimate,
              const sensor::PointCloud& point_cloud, const HybridGrid& hybrid_grid,
              transform::Rigid3d* pose_estimate) const {
    const DeviceHybridGrid device_grid(hybrid_grid);
    return Match(initial_pose_estimate, point_cloud, device_grid, pose_estimate);
  }
  float Match(const transform::Rigid3d& initial_pose_estimate,
              const sensor::PointCloud& point_cloud, const DeviceHybridGrid& hybrid_grid,
              transform::Rigid3d* pose_estimate) const {
    if (pose_estimate == nullptr) std::abort();  // CHECK(:38)
    const std::vector<float> xyz = b200_internal::Flatten(point_cloud);
    double init[7];
    b200_internal::Pose7(initial_pose_estimate, init);
    float score = -1.f;
    double pose[7] = {0., 0., 0., 1., 0., 0., 0.};
    if (!b200_internal::Check(csm_rt_match3d(
            hybrid_grid.handle(), xyz.data(), static_cast<int32_t>(point_cloud.size()), init,
            options_.linear_search_window(), options_.angular_search_window(),
            options_.translation_delta_cost_weight(), options_.rotation_delta_cost_weight(),
            &score, pose, nullptr)))
      return -1.f;
    *pose_estimate = b200_internal::FromPose7(pose);
    return score;
  }

 private:
  const proto::RealTimeCorrelativeScanMatcherOptions options_;
};

// ceres_scan_matcher_3d.h:44-66; grids are device-resident handles.  A pair with an
// intensity grid adds its IntensityCostFunction3D block under HuberLoss (the constraint
// builder passes none, constraint_builder_3d.cc:265-275).  Summary: see
// CeresScanMatcher2D::Summary.
class CeresScanMatcher3D {
 public:
  using Summary = CeresScanMatcher2D::Summary;
  struct PointCloudAndDeviceGrid {
    const sensor::PointCloud* point_cloud;
    const DeviceHybridGrid* hybrid_grid;
    const DeviceIntensityGrid* intensity_hybrid_grid = nullptr;
  };
  struct Job {
    double target_translation[3];
    transform::Rigid3d initial_pose_estimate;
    std::vector<PointCloudAndDeviceGrid> point_clouds_and_hybrid_grids;   // 1 or 2
  };

  explicit CeresScanMatcher3D(const proto::CeresScanMatcherOptions3D& options)
      : options_(options) {}

  template <typename Vector3>
  void Match(const Vector3& target_translation, const transform::Rigid3d& initial_pose_estimate,
             const std::vector<PointCloudAndDeviceGrid>& point_clouds_and_hybrid_grids,
             transform::Rigid3d* const pose_estimate, Summary* const summary) const {
    std::vector<transform::Rigid3d> poses;
    std::vector<Summary> summaries;
    MatchBatch({Job{{target_translation.x(), target_translation.y(), target_translation.z()},
                    initial_pose_estimate, point_clouds_and_hybrid_grids}},
               &poses, &summaries);
    *pose_estimate = poses[0];
    if (summary != nullptr) *summary = summaries[0];
  }

  void MatchBatch(const std::vector<Job>& jobs, std::vector<transform::Rigid3d>* poses,
                  std::vector<Summary>* summaries) const {
    poses->clear();
    if (summaries != nullptr) summaries->clear();
    if (jobs.empty()) return;
    std::vector<std::vector<float>> xyz;
    xyz.reserve(2 * jobs.size());
    std::vector<csm_ceres_job3d> cj(jobs.size());
    std::vector<csm_ceres_intensity_job3d> cij(jobs.size(), csm_ceres_intensity_job3d{});
    bool any_intensity = false;
    for (size_t i = 0; i < jobs.size(); ++i) {
      const Job& job = jobs[i];
      if (job.point_clouds_and_hybrid_grids.empty() ||
          job.point_clouds_and_hybrid_grids.size() > 2)
        std::abort();  // CHECK_EQ(occupied_space_weight_size(), size) (:111-112)
      cj[i] = csm_ceres_job3d{};
      cj[i].num_clouds = static_cast<int32_t>(job.point_clouds_and_hybrid_grids.size());
      for (int b = 0; b < cj[i].num_clouds; ++b) {
        xyz.push_back(b200_internal::Flatten(*job.point_clouds_and_hybrid_grids[b].point_cloud));
        cj[i].grid[b] = job.point_clouds_and_hybrid_grids[b].hybrid_grid->handle();
        cj[i].xyz[b] = xyz.back().data();
        cj[i].num_points[b] =
            static_cast<int32_t>(job.point_clouds_and_hybrid_grids[b].point_cloud->size());
        const PointCloudAndDeviceGrid& pair = job.point_clouds_and_hybrid_grids[b];
        if (pair.intensity_hybrid_grid != nullptr) {
          if (pair.point_cloud->intensities().size() != pair.point_cloud->size())
            std::abort();  // the intensity block reads one intensity per point
          cij[i].intensity_grid[b] = pair.intensity_hybrid_grid->handle();
          cij[i].intensities[b] = pair.point_cloud->intensities().data();
          any_intensity = true;
        }
      }
      for (int k = 0; k < 3; ++k) cj[i].target_translation[k] = job.target_translation[k];
      b200_internal::Pose7(job.initial_pose_estimate, cj[i].initial_pose);
    }
    csm_ceres_options3d o{};
    o.occupied_space_weight[0] = options_.occupied_space_weight(0);
    o.occupied_space_weight[1] =
        options_.occupied_space_weight_size() > 1 ? options_.occupied_space_weight(1) : 1.;
    o.translation_weight = options_.translation_weight();
    o.rotation_weight = options_.rotation_weight();
    o.only_optimize_yaw = options_.only_optimize_yaw() ? 1 : 0;
    o.use_nonmonotonic_steps = options_.ceres_solver_options().use_nonmonotonic_steps() ? 1 : 0;
    o.max_num_iterations = options_.ceres_solver_options().max_num_iterations();
    std::vector<csm_ceres_result3d> res(jobs.size());
    if (any_intensity) {
      csm_ceres_intensity_options3d io{};
      for (int b = 0; b < 2; ++b) {
        const proto::IntensityCostFunctionOptions& ib =
            options_.intensity_cost_function_options(b);
        io.weight[b] = ib.weight();
        io.huber_scale[b] = ib.huber_scale();
        io.intensity_threshold[b] = ib.intensity_threshold();
      }
      b200_internal::Check(csm_ceres_match3d_intensity_batch(
          cj.data(), cij.data(), static_cast<int32_t>(cj.size()), &o, &io, res.data(), nullptr));
    } else {
      b200_internal::Check(csm_ceres_match3d_batch(cj.data(), static_cast<int32_t>(cj.size()),
                                                   &o, res.data(), nullptr));
    }
    for (const csm_ceres_result3d& r : res) {
      poses->push_back(b200_internal::FromPose7(r.pose_estimate));
      if (summaries != nullptr) {
        Summary s;
        s.initial_cost = r.initial_cost;
        s.final_cost = r.final_cost;
        s.iterations = r.iterations;
        s.num_successful_steps = r.num_successful_steps;
        s.termination = r.termination;
        summaries->push_back(s);
      }
    }
  }

 private:
  const proto::CeresScanMatcherOptions3D options_;
};
#endif  // !CSM_ADAPTER_REAL_CARTOGRAPHER

}  // namespace scan_matching
}  // namespace mapping
}  // namespace cartographer

#endif  // CSM_ADAPTER_SCAN_MATCHERS_B200_H_
