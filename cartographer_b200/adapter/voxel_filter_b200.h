// sensor::VoxelFilter (the four overloads) and sensor::AdaptiveVoxelFilter with the reference's
// signatures (sensor/internal/voxel_filter.h) over csm_voxel_filter_batch /
// csm_adaptive_voxel_filter_batch, on device 0 like the other adapter defaults.  The device
// returns the kept input indices, bit for bit those of the reference's reservoir sampling; the
// overloads gather their points and payloads (intensities, times, origin indices) from them.
// Replacing the bodies in voxel_filter.cc with these keeps CreateAdaptiveVoxelFilterOptions as
// it is (INTEGRATION.md §3).
#ifndef CSM_ADAPTER_VOXEL_FILTER_B200_H_
#define CSM_ADAPTER_VOXEL_FILTER_B200_H_

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../include/csm_abi.h"

#if defined(__has_include) && __has_include("cartographer/sensor/point_cloud.h")
#include "cartographer/sensor/point_cloud.h"
#include "cartographer/sensor/proto/adaptive_voxel_filter_options.pb.h"
#include "cartographer/sensor/timed_point_cloud_data.h"
#else
#include "compat.h"
#endif

namespace cartographer {
namespace sensor {

namespace b200_voxel_filter {

// The kept indices of one cloud, points given by position(i).  Refusals and CUDA failures keep
// the reference's CHECK semantics (abort with the ABI's message).
template <class Position>
std::vector<int32_t> KeptIndices(size_t n, Position&& position, float resolution,
                                 const proto::AdaptiveVoxelFilterOptions* options) {
  std::vector<float> xyz;
  xyz.reserve(3 * n);
  for (size_t i = 0; i < n; ++i) {
    const auto& p = position(i);
    xyz.push_back(p.x());
    xyz.push_back(p.y());
    xyz.push_back(p.z());
  }
  const float* clouds[1] = {xyz.data()};
  const int32_t num_points = static_cast<int32_t>(n);
  std::vector<int32_t> kept(n > 0 ? n : 1);
  int32_t num_kept = 0;
  csm_status s;
  if (options != nullptr) {
    const csm_adaptive_voxel_filter_options o = {options->max_length(),
                                                 static_cast<float>(options->min_num_points()),
                                                 options->max_range(), 0};
    s = csm_adaptive_voxel_filter_batch(clouds, &num_points, &o, 1, 0, kept.data(), &num_kept,
                                        nullptr);
  } else {
    s = csm_voxel_filter_batch(clouds, &num_points, &resolution, 1, 0, kept.data(), &num_kept,
                               nullptr);
  }
  if (s != CSM_OK) {
    std::fprintf(stderr, "libcsm_b200: %s\n", csm_last_error_string());
    std::abort();
  }
  kept.resize(num_kept);
  return kept;
}

template <class T>
std::vector<T> Gather(const std::vector<T>& in, const std::vector<int32_t>& kept) {
  std::vector<T> out;
  out.reserve(kept.size());
  for (int32_t i : kept) out.push_back(in[i]);
  return out;
}

// PointCloud: points, and intensities where present (voxel_filter.cc:141-161).
inline PointCloud GatherCloud(const PointCloud& cloud, const std::vector<int32_t>& kept) {
  std::vector<RangefinderPoint> points = Gather(cloud.points(), kept);
  std::vector<float> intensities;
  for (int32_t i : kept)
    if (static_cast<size_t>(i) < cloud.intensities().size())
      intensities.push_back(cloud.intensities()[i]);
  return PointCloud(std::move(points), std::move(intensities));
}

}  // namespace b200_voxel_filter

inline std::vector<RangefinderPoint> VoxelFilter(const std::vector<RangefinderPoint>& points,
                                                 const float resolution) {
  return b200_voxel_filter::Gather(
      points, b200_voxel_filter::KeptIndices(
                  points.size(), [&](size_t i) { return points[i].position; }, resolution,
                  nullptr));
}

inline PointCloud VoxelFilter(const PointCloud& point_cloud, const float resolution) {
  const auto& points = point_cloud.points();
  return b200_voxel_filter::GatherCloud(
      point_cloud, b200_voxel_filter::KeptIndices(
                       points.size(), [&](size_t i) { return points[i].position; }, resolution,
                       nullptr));
}

inline TimedPointCloud VoxelFilter(const TimedPointCloud& timed_point_cloud,
                                   const float resolution) {
  return b200_voxel_filter::Gather(
      timed_point_cloud,
      b200_voxel_filter::KeptIndices(
          timed_point_cloud.size(), [&](size_t i) { return timed_point_cloud[i].position; },
          resolution, nullptr));
}

inline std::vector<TimedPointCloudOriginData::RangeMeasurement> VoxelFilter(
    const std::vector<TimedPointCloudOriginData::RangeMeasurement>& range_measurements,
    const float resolution) {
  return b200_voxel_filter::Gather(
      range_measurements,
      b200_voxel_filter::KeptIndices(
          range_measurements.size(),
          [&](size_t i) { return range_measurements[i].point_time.position; }, resolution,
          nullptr));
}

inline PointCloud AdaptiveVoxelFilter(const PointCloud& point_cloud,
                                      const proto::AdaptiveVoxelFilterOptions& options) {
  const auto& points = point_cloud.points();
  return b200_voxel_filter::GatherCloud(
      point_cloud, b200_voxel_filter::KeptIndices(
                       points.size(), [&](size_t i) { return points[i].position; }, 0.f,
                       &options));
}

}  // namespace sensor
}  // namespace cartographer

#endif  // CSM_ADAPTER_VOXEL_FILTER_B200_H_
