// OverlappingSubmapsTrimmer2D (mapping/internal/2d/overlapping_submaps_trimmer_2d.h) over submaps
// whose grids live on the device: the coverage pass (AddSubmapsToSubmapCoverageGrid2D and
// FindSubmapIdsToTrim) is csm_trim_overlapping_submaps2d; the rest of Trim (:186-210) is restated
// here around it: the early return, ComputeSubmapFreshness, the first submap's limits, the uint16
// conversions and the TrimSubmap calls in SubmapId order.
#ifndef CSM_ADAPTER_POSE_GRAPH_TRIMMER_B200_H_
#define CSM_ADAPTER_POSE_GRAPH_TRIMMER_B200_H_

#include <algorithm>
#include <cstdint>
#include <functional>
#include <map>
#include <vector>

#include "scan_matchers_b200.h"

namespace cartographer {
namespace mapping {

class OverlappingSubmapsTrimmer2D : public PoseGraphTrimmer {
 public:
  // The submap's device grid, which the checkout keeps in place of the host Grid2D: for a
  // finished submap its cropped grid (ComputeCroppedGrid at Submap2D::Finish), for an unfinished
  // one the active, uncropped grid.  Trim asks for the first submap's grid whether or not it is
  // finished, as the reference takes its limits from submap_data.begin(), and reads only its
  // limits; the coverage pass asks only for finished submaps.
  using DeviceGridOf =
      std::function<const scan_matching::DeviceGrid2D&(const SubmapId&, const Submap2D&)>;

  OverlappingSubmapsTrimmer2D(uint16_t fresh_submaps_count, double min_covered_area,
                              uint16_t min_added_submaps_count, DeviceGridOf device_grid)
      : fresh_submaps_count_(fresh_submaps_count),
        min_covered_area_(min_covered_area),
        min_added_submaps_count_(min_added_submaps_count),
        device_grid_(std::move(device_grid)) {}
  ~OverlappingSubmapsTrimmer2D() override = default;

  void Trim(Trimmable* pose_graph) override {
    const auto submap_data = pose_graph->GetOptimizedSubmapData();
    if (submap_data.size() - current_submap_count_ <= min_added_submaps_count_) return;
    // first_submap_map_limits (:192-195), read without a stream synchronisation
    const auto& first = *submap_data.begin();
    const scan_matching::DeviceGrid2D& first_grid = device_grid_(first.id, *first.data.submap);
    double resolution = 0., max_x = 0., max_y = 0.;
    scan_matching::b200_internal::Check(csm_rt_grid2d_limits(first_grid.handle(), &resolution,
                                                             &max_x, &max_y, nullptr, nullptr));
    const std::map<SubmapId, int64_t> freshness = ComputeSubmapFreshness(
        submap_data, pose_graph->GetTrajectoryNodes(), pose_graph->GetConstraints());
    std::vector<SubmapId> ids;
    std::vector<csm_coverage_submap2d> records;
    for (const auto& submap : submap_data) {
      const auto it = freshness.find(submap.id);
      if (it == freshness.end() || !submap.data.submap->insertion_finished()) continue;
      const transform::Rigid3d global_frame_from_local_frame =
          submap.data.pose * submap.data.submap->local_pose().inverse();
      csm_coverage_submap2d r;
      r.grid = device_grid_(submap.id, *submap.data.submap).handle();
      const auto& t = global_frame_from_local_frame.translation();
      const auto& q = global_frame_from_local_frame.rotation();
      r.translation[0] = t.x();
      r.translation[1] = t.y();
      r.translation[2] = t.z();
      r.rotation[0] = q.w();
      r.rotation[1] = q.x();
      r.rotation[2] = q.y();
      r.rotation[3] = q.z();
      r.freshness = it->second;
      ids.push_back(submap.id);
      records.push_back(r);
    }
    // the reference passes this double to a uint16 parameter
    const uint16_t min_covered_cells_count =
        static_cast<uint16_t>(min_covered_area_ / (resolution * resolution));
    std::vector<uint8_t> trim(ids.size());
    std::vector<uint32_t> covered(ids.size());
    scan_matching::b200_internal::Check(csm_trim_overlapping_submaps2d(
        records.data(), static_cast<int32_t>(records.size()), max_x, max_y, resolution,
        fresh_submaps_count_, min_covered_cells_count, trim.data(),
        covered.data(), &last_stats_));
    std::vector<SubmapId> submap_ids_to_remove;
    for (size_t i = 0; i < ids.size(); ++i)
      if (trim[i]) submap_ids_to_remove.push_back(ids[i]);
    current_submap_count_ = submap_data.size() - submap_ids_to_remove.size();
    for (const SubmapId& id : submap_ids_to_remove) pose_graph->TrimSubmap(id);
  }
  bool IsFinished() override { return finished_; }

  // The device call's stats of the last Trim that reached it.
  const csm_coverage_stats2d& last_stats() const { return last_stats_; }

 private:
  // :105-143: the time of the largest NodeId per submap over INTRA_SUBMAP constraints.
  static std::map<SubmapId, int64_t> ComputeSubmapFreshness(
      const MapById<SubmapId, PoseGraphInterface::SubmapData>& submap_data,
      const MapById<NodeId, TrajectoryNode>& trajectory_nodes,
      const std::vector<PoseGraphInterface::Constraint>& constraints) {
    std::map<SubmapId, NodeId> submap_to_latest_node;
    for (const PoseGraphInterface::Constraint& constraint : constraints) {
      if (constraint.tag != PoseGraphInterface::Constraint::INTRA_SUBMAP) continue;
      auto it = submap_to_latest_node.find(constraint.submap_id);
      if (it == submap_to_latest_node.end()) {
        submap_to_latest_node.emplace(constraint.submap_id, constraint.node_id);
        continue;
      }
      it->second = std::max(it->second, constraint.node_id);
    }
    std::map<SubmapId, int64_t> freshness;
    for (const auto& submap_and_node : submap_to_latest_node) {
      if (!submap_data.Contains(submap_and_node.first)) continue;
      if (!trajectory_nodes.Contains(submap_and_node.second)) continue;
      freshness[submap_and_node.first] =
          trajectory_nodes.at(submap_and_node.second).time().time_since_epoch().count();
    }
    return freshness;
  }

  const uint16_t fresh_submaps_count_;
  const double min_covered_area_;
  const uint16_t min_added_submaps_count_;
  const DeviceGridOf device_grid_;
  uint16_t current_submap_count_ = 0;
  bool finished_ = false;
  csm_coverage_stats2d last_stats_{};
};

}  // namespace mapping
}  // namespace cartographer

#endif  // CSM_ADAPTER_POSE_GRAPH_TRIMMER_B200_H_
