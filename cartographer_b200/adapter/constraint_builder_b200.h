// ConstraintBuilder2D / ConstraintBuilder3D with the reference's public surface
//   mapping/internal/constraints/constraint_builder_2d.h:60-107
//   mapping/internal/constraints/constraint_builder_3d.h:59-114
// over the batched C ABI.  The reference schedules one thread-pool task per
// (submap, node) pair (constraint_builder_2d.cc:97-111); here MaybeAdd*Constraint only
// records the pair (same gating: distance, per-submap FixedRatioSampler) and WhenDone
// schedules ONE task that drains the whole queue through csm_match2d_batch /
// csm_match3d_batch, builds the Constraints and runs the callback on the pool thread
// (RunWhenDoneCallback, :279-300).  Observable differences, all inside the contract of
// the header comment ("After all computations are done the callback will be called"):
//   * GetNumFinishedNodes() advances when the queue is drained, not pair by pair;
//   * constraint poses are the fast matcher's estimates unless the refinement of :245-249
//     is switched on: `set_device_refinement(true)` runs CeresScanMatcher2D::Match for all
//     found matches of the queue in one launch (csm_ceres_match2d_batch, with
//     options.ceres_scan_matcher_options()); `set_refiner` installs any other callable —
//     inside a checkout that can be the reference's own ceres_scan_matcher_.Match (2D / 3D
//     :261-275).
#ifndef CSM_ADAPTER_CONSTRAINT_BUILDER_B200_H_
#define CSM_ADAPTER_CONSTRAINT_BUILDER_B200_H_

#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "scan_matchers_b200.h"

namespace cartographer {
namespace mapping {
namespace constraints {

namespace b200_internal {
inline void Require(bool ok, const char* what) {  // glog CHECK semantics
  if (!ok) {
    std::fprintf(stderr, "ConstraintBuilder (b200): CHECK failed: %s\n", what);
    std::abort();
  }
}
// transform::Embed3D (transform/transform.h:104-110)
inline transform::Rigid3d Embed3D(const transform::Rigid2d& t) {
  const double half = 0.5 * t.rotation().angle();
  return transform::Rigid3d({{t.translation().x(), t.translation().y(), 0.}},
                            transform::Quaterniond{std::cos(half), 0., 0., std::sin(half)});
}
}  // namespace b200_internal

// A finished Submap2D whose grid lives on the device, as Submap2D::Finish leaves it when the
// submap was grown by scan_matching::ProbabilityGridRangeDataInserter2D and cropped with
// DeviceGrid2D::ComputeCroppedGrid: what ConstraintBuilder2D reads of it.  Unlike
// DeviceSubmap3D it is not limited to the stand-in build, because ConstraintBuilder2D is not.
// The builder keeps the pointer, so the grid must stay alive (and unchanged) until the
// WhenDone callback of every drain holding one of its pairs has run
// (constraint_builder_2d.h:76-77).  The stack is built from the grid and owns its levels:
// DeleteScanMatcher never touches the grid, and adding the submap again rebuilds the stack.
struct DeviceSubmap2D {
  const scan_matching::DeviceGrid2D* grid;   // the cropped ProbabilityGrid handle
  transform::Rigid2d local_pose_2d;          // ComputeSubmapPose(submap)
};

namespace b200_internal {
// What ConstraintBuilder2D and ConstraintBuilder3D share (constraint_builder_2d.cc:68-75,
// 139-163, 279-316): the queue of pairs, the per-submap FixedRatioSamplers and matchers, the
// node counters and the WhenDone cycle.  A builder gates a pair with Sample, queues it with Push
// and turns the whole queue into constraints in Match, which runs on the pool thread under the
// mutex; the callback runs after it, outside the lock.
template <typename Pending, typename SubmapMatcher>
class ConstraintQueue {
 public:
  using Constraint = PoseGraphInterface::Constraint;
  using Result = std::vector<Constraint>;

  virtual ~ConstraintQueue() {
    std::lock_guard<std::mutex> lock(mutex_);
    Require(pending_.empty(), "WhenDone() was not called");
    Require(num_started_nodes_ == num_finished_nodes_, "unfinished nodes");
    Require(when_done_ == nullptr, "callback still pending");
  }
  ConstraintQueue(const ConstraintQueue&) = delete;
  ConstraintQueue& operator=(const ConstraintQueue&) = delete;

  void NotifyEndOfNode() {  // :139-151
    std::lock_guard<std::mutex> lock(mutex_);
    ++num_started_nodes_;
  }

  // :153-163; `callback` runs in the thread pool after the queue has been drained.
  void WhenDone(const std::function<void(const Result&)>& callback) {
    {
      std::lock_guard<std::mutex> lock(mutex_);
      Require(when_done_ == nullptr, "WhenDone called twice");
      when_done_.reset(new std::function<void(const Result&)>(callback));
    }
    std::unique_ptr<common::Task> task(new common::Task);
    task->SetWorkItem([this] { Drain(); });
    thread_pool_->Schedule(std::move(task));
  }

  int GetNumFinishedNodes() {
    std::lock_guard<std::mutex> lock(mutex_);
    return num_finished_nodes_;
  }

  void DeleteScanMatcher(const SubmapId& submap_id) {  // :307-316
    std::lock_guard<std::mutex> lock(mutex_);
    matchers_.erase(submap_id);
    samplers_.erase(submap_id);
  }

 protected:
  ConstraintQueue(common::ThreadPoolInterface* thread_pool, double sampling_ratio)
      : thread_pool_(thread_pool), sampling_ratio_(sampling_ratio) {}

  // The per-submap FixedRatioSampler of a pair that passed the distance gate (:85-90).
  bool Sample(const SubmapId& submap_id) {
    std::lock_guard<std::mutex> lock(mutex_);
    return samplers_
        .emplace(std::piecewise_construct, std::forward_as_tuple(submap_id),
                 std::forward_as_tuple(sampling_ratio_))
        .first->second.Pulse();
  }
  void Push(const Pending& pending) {
    std::lock_guard<std::mutex> lock(mutex_);
    pending_.push_back(pending);
  }
  // The constraints of the queued pairs, in queue order.
  virtual Result Match(const std::deque<Pending>& pending) = 0;

  std::map<SubmapId, SubmapMatcher> matchers_;   // DispatchScanMatcherConstruction (:165-186)

 private:
  void Drain() {
    Result result;
    std::unique_ptr<std::function<void(const Result&)>> callback;
    {
      std::lock_guard<std::mutex> lock(mutex_);
      Require(when_done_ != nullptr, "no callback");
      result = Match(pending_);
      pending_.clear();
      num_finished_nodes_ = num_started_nodes_;
      callback = std::move(when_done_);
    }
    (*callback)(result);
  }

  common::ThreadPoolInterface* const thread_pool_;
  const double sampling_ratio_;
  std::mutex mutex_;
  std::unique_ptr<std::function<void(const Result&)>> when_done_;
  int num_started_nodes_ = 0;
  int num_finished_nodes_ = 0;
  std::deque<Pending> pending_;
  std::map<SubmapId, common::FixedRatioSampler> samplers_;
};

struct Pending2D {
  SubmapId submap_id;
  const Submap2D* submap;                 // one of the two is set
  const DeviceSubmap2D* device_submap;
  NodeId node_id;
  const TrajectoryNodeData* constant_data;
  transform::Rigid2d initial_pose;
  bool full;
  float min_score;
};
struct SubmapMatcher2D {
  std::unique_ptr<scan_matching::FastCorrelativeScanMatcher2D> matcher;
  // the refinement's upload of a host submap's grid; a device submap's is its own
  std::unique_ptr<scan_matching::DeviceGrid2D> device_grid;
};
}  // namespace b200_internal

class ConstraintBuilder2D
    : public b200_internal::ConstraintQueue<b200_internal::Pending2D,
                                            b200_internal::SubmapMatcher2D> {
 public:
  // (pose_estimate, point cloud, grid) -> refined pose; identity when unset.
  using Refiner = std::function<transform::Rigid2d(
      const transform::Rigid2d&, const sensor::PointCloud&, const Grid2D&)>;

  // `multi_gpu` (optional, csm_ctx_create): one process per GPU; every process must feed
  // the SAME sequence of MaybeAdd*Constraint / WhenDone calls.  The queue is then sharded
  // submap-major (a submap's stack only ever exists on its owner) and every process gets
  // the complete Result after one ncclAllGather inside csm_cb_batch2d_run.
  ConstraintBuilder2D(const proto::ConstraintBuilderOptions& options,
                      common::ThreadPoolInterface* thread_pool, int device = 0,
                      csm_ctx* multi_gpu = nullptr)
      : ConstraintQueue(thread_pool, options.sampling_ratio()),
        options_(options),
        device_(device),
        ctx_(multi_gpu) {
    if (ctx_ != nullptr)
      scan_matching::b200_internal::Check(csm_ctx_info(ctx_, &world_, &rank_, nullptr));
  }

  void set_refiner(const Refiner& refiner) { refiner_ = refiner; }
  // constraint_builder_2d.cc:245-249 on the device.  Single-GPU builders only: with a
  // multi_gpu context the results are exchanged inside csm_cb_batch2d_run, before a
  // refinement could run on the owner.
  void set_device_refinement(bool on) {
    b200_internal::Require(!on || ctx_ == nullptr, "device refinement needs a single-GPU builder");
    device_refinement_ = on;
  }

  // constraint_builder_2d.cc:77-112
  void MaybeAddConstraint(const SubmapId& submap_id, const Submap2D* submap,
                          const NodeId& node_id, const TrajectoryNodeData* constant_data,
                          const transform::Rigid2d& initial_relative_pose) {
    AddLocal(submap_id, submap, nullptr, node_id, constant_data, initial_relative_pose);
  }
  // The same for a submap kept on the device: its stack is built from the grid without a host
  // copy, and the refinement reads the grid directly.  The grid must be a ProbabilityGrid on
  // this builder's device, and the builder a single-GPU one.
  void MaybeAddConstraint(const SubmapId& submap_id, const DeviceSubmap2D* submap,
                          const NodeId& node_id, const TrajectoryNodeData* constant_data,
                          const transform::Rigid2d& initial_relative_pose) {
    RequireUsable(submap);
    AddLocal(submap_id, nullptr, submap, node_id, constant_data, initial_relative_pose);
  }

  // constraint_builder_2d.cc:114-137
  void MaybeAddGlobalConstraint(const SubmapId& submap_id, const Submap2D* submap,
                                const NodeId& node_id, const TrajectoryNodeData* constant_data) {
    AddGlobal(submap_id, submap, nullptr, node_id, constant_data);
  }
  void MaybeAddGlobalConstraint(const SubmapId& submap_id, const DeviceSubmap2D* submap,
                                const NodeId& node_id, const TrajectoryNodeData* constant_data) {
    RequireUsable(submap);
    AddGlobal(submap_id, nullptr, submap, node_id, constant_data);
  }

  // device counters of the last drained queue
  const csm_stats& last_stats() const { return last_stats_; }

 private:
  using Pending = b200_internal::Pending2D;

  // Refusals for a device submap, before anything is queued: its handle exists only in this
  // process and on the device it was made on, and only a ProbabilityGrid has a stack.
  void RequireUsable(const DeviceSubmap2D* submap) const {
    b200_internal::Require(submap != nullptr && submap->grid != nullptr, "grid");
    b200_internal::Require(ctx_ == nullptr, "device submaps need a single-GPU builder");
    b200_internal::Require(submap->grid->device() == device_,
                           "the device submap lives on another device than the builder");
    csm_rt_grid2d_info info;
    scan_matching::b200_internal::Check(
        csm_rt_grid2d_read(submap->grid->handle(), &info, nullptr, 0));
    b200_internal::Require(info.is_tsdf == 0, "device submaps must be ProbabilityGrids");
  }

  static const transform::Rigid2d& LocalPose(const Submap2D* submap,
                                             const DeviceSubmap2D* device_submap) {
    return device_submap != nullptr ? device_submap->local_pose_2d : submap->local_pose_2d();
  }

  void AddLocal(const SubmapId& submap_id, const Submap2D* submap,
                const DeviceSubmap2D* device_submap, const NodeId& node_id,
                const TrajectoryNodeData* constant_data,
                const transform::Rigid2d& initial_relative_pose) {
    if (initial_relative_pose.translation().norm() > options_.max_constraint_distance()) return;
    if (!Sample(submap_id)) return;
    // initial_pose = ComputeSubmapPose(*submap) * initial_relative_pose (:196-197)
    Queue(Pending{submap_id, submap, device_submap, node_id, constant_data,
                  LocalPose(submap, device_submap) * initial_relative_pose, false,
                  static_cast<float>(options_.min_score())});
  }

  void AddGlobal(const SubmapId& submap_id, const Submap2D* submap,
                 const DeviceSubmap2D* device_submap, const NodeId& node_id,
                 const TrajectoryNodeData* constant_data) {
    Queue(Pending{submap_id, submap, device_submap, node_id, constant_data,
                  transform::Rigid2d::Identity(), true,
                  static_cast<float>(options_.global_localization_min_score())});
  }

  void Queue(const Pending& p) {
    if (p.device_submap == nullptr)
      b200_internal::Require(p.submap != nullptr && p.submap->grid() != nullptr, "grid");  // :167
    Push(p);
  }

  // One matcher per submap, built once; a device submap's from its grid, device to device.
  const csm_stack2d* StackFor(const Pending& p) {
    std::unique_ptr<scan_matching::FastCorrelativeScanMatcher2D>& m =
        matchers_[p.submap_id].matcher;
    const auto& fo = options_.fast_correlative_scan_matcher_options();
    if (m == nullptr && p.device_submap != nullptr)
      m.reset(new scan_matching::FastCorrelativeScanMatcher2D(*p.device_submap->grid, fo));
    else if (m == nullptr)
      m.reset(new scan_matching::FastCorrelativeScanMatcher2D(*p.submap->grid(), fo, device_));
    return m->stack();
  }

  Result Match(const std::deque<Pending>& pending) override {
    if (refiner_) {   // Refiner takes a host Grid2D, which a device submap does not have
      for (const Pending& p : pending)
        b200_internal::Require(p.device_submap == nullptr,
                               "set_refiner cannot refine on a device submap");
    }
    const auto& fo = options_.fast_correlative_scan_matcher_options();
    // distinct stacks / clouds of this queue
    std::vector<const csm_stack2d*> stacks;
    std::vector<int32_t> owners;
    std::map<SubmapId, int> stack_index;
    std::vector<csm_cloud*> clouds;
    std::map<const TrajectoryNodeData*, int> cloud_index;
    std::vector<csm_job2d> jobs(pending.size());
    for (size_t i = 0; i < pending.size(); ++i) {
      const Pending& p = pending[i];
      auto si = stack_index.find(p.submap_id);
      if (si == stack_index.end()) {
        si = stack_index.emplace(p.submap_id, static_cast<int>(stacks.size())).first;
        const int owner = OwnerOf(p.submap_id);
        owners.push_back(owner);
        stacks.push_back(owner == rank_ ? StackFor(p) : nullptr);
      }
      auto ci = cloud_index.find(p.constant_data);
      if (ci == cloud_index.end()) {
        const sensor::PointCloud& pc = p.constant_data->filtered_gravity_aligned_point_cloud;
        const std::vector<float> xyz = scan_matching::b200_internal::Flatten(pc);
        csm_cloud* cloud = nullptr;
        scan_matching::b200_internal::Check(
            csm_cloud_create(xyz.data(), static_cast<int32_t>(pc.size()), device_, &cloud));
        ci = cloud_index.emplace(p.constant_data, static_cast<int>(clouds.size())).first;
        clouds.push_back(cloud);
      }
      csm_job2d& j = jobs[i];
      j = csm_job2d{};
      j.stack_index = si->second;
      j.cloud_index = ci->second;
      j.full_submap = p.full ? 1 : 0;
      j.initial_pose[0] = p.initial_pose.translation().x();
      j.initial_pose[1] = p.initial_pose.translation().y();
      j.initial_pose[2] = p.initial_pose.rotation().angle();
      j.min_score = p.min_score;
    }
    std::vector<csm_result2d> results(jobs.size());
    if (!jobs.empty()) {
      const auto run = [&](const csm_job2d* js, int32_t n, csm_result2d* rs) {
        const csm_cloud* const* cl = const_cast<const csm_cloud* const*>(clouds.data());
        if (ctx_ != nullptr)
          return csm_cb_batch2d_run(ctx_, stacks.data(), static_cast<int32_t>(stacks.size()), cl,
                                    static_cast<int32_t>(clouds.size()), js, n, owners.data(),
                                    fo.linear_search_window(), fo.angular_search_window(), rs,
                                    &last_stats_);
        return csm_match2d_batch(stacks.data(), static_cast<int32_t>(stacks.size()), cl,
                                 static_cast<int32_t>(clouds.size()), js, n,
                                 fo.linear_search_window(), fo.angular_search_window(), rs,
                                 &last_stats_);
      };
      if (!scan_matching::b200_internal::Check(
              run(jobs.data(), static_cast<int32_t>(jobs.size()), results.data()))) {
        // An engine capacity limit was hit somewhere in the batch: run the pairs one by
        // one; a pair that still exceeds it yields no constraint (the reference would
        // have produced a match or none — it never aborts here).
        for (size_t i = 0; i < jobs.size(); ++i) {
          results[i] = csm_result2d{};
          if (!scan_matching::b200_internal::Check(run(&jobs[i], 1, &results[i])))
            results[i].found = 0;
        }
      }
    }
    for (csm_cloud* c : clouds) csm_cloud_destroy(c);
    // ceres_scan_matcher_.Match(pose_estimate.translation(), pose_estimate, cloud, grid,
    // &pose_estimate, ...) for every found match (:245-249), one launch for the queue
    std::vector<transform::Rigid2d> refined;
    std::vector<size_t> refined_of(pending.size(), 0);
    if (device_refinement_) {
      std::vector<scan_matching::CeresScanMatcher2D::Job> rjobs;
      for (size_t i = 0; i < pending.size(); ++i) {
        if (!results[i].found) continue;
        const Pending& p = pending[i];
        const scan_matching::DeviceGrid2D* grid = nullptr;
        if (p.device_submap != nullptr) {   // the submap's own grid
          grid = p.device_submap->grid;
        } else {
          std::unique_ptr<scan_matching::DeviceGrid2D>& upload =
              matchers_[p.submap_id].device_grid;
          if (upload == nullptr)
            upload.reset(new scan_matching::DeviceGrid2D(*p.submap->grid(), device_));
          grid = upload.get();
        }
        refined_of[i] = rjobs.size();
        rjobs.push_back(scan_matching::CeresScanMatcher2D::Job{
            {results[i].pose_estimate[0], results[i].pose_estimate[1]},
            transform::Rigid2d({results[i].pose_estimate[0], results[i].pose_estimate[1]},
                               results[i].pose_estimate[2]),
            &p.constant_data->filtered_gravity_aligned_point_cloud, grid});
      }
      scan_matching::CeresScanMatcher2D(options_.ceres_scan_matcher_options(), device_)
          .MatchBatch(rjobs, &refined, nullptr);
    }
    Result result;
    for (size_t i = 0; i < pending.size(); ++i) {
      if (!results[i].found) continue;  // below min_score: no constraint (:253-261)
      const Pending& p = pending[i];
      transform::Rigid2d pose_estimate({results[i].pose_estimate[0], results[i].pose_estimate[1]},
                                       results[i].pose_estimate[2]);
      if (device_refinement_) pose_estimate = refined[refined_of[i]];
      if (refiner_)
        pose_estimate = refiner_(pose_estimate,
                                 p.constant_data->filtered_gravity_aligned_point_cloud,
                                 *p.submap->grid());
      // constraint_transform = ComputeSubmapPose(*submap).inverse() * pose_estimate (:251-252)
      const transform::Rigid2d constraint_transform =
          LocalPose(p.submap, p.device_submap).inverse() * pose_estimate;
      result.push_back(Constraint{p.submap_id,
                                  p.node_id,
                                  {b200_internal::Embed3D(constraint_transform),
                                   options_.loop_closure_translation_weight(),
                                   options_.loop_closure_rotation_weight()},
                                  Constraint::INTER_SUBMAP});
    }
    return result;
  }

  // submap-major ownership, stable across drains
  int OwnerOf(const SubmapId& id) const {
    return world_ <= 1 ? 0 : static_cast<int>((static_cast<unsigned>(id.trajectory_id) * 7919u +
                                               static_cast<unsigned>(id.submap_index)) %
                                              static_cast<unsigned>(world_));
  }

  const proto::ConstraintBuilderOptions options_;
  const int device_;
  csm_ctx* const ctx_;
  int32_t world_ = 1, rank_ = 0;
  Refiner refiner_;
  bool device_refinement_ = false;
  csm_stats last_stats_{};
};

#ifndef CSM_ADAPTER_REAL_CARTOGRAPHER
// A Submap3D whose grids live on the device, as Submap3D::InsertData leaves them when it
// inserts through scan_matching::RangeDataInserter3D: what ConstraintBuilder3D reads of it.
// The builder keeps the pointers, so the grids and the histogram must stay alive (and
// unchanged) until the WhenDone callback has run (constraint_builder_2d.h:76-77).
struct DeviceSubmap3D {
  const scan_matching::DeviceHybridGrid* high_resolution_hybrid_grid;
  const scan_matching::DeviceHybridGrid* low_resolution_hybrid_grid;
  const std::vector<float>* rotational_scan_matcher_histogram;
  int grid_size_in_voxels = 0;   // HybridGrid::grid_size(); 0 derives it from the grid
};

namespace b200_internal {
struct Pending3D {
  SubmapId submap_id;
  const Submap3D* submap;                 // one of the two is set
  const DeviceSubmap3D* device_submap;
  NodeId node_id;
  const TrajectoryNodeData* constant_data;
  transform::Rigid3d global_node_pose, global_submap_pose;
  bool full;
  float min_score;
};
struct SubmapMatcher3D {
  std::unique_ptr<scan_matching::FastCorrelativeScanMatcher3D> matcher;
  // the refinement's uploads of a host submap's high / low resolution grids
  std::unique_ptr<scan_matching::DeviceHybridGrid> high, low;
};
}  // namespace b200_internal

class ConstraintBuilder3D
    : public b200_internal::ConstraintQueue<b200_internal::Pending3D,
                                            b200_internal::SubmapMatcher3D> {
 public:
  ConstraintBuilder3D(const proto::ConstraintBuilderOptions& options,
                      common::ThreadPoolInterface* thread_pool, int device = 0)
      : ConstraintQueue(thread_pool, options.sampling_ratio()),
        options_(options),
        device_(device) {}

  // constraint_builder_3d.cc:265-275 on the device: every found match of a drained queue is
  // refined by CeresScanMatcher3D (options.ceres_scan_matcher_options_3d()) in one launch.
  void set_device_refinement(bool on) { device_refinement_ = on; }

  // constraint_builder_3d.cc:79-114
  void MaybeAddConstraint(const SubmapId& submap_id, const Submap3D* submap,
                          const NodeId& node_id, const TrajectoryNodeData* constant_data,
                          const transform::Rigid3d& global_node_pose,
                          const transform::Rigid3d& global_submap_pose) {
    AddLocal(submap_id, submap, nullptr, node_id, constant_data, global_node_pose,
             global_submap_pose);
  }
  // The same for a submap kept on the device: its matcher is built from its grids without a
  // host copy, and the refinement reads them directly.
  void MaybeAddConstraint(const SubmapId& submap_id, const DeviceSubmap3D* submap,
                          const NodeId& node_id, const TrajectoryNodeData* constant_data,
                          const transform::Rigid3d& global_node_pose,
                          const transform::Rigid3d& global_submap_pose) {
    AddLocal(submap_id, nullptr, submap, node_id, constant_data, global_node_pose,
             global_submap_pose);
  }

  // constraint_builder_3d.cc:116-142
  void MaybeAddGlobalConstraint(const SubmapId& submap_id, const Submap3D* submap,
                                const NodeId& node_id, const TrajectoryNodeData* constant_data,
                                const transform::Quaterniond& global_node_rotation,
                                const transform::Quaterniond& global_submap_rotation) {
    AddGlobal(submap_id, submap, nullptr, node_id, constant_data, global_node_rotation,
              global_submap_rotation);
  }
  void MaybeAddGlobalConstraint(const SubmapId& submap_id, const DeviceSubmap3D* submap,
                                const NodeId& node_id, const TrajectoryNodeData* constant_data,
                                const transform::Quaterniond& global_node_rotation,
                                const transform::Quaterniond& global_submap_rotation) {
    AddGlobal(submap_id, nullptr, submap, node_id, constant_data, global_node_rotation,
              global_submap_rotation);
  }

 private:
  using Pending = b200_internal::Pending3D;

  void AddLocal(const SubmapId& submap_id, const Submap3D* submap,
                const DeviceSubmap3D* device_submap, const NodeId& node_id,
                const TrajectoryNodeData* constant_data,
                const transform::Rigid3d& global_node_pose,
                const transform::Rigid3d& global_submap_pose) {
    // |(global_submap_pose^-1 * global_node_pose).translation()| = |t_node - t_submap|
    const double dx = global_node_pose.translation().x() - global_submap_pose.translation().x();
    const double dy = global_node_pose.translation().y() - global_submap_pose.translation().y();
    const double dz = global_node_pose.translation().z() - global_submap_pose.translation().z();
    if (std::sqrt(dx * dx + dy * dy + dz * dz) > options_.max_constraint_distance()) return;
    if (!Sample(submap_id)) return;
    Push(Pending{submap_id, submap, device_submap, node_id, constant_data, global_node_pose,
                 global_submap_pose, false, static_cast<float>(options_.min_score())});
  }

  void AddGlobal(const SubmapId& submap_id, const Submap3D* submap,
                 const DeviceSubmap3D* device_submap, const NodeId& node_id,
                 const TrajectoryNodeData* constant_data,
                 const transform::Quaterniond& global_node_rotation,
                 const transform::Quaterniond& global_submap_rotation) {
    Push(Pending{submap_id, submap, device_submap, node_id, constant_data,
                 transform::Rigid3d({{0., 0., 0.}}, global_node_rotation),
                 transform::Rigid3d({{0., 0., 0.}}, global_submap_rotation), true,
                 static_cast<float>(options_.global_localization_min_score())});
  }

  // One matcher per submap, built once (constraint_builder_3d.cc:172-198); a device submap's
  // from its grids, device to device.
  const csm_matcher3d* MatcherFor(const Pending& p) {
    std::unique_ptr<scan_matching::FastCorrelativeScanMatcher3D>& m =
        matchers_[p.submap_id].matcher;
    const auto& fo = options_.fast_correlative_scan_matcher_options_3d();
    if (m == nullptr && p.device_submap != nullptr) {
      const DeviceSubmap3D& d = *p.device_submap;
      m.reset(new scan_matching::FastCorrelativeScanMatcher3D(
          *d.high_resolution_hybrid_grid, d.low_resolution_hybrid_grid,
          d.rotational_scan_matcher_histogram, fo, d.grid_size_in_voxels));
    } else if (m == nullptr) {
      m.reset(new scan_matching::FastCorrelativeScanMatcher3D(
          p.submap->high_resolution_hybrid_grid(), &p.submap->low_resolution_hybrid_grid(),
          &p.submap->rotational_scan_matcher_histogram(), fo, device_));
    }
    return m->matcher();
  }

  Result Match(const std::deque<Pending>& pending) override {
    std::vector<const csm_matcher3d*> matchers;
    std::map<SubmapId, int> matcher_index;
    std::vector<csm_node3d> nodes;
    std::deque<std::vector<float>> buffers;  // keeps the flattened clouds alive
    std::map<const TrajectoryNodeData*, int> node_index;
    std::vector<csm_job3d> jobs(pending.size());
    for (size_t i = 0; i < pending.size(); ++i) {
      const Pending& p = pending[i];
      auto mi = matcher_index.find(p.submap_id);
      if (mi == matcher_index.end()) {
        mi = matcher_index.emplace(p.submap_id, static_cast<int>(matchers.size())).first;
        matchers.push_back(MatcherFor(p));
      }
      auto ni = node_index.find(p.constant_data);
      if (ni == node_index.end()) {
        buffers.emplace_back();
        std::vector<float>* high = &buffers.back();
        buffers.emplace_back();
        ni = node_index.emplace(p.constant_data, static_cast<int>(nodes.size())).first;
        nodes.push_back(
            scan_matching::b200_internal::Node3D(*p.constant_data, high, &buffers.back()));
      }
      csm_job3d& j = jobs[i];
      j.matcher_index = mi->second;
      j.node_index = ni->second;
      j.full_submap = p.full ? 1 : 0;
      j.min_score = p.min_score;
      scan_matching::b200_internal::Pose7(p.global_node_pose, j.global_node_pose);
      scan_matching::b200_internal::Pose7(p.global_submap_pose, j.global_submap_pose);
    }
    std::vector<csm_result3d> results(jobs.size());
    if (!jobs.empty()) {
      scan_matching::b200_internal::Check(csm_match3d_batch(
          matchers.data(), static_cast<int32_t>(matchers.size()), nodes.data(),
          static_cast<int32_t>(nodes.size()), jobs.data(), static_cast<int32_t>(jobs.size()),
          0, results.data(), nullptr));
    }
    // ceres_scan_matcher_.Match(pose_estimate.translation(), pose_estimate, {{high cloud,
    // high grid}, {low cloud, low grid}}, &constraint_transform, ...) for every found
    // match (constraint_builder_3d.cc:265-275), one launch for the queue
    std::vector<transform::Rigid3d> refined;
    std::vector<size_t> refined_of(pending.size(), 0);
    if (device_refinement_) {
      std::vector<scan_matching::CeresScanMatcher3D::Job> rjobs;
      for (size_t i = 0; i < pending.size(); ++i) {
        if (!results[i].found) continue;
        const Pending& p = pending[i];
        const scan_matching::DeviceHybridGrid* high;
        const scan_matching::DeviceHybridGrid* low;
        if (p.device_submap != nullptr) {   // the submap's own grids
          high = p.device_submap->high_resolution_hybrid_grid;
          low = p.device_submap->low_resolution_hybrid_grid;
        } else {
          b200_internal::SubmapMatcher3D& uploads = matchers_[p.submap_id];
          if (uploads.high == nullptr) {
            uploads.high.reset(new scan_matching::DeviceHybridGrid(
                p.submap->high_resolution_hybrid_grid(), device_));
            uploads.low.reset(new scan_matching::DeviceHybridGrid(
                p.submap->low_resolution_hybrid_grid(), device_));
          }
          high = uploads.high.get();
          low = uploads.low.get();
        }
        const csm_result3d& r = results[i];
        scan_matching::CeresScanMatcher3D::Job job;
        for (int k = 0; k < 3; ++k) job.target_translation[k] = r.pose_estimate[k];
        job.initial_pose_estimate = scan_matching::b200_internal::FromPose7(r.pose_estimate);
        job.point_clouds_and_hybrid_grids = {
            {&p.constant_data->high_resolution_point_cloud, high},
            {&p.constant_data->low_resolution_point_cloud, low}};
        refined_of[i] = rjobs.size();
        rjobs.push_back(job);
      }
      scan_matching::CeresScanMatcher3D(options_.ceres_scan_matcher_options_3d())
          .MatchBatch(rjobs, &refined, nullptr);
    }
    Result result;
    for (size_t i = 0; i < pending.size(); ++i) {
      const csm_result3d& r = results[i];
      if (!r.found) continue;
      // constraint_transform = the matcher's pose_estimate, refined when
      // set_device_refinement(true) (constraint_builder_3d.cc:261-275)
      const transform::Rigid3d pose_estimate =
          device_refinement_ ? refined[refined_of[i]]
                             : scan_matching::b200_internal::FromPose7(r.pose_estimate);
      result.push_back(Constraint{
          pending[i].submap_id,
          pending[i].node_id,
          {pose_estimate, options_.loop_closure_translation_weight(),
           options_.loop_closure_rotation_weight()},
          Constraint::INTER_SUBMAP});
    }
    return result;
  }

  const proto::ConstraintBuilderOptions options_;
  const int device_;
  bool device_refinement_ = false;
};
#endif  // !CSM_ADAPTER_REAL_CARTOGRAPHER

}  // namespace constraints

#ifndef CSM_ADAPTER_REAL_CARTOGRAPHER
// A ProbabilityGrid Submap2D (mapping/2d/submap_2d.h:37-71) whose grid lives on the device,
// filled by ActiveSubmaps2D below.  grid() is the active grid until Finish, then its crop;
// device_submap() is the view ConstraintBuilder2D reads of a finished submap.
class DeviceSubmap2D {
 public:
  DeviceSubmap2D(float origin_x, float origin_y, float resolution, int device)
      : local_pose_(transform::Rigid3d(
            {{static_cast<double>(origin_x), static_cast<double>(origin_y), 0.}},
            transform::Quaterniond{1., 0., 0., 0.})),   // Rigid3d::Translation
        grid_(new scan_matching::DeviceGrid2D(CreateGridLimits(origin_x, origin_y, resolution),
                                              device)),
        view_{nullptr, transform::Rigid2d({static_cast<double>(origin_x),
                                           static_cast<double>(origin_y)}, 0.)} {}
  DeviceSubmap2D(const DeviceSubmap2D&) = delete;
  DeviceSubmap2D& operator=(const DeviceSubmap2D&) = delete;

  const transform::Rigid3d& local_pose() const { return local_pose_; }
  int num_range_data() const { return num_range_data_; }
  bool insertion_finished() const { return insertion_finished_; }
  const scan_matching::DeviceGrid2D& grid() const { return *grid_; }
  // ConstraintBuilder2D's view: the cropped grid and ComputeSubmapPose's pose.
  const constraints::DeviceSubmap2D& device_submap() const {
    constraints::b200_internal::Require(insertion_finished_, "insertion_finished()");
    return view_;
  }

  // ActiveSubmaps2D::CreateGrid (submap_2d.cc:192-204): 100 x 100 cells with
  // max = origin.cast<double>() + 0.5 * 100 * resolution, resolution the float option.
  static MapLimits CreateGridLimits(float origin_x, float origin_y, float resolution) {
    constexpr int kInitialSubmapSize = 100;
    const double r = resolution;
    return MapLimits(r, static_cast<double>(origin_x) + 0.5 * kInitialSubmapSize * r,
                     static_cast<double>(origin_y) + 0.5 * kInitialSubmapSize * r,
                     CellLimits{kInitialSubmapSize, kInitialSubmapSize});
  }

 private:
  friend class ActiveSubmaps2D;
  // Submap2D::Finish (:146-151): grid_ = grid_->ComputeCroppedGrid(), which drops the
  // uncropped handle.
  void Finish() {
    constraints::b200_internal::Require(!insertion_finished_, "!insertion_finished()");
    grid_ = grid_->ComputeCroppedGrid();
    view_.grid = grid_.get();
    insertion_finished_ = true;
  }

  const transform::Rigid3d local_pose_;
  std::unique_ptr<scan_matching::DeviceGrid2D> grid_;
  constraints::DeviceSubmap2D view_;
  int num_range_data_ = 0;
  bool insertion_finished_ = false;
};

// ActiveSubmaps2D (submap_2d.cc:153-236) over device grids: each scan goes into the (at most
// two) active submaps with one csm_range_inserter2d_insert_submaps call.  ProbabilityGrid
// submaps only: a TSDF2D crop has no device form.  Submaps are shared, so one the pose graph
// still holds outlives its eviction.
class ActiveSubmaps2D {
 public:
  ActiveSubmaps2D(const proto::SubmapsOptions2D& options, int device = 0)
      : options_(Checked(options)),
        device_(device),
        range_data_inserter_(options.range_data_inserter_options()
                                 .probability_grid_range_data_inserter_options_2d(),
                             device) {}
  ActiveSubmaps2D(const ActiveSubmaps2D&) = delete;
  ActiveSubmaps2D& operator=(const ActiveSubmaps2D&) = delete;

  std::vector<std::shared_ptr<const DeviceSubmap2D>> InsertRangeData(
      const sensor::RangeData& range_data) {
    if (submaps_.empty() || submaps_.back()->num_range_data() == options_.num_range_data())
      AddSubmap(range_data.origin.x(), range_data.origin.y());
    std::vector<scan_matching::DeviceGrid2D*> grids;
    for (auto& submap : submaps_) {
      constraints::b200_internal::Require(!submap->insertion_finished(),
                                          "!insertion_finished()");
      grids.push_back(submap->grid_.get());
    }
    range_data_inserter_.InsertSubmaps(range_data, grids);
    for (auto& submap : submaps_) ++submap->num_range_data_;
    if (submaps_.front()->num_range_data() == 2 * options_.num_range_data())
      submaps_.front()->Finish();
    return submaps();
  }

  std::vector<std::shared_ptr<const DeviceSubmap2D>> submaps() const {
    return std::vector<std::shared_ptr<const DeviceSubmap2D>>(submaps_.begin(), submaps_.end());
  }

 private:
  // CreateSubmapsOptions2D's checks (submap_2d.cc:45-69), and the device's grid type
  static const proto::SubmapsOptions2D& Checked(const proto::SubmapsOptions2D& options) {
    constraints::b200_internal::Require(options.num_range_data() > 0,
                                        "num_range_data() > 0");
    constraints::b200_internal::Require(
        options.grid_options_2d().grid_type() == proto::GridOptions2D::PROBABILITY_GRID &&
            options.range_data_inserter_options().range_data_inserter_type() ==
                proto::RangeDataInserterOptions::PROBABILITY_GRID_INSERTER_2D,
        "ProbabilityGrid submaps (a TSDF2D crop has no device form)");
    return options;
  }
  void AddSubmap(float origin_x, float origin_y) {
    if (submaps_.size() >= 2) {
      constraints::b200_internal::Require(submaps_.front()->insertion_finished(),
                                          "submaps_.front()->insertion_finished()");
      submaps_.erase(submaps_.begin());
    }
    submaps_.emplace_back(new DeviceSubmap2D(origin_x, origin_y,
                                             options_.grid_options_2d().resolution(), device_));
  }

  const proto::SubmapsOptions2D options_;
  const int device_;
  scan_matching::ProbabilityGridRangeDataInserter2D range_data_inserter_;
  std::vector<std::shared_ptr<DeviceSubmap2D>> submaps_;
};

// A Submap3D (mapping/3d/submap_3d.h:47-103) whose grids live on the device, filled by
// ActiveSubmaps3D below.  device_submap() is the view ConstraintBuilder3D reads; the
// rotational scan matcher histogram is accumulated on the host.
class DeviceSubmap3D {
 public:
  DeviceSubmap3D(float high_resolution, float low_resolution,
                 const transform::Rigid3d& local_submap_pose, int histogram_size, int device)
      : local_pose_(local_submap_pose),
        high_(high_resolution, device),
        low_(low_resolution, device),
        intensity_(new scan_matching::DeviceIntensityGrid(high_resolution, device)),
        histogram_(histogram_size, 0.f),
        view_{&high_, &low_, &histogram_, 0} {}
  DeviceSubmap3D(const DeviceSubmap3D&) = delete;
  DeviceSubmap3D& operator=(const DeviceSubmap3D&) = delete;

  const transform::Rigid3d& local_pose() const { return local_pose_; }
  int num_range_data() const { return num_range_data_; }
  bool insertion_finished() const { return insertion_finished_; }
  const scan_matching::DeviceHybridGrid& high_resolution_hybrid_grid() const { return high_; }
  const scan_matching::DeviceHybridGrid& low_resolution_hybrid_grid() const { return low_; }
  const scan_matching::DeviceIntensityGrid* high_resolution_intensity_hybrid_grid() const {
    return intensity_.get();
  }
  const std::vector<float>& rotational_scan_matcher_histogram() const { return histogram_; }
  const constraints::DeviceSubmap3D& device_submap() const { return view_; }

 private:
  friend class ActiveSubmaps3D;
  scan_matching::RangeDataInserter3D::SubmapGrids grids() {
    return {local_pose_, &high_, &low_, intensity_.get()};
  }
  // submap_3d.cc:288-293, after the grids took the scan
  void Inserted(const transform::Quaterniond& local_from_gravity_aligned,
                const std::vector<float>& scan_histogram_in_gravity) {
    constraints::b200_internal::Require(!insertion_finished_, "!insertion_finished()");
    ++num_range_data_;
    const float yaw_in_submap_from_gravity = transform::GetYaw(
        local_pose_.inverse().rotation() * local_from_gravity_aligned);
    const std::vector<float> rotated = scan_matching::RotationalScanMatcher::RotateHistogram(
        scan_histogram_in_gravity, yaw_in_submap_from_gravity);
    for (size_t i = 0; i < histogram_.size(); ++i) histogram_[i] += rotated[i];
  }

  const transform::Rigid3d local_pose_;
  scan_matching::DeviceHybridGrid high_, low_;
  std::unique_ptr<scan_matching::DeviceIntensityGrid> intensity_;
  std::vector<float> histogram_;
  const constraints::DeviceSubmap3D view_;
  int num_range_data_ = 0;
  bool insertion_finished_ = false;
};

// ActiveSubmaps3D (submap_3d.cc:296-351) over device grids: each scan goes into the (at most
// two) active submaps with one csm_range_inserter3d_insert_submaps call.  Submaps are shared,
// so one the pose graph still holds outlives its eviction.
class ActiveSubmaps3D {
 public:
  ActiveSubmaps3D(const proto::SubmapsOptions3D& options, int device = 0)
      : options_(options),
        device_(device),
        range_data_inserter_(options.range_data_inserter_options(), device) {}
  ActiveSubmaps3D(const ActiveSubmaps3D&) = delete;
  ActiveSubmaps3D& operator=(const ActiveSubmaps3D&) = delete;

  std::vector<std::shared_ptr<const DeviceSubmap3D>> InsertData(
      const sensor::RangeData& range_data,
      const transform::Quaterniond& local_from_gravity_aligned,
      const std::vector<float>& rotational_scan_matcher_histogram_in_gravity) {
    if (submaps_.empty() || submaps_.back()->num_range_data() == options_.num_range_data()) {
      AddSubmap(transform::Rigid3d({{range_data.origin.x(), range_data.origin.y(),
                                     range_data.origin.z()}},
                                   local_from_gravity_aligned),
                static_cast<int>(rotational_scan_matcher_histogram_in_gravity.size()));
    }
    std::vector<scan_matching::RangeDataInserter3D::SubmapGrids> grids;
    for (auto& submap : submaps_) {
      constraints::b200_internal::Require(!submap->insertion_finished(),
                                          "!insertion_finished()");
      grids.push_back(submap->grids());
    }
    range_data_inserter_.InsertSubmaps(range_data, grids,
                                       static_cast<float>(options_.high_resolution_max_range()));
    for (auto& submap : submaps_)
      submap->Inserted(local_from_gravity_aligned, rotational_scan_matcher_histogram_in_gravity);
    if (submaps_.front()->num_range_data() == 2 * options_.num_range_data())
      submaps_.front()->insertion_finished_ = true;   // Submap3D::Finish
    return submaps();
  }

  std::vector<std::shared_ptr<const DeviceSubmap3D>> submaps() const {
    return std::vector<std::shared_ptr<const DeviceSubmap3D>>(submaps_.begin(), submaps_.end());
  }

 private:
  void AddSubmap(const transform::Rigid3d& local_submap_pose, int histogram_size) {
    if (submaps_.size() >= 2) {
      constraints::b200_internal::Require(submaps_.front()->insertion_finished(),
                                          "submaps_.front()->insertion_finished()");
      submaps_.front()->intensity_.reset();   // ForgetIntensityHybridGrid
      submaps_.erase(submaps_.begin());
    }
    submaps_.emplace_back(new DeviceSubmap3D(
        static_cast<float>(options_.high_resolution()),
        static_cast<float>(options_.low_resolution()), local_submap_pose, histogram_size,
        device_));
  }

  const proto::SubmapsOptions3D options_;
  const int device_;
  scan_matching::RangeDataInserter3D range_data_inserter_;
  std::vector<std::shared_ptr<DeviceSubmap3D>> submaps_;
};
#endif  // !CSM_ADAPTER_REAL_CARTOGRAPHER

}  // namespace mapping
}  // namespace cartographer

#endif  // CSM_ADAPTER_CONSTRAINT_BUILDER_B200_H_
