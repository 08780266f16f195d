// Compiles the drop-in adapter classes against the stand-in headers and links
// them to libcsm_b200.so.  With a GPU it runs one match through the reference-
// shaped C++ API; without one it only checks that the ABI reports CSM_E_CUDA
// (no CPU fallback) — either way the binary proves the adapter builds and links.
#include <cmath>
#include <cstdio>
#include <cstring>

#include "constraint_builder_b200.h"
#include "scan_matchers_b200.h"

using namespace cartographer;

// RESULT lines are parsed by tests/test_gpu_adapter.py and compared with the oracle:
// float scores as their bit patterns, doubles with 17 significant digits.
static unsigned Bits(float f) {
  unsigned u;
  std::memcpy(&u, &f, 4);
  return u;
}

// Host-only part (runs everywhere): the builder's gating and WhenDone cycle when no
// pair survives the gates — nothing reaches the device — and the sampler's sequence
// (common/fixed_ratio_sampler_test.cc).
static int HostOnlyChecks() {
  using mapping::constraints::ConstraintBuilder2D;
  common::FixedRatioSampler half(0.5);
  const bool want[6] = {true, false, true, false, true, false};
  for (bool w : want)
    if (half.Pulse() != w) return 1;
  mapping::constraints::proto::ConstraintBuilderOptions bo;
  bo.sampling_ratio_ = 1.0;
  bo.max_constraint_distance_ = 1.0;
  common::InlineThreadPool pool;
  ConstraintBuilder2D builder(bo, &pool);
  const std::vector<uint16_t> cells(16, 0);
  mapping::Grid2D grid(mapping::MapLimits(0.05, 0.2, 0.2, mapping::CellLimits{4, 4}), 0.1f, 0.9f,
                       cells);
  mapping::Submap2D submap(&grid, transform::Rigid2d());
  mapping::TrajectoryNodeData node;
  builder.MaybeAddConstraint(mapping::SubmapId{0, 0}, &submap, mapping::NodeId{0, 0}, &node,
                             transform::Rigid2d({5., 0.}, 0.));  // beyond max_constraint_distance
  builder.NotifyEndOfNode();
  int calls = 0;
  size_t constraints = 99;
  builder.WhenDone([&](const ConstraintBuilder2D::Result& r) { ++calls; constraints = r.size(); });
  if (calls != 1 || constraints != 0 || builder.GetNumFinishedNodes() != 1) return 1;
  // Rigid2d algebra used for the constraint transform
  const transform::Rigid2d a({1., 2.}, 0.3);
  const transform::Rigid2d id = a.inverse() * a;
  if (std::fabs(id.translation().x()) > 1e-12 || std::fabs(id.translation().y()) > 1e-12 ||
      std::fabs(id.rotation().angle()) > 1e-12)
    return 1;
  std::printf("adapter_selftest: host-only checks passed\n");
  return 0;
}

int main() {
  if (HostOnlyChecks() != 0) {
    std::printf("adapter_selftest: host-only checks FAILED\n");
    return 1;
  }
  int32_t devices = 0;
  if (csm_device_count(&devices) != CSM_OK || devices == 0) {
    std::printf("adapter_selftest: no CUDA device (%s) — link check only\n",
                csm_last_error_string());
    return 0;
  }
  const int n = 120;
  std::vector<uint16_t> cells(n * n, 0);
  for (int i = 20; i < 100; ++i) {  // an L-shaped wall, p ~ 0.8
    cells[40 * n + i] = 5000;
    cells[i * n + 30] = 5000;
  }
  mapping::Grid2D grid(mapping::MapLimits(0.05, 3.0, 3.0, mapping::CellLimits{n, n}), 0.1f, 0.9f,
                       cells);
  mapping::scan_matching::proto::FastCorrelativeScanMatcherOptions2D options;
  options.set_linear_search_window(1.0);
  options.set_angular_search_window(0.3);
  options.set_branch_and_bound_depth(4);
  mapping::scan_matching::FastCorrelativeScanMatcher2D matcher(grid, options);
  sensor::PointCloud cloud;
  for (int i = 20; i < 100; i += 2) {
    // world coordinates of the wall cells: x = max_x - (cy + .5) res, y = max_y - (cx + .5) res
    cloud.push_back({{{float(3.0 - (40 + 0.5) * 0.05), float(3.0 - (i + 0.5) * 0.05), 0.f}}});
    cloud.push_back({{{float(3.0 - (i + 0.5) * 0.05), float(3.0 - (30 + 0.5) * 0.05), 0.f}}});
  }
  float score = 0.f;
  transform::Rigid2d pose;
  const bool found = matcher.Match(transform::Rigid2d({0.2, -0.15}, 0.05), cloud, 0.5f, &score, &pose);
  std::printf("adapter_selftest: found=%d score=%.4f pose=(%.3f, %.3f, %.4f)\n", found, score,
              pose.translation().x(), pose.translation().y(), pose.rotation().angle());
  std::printf("RESULT fast2d %d %08x %.17g %.17g %.17g\n", found ? 1 : 0, Bits(score),
              pose.translation().x(), pose.translation().y(), pose.rotation().angle());
  if (!found || std::fabs(pose.translation().x()) > 0.051 || std::fabs(pose.translation().y()) > 0.051)
    return 1;
  {
    float score_f = 0.f;
    transform::Rigid2d pose_f;
    const bool found_f = matcher.MatchFullSubmap(cloud, 0.5f, &score_f, &pose_f);
    std::printf("RESULT fast2d_full %d %08x %.17g %.17g %.17g\n", found_f ? 1 : 0, Bits(score_f),
                pose_f.translation().x(), pose_f.translation().y(), pose_f.rotation().angle());
  }
  // ---- RealTimeCorrelativeScanMatcher2D: Match and the public ScoreCandidates ----
  {
    mapping::scan_matching::proto::RealTimeCorrelativeScanMatcherOptions ro;
    ro.set_linear_search_window(0.1);
    ro.set_angular_search_window(0.1);
    ro.set_translation_delta_cost_weight(0.1);
    ro.set_rotation_delta_cost_weight(0.1);
    mapping::scan_matching::RealTimeCorrelativeScanMatcher2D rt(ro);
    transform::Rigid2d rt_pose;
    const double rt_score = rt.Match(transform::Rigid2d({0.06, -0.04}, 0.02), cloud, grid, &rt_pose);
    std::printf("RESULT rt2d %08x %.17g %.17g %.17g\n", Bits(static_cast<float>(rt_score)),
                rt_pose.translation().x(), rt_pose.translation().y(), rt_pose.rotation().angle());
    if (std::fabs(rt_pose.translation().x()) > 0.051 || std::fabs(rt_pose.translation().y()) > 0.051)
      return 1;
    // three candidates on one un-rotated discrete scan (cells of the wall points themselves)
    const mapping::scan_matching::SearchParameters sp(2, 0, 0.01, 0.05);
    mapping::scan_matching::DiscreteScan2D scan;
    for (int i = 20; i < 100; i += 2) {
      scan.push_back(mapping::scan_matching::Array2i{{i, 40}});
      scan.push_back(mapping::scan_matching::Array2i{{30, i}});
    }
    std::vector<mapping::scan_matching::Candidate2D> cands;
    cands.emplace_back(0, 0, 0, sp);
    cands.emplace_back(0, 1, 0, sp);
    cands.emplace_back(0, -2, 2, sp);
    rt.ScoreCandidates(grid, {scan}, sp, &cands);
    std::printf("RESULT rt2d_candidates %08x %08x %08x\n", Bits(cands[0].score),
                Bits(cands[1].score), Bits(cands[2].score));
    if (!(cands[0].score > cands[1].score && cands[1].score > cands[2].score)) return 1;
  }

  // ---- 3D: the reference's 12-point axis cloud inserted at a known pose ----
  mapping::HybridGrid hybrid(0.05f);
  sensor::PointCloud cloud3;
  const float tx = 0.2f, ty = -0.15f, tz = 0.1f;
  for (int axis = 0; axis < 3; ++axis)
    for (float d = 4.f; d <= 5.5f; d += 0.5f) {
      float p[3] = {0.f, 0.f, 0.f};
      p[axis] = d;
      cloud3.push_back({{{p[0], p[1], p[2]}}});
      hybrid.Set(static_cast<int>(std::lround((p[0] + tx) / 0.05f)),
                 static_cast<int>(std::lround((p[1] + ty) / 0.05f)),
                 static_cast<int>(std::lround((p[2] + tz) / 0.05f)), 24575 /* p ~ 0.7 */);
    }
  mapping::scan_matching::proto::FastCorrelativeScanMatcherOptions3D o3;
  o3.o.branch_and_bound_depth = 6;
  o3.o.full_resolution_depth = 6;
  o3.o.min_rotational_score = 0.1;
  o3.o.min_low_resolution_score = 0.15;
  o3.o.linear_xy_search_window = 0.8;
  o3.o.linear_z_search_window = 0.8;
  o3.o.angular_search_window = 0.3;
  const std::vector<float> histogram(10, 0.f);
  mapping::scan_matching::FastCorrelativeScanMatcher3D matcher3(hybrid, &hybrid, &histogram, o3);
  mapping::TrajectoryNodeData data;
  data.high_resolution_point_cloud = cloud3;
  data.low_resolution_point_cloud = cloud3;
  data.rotational_scan_matcher_histogram = histogram;
  const auto result = matcher3.Match(transform::Rigid3d(), transform::Rigid3d(), data, 0.1f);
  if (!result) { std::printf("adapter_selftest: 3D match failed\n"); return 1; }
  std::printf("adapter_selftest: 3D score=%.4f t=(%.3f, %.3f, %.3f) low=%.3f\n", result->score,
              result->pose_estimate.translation().x(), result->pose_estimate.translation().y(),
              result->pose_estimate.translation().z(), result->low_resolution_score);
  std::printf("RESULT fast3d %08x %.17g %.17g %.17g %.17g %.17g %.17g %.17g %08x %08x\n",
              Bits(result->score), result->pose_estimate.translation().x(),
              result->pose_estimate.translation().y(), result->pose_estimate.translation().z(),
              result->pose_estimate.rotation().w(), result->pose_estimate.rotation().x(),
              result->pose_estimate.rotation().y(), result->pose_estimate.rotation().z(),
              Bits(result->rotational_score), Bits(result->low_resolution_score));
  if (std::fabs(result->pose_estimate.translation().x() - tx) > 0.051 ||
      std::fabs(result->pose_estimate.translation().y() - ty) > 0.051 ||
      std::fabs(result->pose_estimate.translation().z() - tz) > 0.051)
    return 1;
  // ---- RealTimeCorrelativeScanMatcher3D on the same grid ----
  {
    mapping::scan_matching::proto::RealTimeCorrelativeScanMatcherOptions ro;
    ro.set_linear_search_window(0.1);
    ro.set_angular_search_window(0.01);
    ro.set_translation_delta_cost_weight(0.1);
    ro.set_rotation_delta_cost_weight(1.0);
    mapping::scan_matching::RealTimeCorrelativeScanMatcher3D rt3(ro);
    transform::Rigid3d pose3;
    const float s3 = rt3.Match(transform::Rigid3d({{0.25, -0.1, 0.05}}, transform::Quaterniond{1., 0., 0., 0.}),
                               cloud3, hybrid, &pose3);
    std::printf("RESULT rt3d %08x %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", Bits(s3),
                pose3.translation().x(), pose3.translation().y(), pose3.translation().z(),
                pose3.rotation().w(), pose3.rotation().x(), pose3.rotation().y(),
                pose3.rotation().z());
    if (std::fabs(pose3.translation().x() - tx) > 0.051 ||
        std::fabs(pose3.translation().y() - ty) > 0.051 ||
        std::fabs(pose3.translation().z() - tz) > 0.051)
      return 1;
  }

  // ---- ConstraintBuilder2D / 3D: the reference's call cycle (constraint_builder_2d_test.cc:58-112) ----
  {
    using mapping::constraints::ConstraintBuilder2D;
    mapping::constraints::proto::ConstraintBuilderOptions bo;
    bo.sampling_ratio_ = 1.0;
    bo.max_constraint_distance_ = 10.0;
    bo.min_score_ = 0.5;
    bo.global_localization_min_score_ = 0.4;
    bo.fast2d_ = options;
    common::InlineThreadPool pool;
    ConstraintBuilder2D builder(bo, &pool);
    const transform::Rigid2d submap_pose({0.1, -0.05}, 0.02);
    mapping::Submap2D submap(&grid, submap_pose);
    mapping::TrajectoryNodeData node;
    node.filtered_gravity_aligned_point_cloud = cloud;
    const mapping::SubmapId sid{0, 0};
    // initial pose (map <- node) = submap_pose * relative; ask for the same start as above
    const transform::Rigid2d relative = submap_pose.inverse() * transform::Rigid2d({0.2, -0.15}, 0.05);
    builder.MaybeAddConstraint(sid, &submap, mapping::NodeId{0, 0}, &node, relative);
    builder.MaybeAddConstraint(sid, &submap, mapping::NodeId{0, 1}, &node,
                               transform::Rigid2d({100., 0.}, 0.));  // beyond max distance: skipped
    builder.MaybeAddGlobalConstraint(sid, &submap, mapping::NodeId{0, 2}, &node);
    builder.NotifyEndOfNode();
    int calls = 0;
    ConstraintBuilder2D::Result got;
    builder.WhenDone([&](const ConstraintBuilder2D::Result& r) { ++calls; got = r; });
    std::printf("adapter_selftest: ConstraintBuilder2D %d callback(s), %zu constraints, finished nodes %d, %lld candidates\n",
                calls, got.size(), builder.GetNumFinishedNodes(),
                static_cast<long long>(builder.last_stats().candidates_scored));
    if (calls != 1 || got.size() != 2 || builder.GetNumFinishedNodes() != 1) return 1;
    for (const auto& c : got)
      std::printf("RESULT cb2d %d %.17g %.17g %.17g\n", c.node_id.node_index,
                  c.pose.zbar_ij.translation().x(), c.pose.zbar_ij.translation().y(),
                  2. * std::atan2(c.pose.zbar_ij.rotation().z(), c.pose.zbar_ij.rotation().w()));
    for (const auto& c : got) {
      // zbar_ij = submap_pose^-1 * pose_estimate, pose_estimate ~ identity
      const transform::Rigid2d want = submap_pose.inverse();
      if (c.tag != ConstraintBuilder2D::Constraint::INTER_SUBMAP ||
          std::fabs(c.pose.zbar_ij.translation().x() - want.translation().x()) > 0.051 ||
          std::fabs(c.pose.zbar_ij.translation().y() - want.translation().y()) > 0.051)
        return 1;
    }
    if (got[0].node_id.node_index != 0 || got[1].node_id.node_index != 2) return 1;
    builder.DeleteScanMatcher(sid);

    // the same queue with the refinement of constraint_builder_2d.cc:245-249 on the device,
    // and CeresScanMatcher2D::Match called directly (ceres_scan_matcher_2d.h:50-55)
    ConstraintBuilder2D refining(bo, &pool);
    refining.set_device_refinement(true);
    refining.MaybeAddConstraint(sid, &submap, mapping::NodeId{0, 0}, &node, relative);
    refining.MaybeAddGlobalConstraint(sid, &submap, mapping::NodeId{0, 2}, &node);
    refining.NotifyEndOfNode();
    ConstraintBuilder2D::Result got_refined;
    refining.WhenDone([&](const ConstraintBuilder2D::Result& r) { got_refined = r; });
    if (got_refined.size() != 2) return 1;
    for (const auto& c : got_refined)
      std::printf("RESULT cb2d_refined %d %.17g %.17g %.17g\n", c.node_id.node_index,
                  c.pose.zbar_ij.translation().x(), c.pose.zbar_ij.translation().y(),
                  2. * std::atan2(c.pose.zbar_ij.rotation().z(), c.pose.zbar_ij.rotation().w()));
    refining.DeleteScanMatcher(sid);
    mapping::scan_matching::CeresScanMatcher2D ceres(bo.ceres_scan_matcher_options());
    const transform::Rigid2d start({0.03, -0.02}, 0.01);
    transform::Rigid2d refined_pose;
    mapping::scan_matching::CeresScanMatcher2D::Summary summary;
    ceres.Match(start.translation(), start, cloud, grid, &refined_pose, &summary);
    std::printf("RESULT ceres2d %.17g %.17g %.17g %.17g %.17g %d %d %d\n",
                refined_pose.translation().x(), refined_pose.translation().y(),
                refined_pose.rotation().angle(), summary.initial_cost, summary.final_cost,
                summary.iterations, summary.num_successful_steps, summary.termination);
    if (!(summary.final_cost <= summary.initial_cost)) return 1;
  }
  {
    using mapping::constraints::ConstraintBuilder3D;
    mapping::constraints::proto::ConstraintBuilderOptions bo;
    bo.sampling_ratio_ = 1.0;
    bo.min_score_ = 0.1;
    bo.global_localization_min_score_ = 0.1;
    bo.fast3d_ = o3;
    common::InlineThreadPool pool;
    ConstraintBuilder3D builder(bo, &pool);
    mapping::Submap3D submap(&hybrid, &hybrid, &histogram);
    const mapping::SubmapId sid{0, 0};
    builder.MaybeAddConstraint(sid, &submap, mapping::NodeId{0, 0}, &data, transform::Rigid3d(),
                               transform::Rigid3d());
    builder.MaybeAddGlobalConstraint(sid, &submap, mapping::NodeId{0, 1}, &data,
                                     transform::Quaterniond{1., 0., 0., 0.},
                                     transform::Quaterniond{1., 0., 0., 0.});
    builder.NotifyEndOfNode();
    ConstraintBuilder3D::Result got;
    builder.WhenDone([&](const ConstraintBuilder3D::Result& r) { got = r; });
    std::printf("adapter_selftest: ConstraintBuilder3D %zu constraints, finished nodes %d\n",
                got.size(), builder.GetNumFinishedNodes());
    if (got.empty() || builder.GetNumFinishedNodes() != 1) return 1;
    if (std::fabs(got[0].pose.zbar_ij.translation().x() - tx) > 0.051 ||
        std::fabs(got[0].pose.zbar_ij.translation().y() - ty) > 0.051 ||
        std::fabs(got[0].pose.zbar_ij.translation().z() - tz) > 0.051)
      return 1;
    builder.DeleteScanMatcher(sid);

    // the local pair again with the refinement of constraint_builder_3d.cc:265-275 on the
    // device, and CeresScanMatcher3D::Match called directly
    ConstraintBuilder3D refining(bo, &pool);
    refining.set_device_refinement(true);
    refining.MaybeAddConstraint(sid, &submap, mapping::NodeId{0, 0}, &data, transform::Rigid3d(),
                                transform::Rigid3d());
    refining.NotifyEndOfNode();
    ConstraintBuilder3D::Result got_refined;
    refining.WhenDone([&](const ConstraintBuilder3D::Result& r) { got_refined = r; });
    if (got_refined.size() != 1) return 1;
    {
      const transform::Rigid3d& z = got_refined[0].pose.zbar_ij;
      std::printf("RESULT cb3d_refined %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n",
                  z.translation().x(), z.translation().y(), z.translation().z(), z.rotation().w(),
                  z.rotation().x(), z.rotation().y(), z.rotation().z());
    }
    refining.DeleteScanMatcher(sid);
    const mapping::scan_matching::DeviceHybridGrid device_grid(hybrid);
    mapping::scan_matching::CeresScanMatcher3D ceres3(bo.ceres_scan_matcher_options_3d());
    const transform::Rigid3d start({{0.22, -0.13, 0.08}}, transform::Quaterniond{1., 0., 0., 0.});
    transform::Rigid3d refined_pose;
    mapping::scan_matching::CeresScanMatcher3D::Summary summary3;
    ceres3.Match(start.translation(), start, {{&data.high_resolution_point_cloud, &device_grid}},
                 &refined_pose, &summary3);
    std::printf("RESULT ceres3d %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %d %d %d\n",
                refined_pose.translation().x(), refined_pose.translation().y(),
                refined_pose.translation().z(), refined_pose.rotation().w(),
                refined_pose.rotation().x(), refined_pose.rotation().y(),
                refined_pose.rotation().z(), summary3.initial_cost, summary3.final_cost,
                summary3.iterations, summary3.num_successful_steps, summary3.termination);
    if (!(summary3.final_cost <= summary3.initial_cost)) return 1;

    // ... with an intensity block on the pair (ceres_scan_matcher_3d.cc:123-139): intensity
    // 50 at the cloud's cells, one retroreflection above the threshold
    mapping::IntensityHybridGrid intensity_grid(0.05f);
    for (const auto& v : hybrid.voxels()) intensity_grid.AddIntensity(v.x, v.y, v.z, 50.f);
    std::vector<float> intensities(data.high_resolution_point_cloud.size(), 50.f);
    intensities[3] = 150.f;
    const sensor::PointCloud cloud_i(data.high_resolution_point_cloud.points(), intensities);
    const mapping::scan_matching::DeviceIntensityGrid device_intensity(intensity_grid);
    mapping::scan_matching::proto::CeresScanMatcherOptions3D oi =
        bo.ceres_scan_matcher_options_3d();
    oi.mutable_intensity_cost_function_options(0)->set_weight(0.5);
    oi.mutable_intensity_cost_function_options(0)->set_huber_scale(0.3);
    oi.mutable_intensity_cost_function_options(0)->set_intensity_threshold(100.f);
    mapping::scan_matching::CeresScanMatcher3D ceres3i(oi);
    ceres3i.Match(start.translation(), start, {{&cloud_i, &device_grid, &device_intensity}},
                  &refined_pose, &summary3);
    std::printf(
        "RESULT ceres3d_intensity %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g %d %d "
        "%d\n",
        refined_pose.translation().x(), refined_pose.translation().y(),
        refined_pose.translation().z(), refined_pose.rotation().w(), refined_pose.rotation().x(),
        refined_pose.rotation().y(), refined_pose.rotation().z(), summary3.initial_cost,
        summary3.final_cost, summary3.iterations, summary3.num_successful_steps,
        summary3.termination);
    if (!(summary3.final_cost <= summary3.initial_cost)) return 1;
  }
  // ---- RangeDataInserter3D on device grids: the reference's InsertPointCloudWithIntensities
  // (range_data_inserter_3d_test.cc:57-69), twice, into empty 1 m grids ----
  {
    mapping::proto::RangeDataInserterOptions3D io;
    io.set_hit_probability(0.7);
    io.set_miss_probability(0.4);
    io.set_num_free_space_voxels(1000);
    io.set_intensity_threshold(100.f);
    const mapping::scan_matching::RangeDataInserter3D inserter(io);
    mapping::scan_matching::DeviceHybridGrid grid(1.f, 0);
    mapping::scan_matching::DeviceIntensityGrid intensity(1.f, 0);
    sensor::RangeData range_data;
    range_data.origin = {{0.f, 0.f, -4.f}};
    range_data.returns = sensor::PointCloud(
        {{{{-3.f, -1.f, 4.f}}}, {{{-2.f, 0.f, 4.f}}}, {{{-1.f, 1.f, 4.f}}}, {{{0.f, 2.f, 4.f}}}},
        {7.f, 8.f, 9.f, 10.f});
    for (int i = 0; i < 2; ++i) inserter.Insert(range_data, &grid, &intensity);
    int32_t lo[3], dims[3];
    if (csm_grid3d_read(grid.handle(), lo, dims, nullptr) != CSM_OK) return 1;
    std::vector<uint16_t> values(static_cast<size_t>(dims[0]) * dims[1] * dims[2]);
    if (csm_grid3d_read(grid.handle(), lo, dims, values.data()) != CSM_OK) return 1;
    std::printf("RESULT insert3d %d %d %d %d %d %d", lo[0], lo[1], lo[2], dims[0], dims[1], dims[2]);
    for (uint16_t v : values) std::printf(" %u", v);
    std::printf("\n");
    if (csm_intensity_grid3d_read(intensity.handle(), lo, dims, nullptr, nullptr, nullptr) != CSM_OK)
      return 1;
    const size_t vox = static_cast<size_t>(dims[0]) * dims[1] * dims[2];
    std::vector<float> mean(vox), sum(vox);
    std::vector<int32_t> count(vox);
    if (csm_intensity_grid3d_read(intensity.handle(), lo, dims, mean.data(), sum.data(),
                                  count.data()) != CSM_OK)
      return 1;
    std::printf("RESULT insert3d_intensity %d %d %d %d %d %d", lo[0], lo[1], lo[2], dims[0],
                dims[1], dims[2]);
    for (size_t i = 0; i < vox; ++i)
      std::printf(" %08x:%08x:%d", Bits(mean[i]), Bits(sum[i]), count[i]);
    std::printf("\n");
  }
  // ---- ProbabilityGridRangeDataInserter2D on a device grid: the reference's InsertPointCloud
  // (range_data_inserter_2d_test.cc:47-58) with one miss, then a return that makes the grid
  // grow; the cropped grid and a stack built from it ----
  {
    mapping::proto::ProbabilityGridRangeDataInserterOptions2D io;
    io.set_hit_probability(0.7);
    io.set_miss_probability(0.4);
    io.set_insert_free_space(true);
    const mapping::scan_matching::ProbabilityGridRangeDataInserter2D inserter(io);
    mapping::scan_matching::DeviceGrid2D grid(
        mapping::MapLimits(1., 1., 5., mapping::CellLimits{5, 5}), 0);
    sensor::RangeData range_data;
    range_data.origin = {{-0.5f, 0.5f, 0.f}};
    range_data.returns = sensor::PointCloud(
        {{{{-3.5f, 0.5f, 0.f}}}, {{{-2.5f, 1.5f, 0.f}}}, {{{-1.5f, 2.5f, 0.f}}},
         {{{-0.5f, 3.5f, 0.f}}}},
        {});
    range_data.misses = sensor::PointCloud({{{{0.5f, 4.5f, 0.f}}}}, {});
    inserter.Insert(range_data, &grid);
    sensor::RangeData far;
    far.origin = {{-0.5f, 0.5f, 0.f}};
    far.returns = sensor::PointCloud({{{{-6.5f, 0.5f, 0.f}}}}, {});
    inserter.Insert(far, &grid);
    const std::unique_ptr<mapping::scan_matching::DeviceGrid2D> cropped = grid.ComputeCroppedGrid();
    for (const mapping::scan_matching::DeviceGrid2D* g : {&grid, cropped.get()}) {
      std::vector<uint16_t> cells;
      const csm_rt_grid2d_info info = g->Read(&cells);
      std::printf("RESULT %s %.17g %.17g %.17g %d %d %d %d %d %d %d", g == &grid ? "insert2d" : "crop2d",
                  info.resolution, info.max_x, info.max_y, info.num_x_cells, info.num_y_cells,
                  info.known_empty, info.known_min_x, info.known_min_y, info.known_max_x,
                  info.known_max_y);
      for (uint16_t v : cells) std::printf(" %u", v);
      std::printf("\n");
    }
    mapping::scan_matching::proto::FastCorrelativeScanMatcherOptions2D fo;
    fo.set_linear_search_window(3.);
    fo.set_angular_search_window(0.5);
    fo.set_branch_and_bound_depth(2);
    const mapping::scan_matching::FastCorrelativeScanMatcher2D matcher(*cropped, fo);
    int32_t wx = 0, wy = 0;
    if (csm_stack2d_read_level(matcher.stack(), 1, nullptr, &wx, &wy) != CSM_OK) return 1;
    std::vector<uint8_t> level(static_cast<size_t>(wx) * wy);
    if (csm_stack2d_read_level(matcher.stack(), 1, level.data(), &wx, &wy) != CSM_OK) return 1;
    std::printf("RESULT stack2d %d %d", wx, wy);
    for (uint8_t v : level) std::printf(" %u", v);
    std::printf("\n");
  }
  // ---- TSDFRangeDataInserter2D on a device grid: the reference's InsertPoint
  // (tsdf_range_data_inserter_2d_test.cc:50-57, the 8 x 1 grid that grows), then two returns
  // with the lua defaults' normal projection and weighting ----
  {
    mapping::proto::TSDFRangeDataInserterOptions2D to;
    to.set_truncation_distance(2.0);
    to.set_maximum_weight(10.);
    to.set_update_free_space(false);
    to.mutable_normal_estimation_options()->set_num_normal_samples(2);
    to.mutable_normal_estimation_options()->set_sample_radius(10.);
    to.set_project_sdf_distance_to_scan_normal(false);
    const mapping::scan_matching::TSDFRangeDataInserter2D plain(to);
    to.set_project_sdf_distance_to_scan_normal(true);
    to.set_update_weight_angle_scan_normal_to_ray_kernel_bandwidth(0.5);
    to.set_update_weight_distance_cell_to_hit_kernel_bandwidth(0.5);
    const mapping::scan_matching::TSDFRangeDataInserter2D weighted(to);
    mapping::scan_matching::DeviceGrid2D grid(
        mapping::MapLimits(1., 1., 7., mapping::CellLimits{8, 1}), 2.f, 10.f, 0);
    sensor::RangeData range_data;
    range_data.origin = {{-0.5f, -0.5f, 0.f}};
    range_data.returns = sensor::PointCloud({{{{-0.5f, 3.5f, 0.f}}}}, {});
    plain.Insert(range_data, &grid);
    range_data.returns = sensor::PointCloud({{{{-0.5f, 3.5f, 0.f}}}, {{{5.5f, 3.5f, 0.f}}}}, {});
    weighted.Insert(range_data, &grid);
    std::vector<uint16_t> tsd, weights;
    const csm_rt_grid2d_info info = grid.Read(&tsd);
    grid.ReadWeights(&weights);
    std::printf("RESULT insert_tsdf2d %.17g %.17g %.17g %d %d %d %d %d %d %d", info.resolution,
                info.max_x, info.max_y, info.num_x_cells, info.num_y_cells, info.known_empty,
                info.known_min_x, info.known_min_y, info.known_max_x, info.known_max_y);
    for (uint16_t v : tsd) std::printf(" %u", v);
    for (uint16_t v : weights) std::printf(" %u", v);
    std::printf("\n");
  }
  return 0;
}
