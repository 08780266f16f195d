// Compiles the drop-in adapter classes against the stand-in headers and links
// them to libcsm_b200.so.  With a GPU it runs one match through the reference-
// shaped C++ API; without one it only checks that the ABI reports CSM_E_CUDA
// (no CPU fallback) — either way the binary proves the adapter builds and links.
#include <cmath>
#include <cstdio>
#include <cstring>

#include "constraint_builder_b200.h"
#include "points_processor_b200.h"
#include "pose_graph_trimmer_b200.h"
#include "scan_matchers_b200.h"
#include "voxel_filter_b200.h"

using namespace cartographer;

// RESULT lines are parsed by tests/test_gpu_adapter.py and compared with the oracle:
// float scores as their bit patterns, doubles with 17 significant digits.
static unsigned Bits(float f) {
  unsigned u;
  std::memcpy(&u, &f, 4);
  return u;
}

// Host-only part (runs everywhere): the builders' gating and WhenDone cycle when no
// pair survives the gates — nothing reaches the device — and the sampler's sequence
// (common/fixed_ratio_sampler_test.cc).
// A serialised grid (DeviceHybridGrid / DeviceGrid2D::ToProto, the bytes in this stand-in
// build) as one hex RESULT line.
static void PrintBytes(const char* name, const std::string& bytes) {
  std::printf("RESULT %s ", name);
  for (unsigned char c : bytes) std::printf("%02x", c);
  std::printf("\n");
}

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
  // the same cycle through ConstraintBuilder3D
  using mapping::constraints::ConstraintBuilder3D;
  ConstraintBuilder3D builder3d(bo, &pool);
  const mapping::Submap3D submap3d(nullptr, nullptr, nullptr);  // never read: the pair is gated
  builder3d.MaybeAddConstraint(mapping::SubmapId{0, 0}, &submap3d, mapping::NodeId{0, 0}, &node,
                               transform::Rigid3d({{5., 0., 0.}},  // beyond max_constraint_distance
                                                  transform::Quaterniond{1., 0., 0., 0.}),
                               transform::Rigid3d());
  builder3d.NotifyEndOfNode();
  calls = 0;
  constraints = 99;
  builder3d.WhenDone([&](const ConstraintBuilder3D::Result& r) { ++calls; constraints = r.size(); });
  if (calls != 1 || constraints != 0 || builder3d.GetNumFinishedNodes() != 1) return 1;
  // Rigid2d algebra used for the constraint transform
  const transform::Rigid2d a({1., 2.}, 0.3);
  const transform::Rigid2d id = a.inverse() * a;
  if (std::fabs(id.translation().x()) > 1e-12 || std::fabs(id.translation().y()) > 1e-12 ||
      std::fabs(id.rotation().angle()) > 1e-12)
    return 1;
  std::printf("adapter_selftest: host-only checks passed\n");
  return 0;
}

// ---- OverlappingSubmapsTrimmer2D: the reference's overlapping_submaps_trimmer_2d_test.cc cases
// on device grids, and one random map whose inputs and outcome are printed ----
namespace trimmer_cases {
using mapping::NodeId;
using mapping::PoseGraphInterface;
using mapping::SubmapId;
using mapping::scan_matching::DeviceGrid2D;

transform::Rigid3d Embed3D(double x, double y, double theta) {
  return transform::Rigid3d({{x, y, 0.}}, transform::Quaterniond{std::cos(theta / 2), 0., 0.,
                                                                  std::sin(theta / 2)});
}

class FakeTrimmable : public mapping::Trimmable {
 public:
  mapping::MapById<SubmapId, PoseGraphInterface::SubmapData> GetOptimizedSubmapData()
      const override {
    return submap_data;
  }
  const mapping::MapById<NodeId, mapping::TrajectoryNode>& GetTrajectoryNodes() const override {
    return nodes;
  }
  const std::vector<PoseGraphInterface::Constraint>& GetConstraints() const override {
    return constraints;
  }
  void TrimSubmap(const SubmapId& id) override { trimmed.push_back(id); }

  // AddSquareSubmap: num_cells x num_cells cells of value 1, resolution 1, max = corner
  void AddSquareSubmap(const transform::Rigid3d& global, const transform::Rigid3d& local,
                       double corner_x, double corner_y, int index, int num_cells,
                       bool finished) {
    const mapping::Grid2D grid(
        mapping::MapLimits(1.0, corner_x, corner_y, mapping::CellLimits{num_cells, num_cells}),
        0.1f, 0.9f, std::vector<uint16_t>(num_cells * num_cells, 1));
    grids[SubmapId{0, index}] = std::make_shared<DeviceGrid2D>(grid);
    submap_data.Insert(SubmapId{0, index},
                       {std::make_shared<const mapping::Submap2D>(local, finished), global});
  }
  void AddNode(int index, int64_t time) {
    mapping::TrajectoryNode n;
    n.time_.ticks = time;
    nodes.Insert(NodeId{0, index}, n);
  }
  void AddConstraint(int submap, int node, bool intra) {
    PoseGraphInterface::Constraint c;
    c.submap_id = SubmapId{0, submap};
    c.node_id = NodeId{0, node};
    c.tag = intra ? PoseGraphInterface::Constraint::INTRA_SUBMAP
                  : PoseGraphInterface::Constraint::INTER_SUBMAP;
    constraints.push_back(c);
  }
  mapping::OverlappingSubmapsTrimmer2D::DeviceGridOf DeviceGrids() {
    return [this](const SubmapId& id, const mapping::Submap2D&) -> const DeviceGrid2D& {
      return *grids.at(id);
    };
  }
  std::string Trimmed() const {
    std::string s;
    for (const SubmapId& id : trimmed) s += std::to_string(id.submap_index) + ",";
    return s;
  }

  mapping::MapById<SubmapId, PoseGraphInterface::SubmapData> submap_data;
  mapping::MapById<NodeId, mapping::TrajectoryNode> nodes;
  std::vector<PoseGraphInterface::Constraint> constraints;
  std::vector<SubmapId> trimmed;
  std::map<SubmapId, std::shared_ptr<DeviceGrid2D>> grids;
};

int Expect(const char* name, const FakeTrimmable& g, const char* want) {
  const bool ok = g.Trimmed() == want;
  std::printf("RESULT trimmer2d_%s %s %s\n", name, ok ? "ok" : "FAILED", g.Trimmed().c_str());
  return ok ? 0 : 1;
}

void TwoOverlapping(FakeTrimmable* g, bool finished0) {
  const transform::Rigid3d id;
  g->AddSquareSubmap(id, id, 1., 1., 0, 1, finished0);
  g->AddSquareSubmap(id, id, 1., 1., 1, 1, true);
  g->AddNode(0, 1000);
  g->AddNode(1, 2000);
  g->AddConstraint(0, 0, true);
  g->AddConstraint(1, 1, true);
}

int Run() {
  using Trimmer = mapping::OverlappingSubmapsTrimmer2D;
  const transform::Rigid3d id;
  int failed = 0;
  {
    FakeTrimmable g;
    Trimmer t(1, 0, 0, g.DeviceGrids());
    t.Trim(&g);
    failed += Expect("EmptyPoseGraph", g, "");
  }
  {
    FakeTrimmable g;
    TwoOverlapping(&g, true);
    Trimmer t(1, 0, 0, g.DeviceGrids());
    t.Trim(&g);
    failed += Expect("TrimOneOfTwoOverlappingSubmaps", g, "0,");
  }
  {
    FakeTrimmable g;
    TwoOverlapping(&g, true);
    Trimmer t(1, 0, 2, g.DeviceGrids());
    t.Trim(&g);
    failed += Expect("TestMinAddedSubmapsCountParam_first", g, "");
    g.AddSquareSubmap(id, id, 1., 1., 2, 1, true);
    g.AddNode(2, 3000);
    g.AddConstraint(2, 2, true);
    t.Trim(&g);
    failed += Expect("TestMinAddedSubmapsCountParam", g, "0,1,");
  }
  {
    FakeTrimmable g;
    TwoOverlapping(&g, false);
    Trimmer t(1, 0, 0, g.DeviceGrids());
    t.Trim(&g);
    failed += Expect("DoNotTrimUnfinishedSubmap", g, "");
  }
  {
    FakeTrimmable g;
    g.AddSquareSubmap(id, id, 1., 1., 0, 1, true);
    g.AddSquareSubmap(id, id, 1., 1., 1, 1, true);
    g.AddNode(0, 1000);
    g.AddNode(1, 2000);
    g.AddNode(2, 3000);
    g.AddConstraint(0, 0, false);
    g.AddConstraint(0, 2, true);
    g.AddConstraint(1, 1, true);
    Trimmer t(1, 0, 0, g.DeviceGrids());
    t.Trim(&g);
    failed += Expect("UseOnlyIntraSubmapsToComputeFreshness", g, "1,");
  }
  {
    FakeTrimmable g;
    g.AddSquareSubmap(id, id, 1., 1., 0, 2, true);
    g.AddSquareSubmap(Embed3D(1., 1., 0.), id, 1., 1., 1, 2, true);
    g.AddNode(0, 1000);
    g.AddNode(1, 2000);
    g.AddConstraint(0, 0, true);
    g.AddConstraint(1, 1, true);
    Trimmer t(1, 4, 0, g.DeviceGrids());
    t.Trim(&g);
    failed += Expect("TrimSubmapWithLowCoveredCellsCount", g, "0,");
  }
  {
    FakeTrimmable g;
    g.AddSquareSubmap(id, id, 1., 1., 0, 1, true);
    const transform::Rigid3d transform = Embed3D(1., 1., M_PI / 2);
    g.AddSquareSubmap(transform, transform, 1., 1., 1, 1, true);
    g.AddNode(0, 1000);
    g.AddNode(1, 2000);
    g.AddConstraint(0, 0, true);
    g.AddConstraint(1, 1, true);
    Trimmer t(1, 0, 0, g.DeviceGrids());
    t.Trim(&g);
    failed += Expect("TestTransformations", g, "0,");
  }
  {
    // 40 random 60 x 60 submaps at 5 cm along a circle with random yaw, a few shared times
    FakeTrimmable g;
    uint64_t state = 12345;
    auto next = [&state]() {
      state = state * 6364136223846793005ull + 1442695040888963407ull;
      return static_cast<double>(state >> 11) / 9007199254740992.;
    };
    const int n = 40, size = 60;
    std::vector<std::vector<uint16_t>> cells(n);
    std::vector<transform::Rigid3d> composed(n);
    std::vector<double> limits(3 * n);
    for (int i = 0; i < n; ++i) {
      const double a = 2 * M_PI * i / 12, x = 1.0 * std::cos(a), y = 1.0 * std::sin(a);
      cells[i].resize(size * size);
      for (auto& c : cells[i]) c = next() < 0.7 ? static_cast<uint16_t>(1 + next() * 32766) : 0;
      const double mx = x + size / 2 * 0.05, my = y + size / 2 * 0.05;
      limits[3 * i] = mx;
      limits[3 * i + 1] = my;
      limits[3 * i + 2] = 0.05;
      const mapping::Grid2D grid(mapping::MapLimits(0.05, mx, my, mapping::CellLimits{size, size}),
                                 0.1f, 0.9f, cells[i]);
      g.grids[SubmapId{0, i}] = std::make_shared<DeviceGrid2D>(grid);
      const transform::Rigid3d local = Embed3D(x, y, 2 * M_PI * next());
      const transform::Rigid3d global = Embed3D(x + 0.1 * next(), y - 0.1 * next(), 2 * M_PI * next());
      g.submap_data.Insert(SubmapId{0, i},
                           {std::make_shared<const mapping::Submap2D>(local, true), global});
      composed[i] = global * local.inverse();
      g.AddNode(i, i % 9 == 4 ? 1000 * (i - 1) : 1000 * i);
      g.AddConstraint(i, i, true);
    }
    Trimmer t(2, 0.5, 0, g.DeviceGrids());
    t.Trim(&g);
    // the inputs of the coverage pass and its outcome, which the GPU test checks against the
    // CPU restatement (tests/trimmer2d_oracle.cc)
    for (int i = 0; i < n; ++i) {
      const auto& tr = composed[i].translation();
      const auto& q = composed[i].rotation();
      std::printf("RESULT trimmer2d_random_submap %d %lld %.17g %.17g %.17g %.17g %.17g %.17g "
                  "%.17g %.17g %.17g %.17g %d ",
                  i, static_cast<long long>(i % 9 == 4 ? 1000 * (i - 1) : 1000 * i),
                  limits[3 * i], limits[3 * i + 1], limits[3 * i + 2], tr.x(), tr.y(), tr.z(),
                  q.w(), q.x(), q.y(), q.z(), size);
      for (uint16_t c : cells[i]) std::printf("%04x", c);
      std::printf("\n");
    }
    std::printf("RESULT trimmer2d_random_map %s\n", g.Trimmed().c_str());
    std::printf("RESULT trimmer2d_random_map_stats %lld %lld\n",
                static_cast<long long>(t.last_stats().entries),
                static_cast<long long>(t.last_stats().coverage_cells));
  }
  return failed;
}
}  // namespace trimmer_cases

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
    PrintBytes("grid_to_proto_insert3d", grid.ToProto());
    // Submap3D::ToResponseProto on device grids: the version, then the high-resolution grid's
    // texture and the low-resolution grid's (a fresh one here: no voxel, the 2 x 2 texture)
    {
      const transform::Rigid3d pose({{0.5, -0.25, 0.125}},
                                    {0.96592582628906831, 0., 0., 0.25881904510252074});
      const mapping::scan_matching::DeviceHybridGrid low(2.f, 0);
      std::string high_texture, low_texture;
      grid.AddToTextureProto(pose, &high_texture);
      low.AddToTextureProto(pose, &low_texture);
      std::printf("RESULT texture_response3d 2\n");
      PrintBytes("texture_response3d_high", high_texture);
      PrintBytes("texture_response3d_low", low_texture);
    }
  }
  // ---- ActiveSubmaps2D over device grids: seven scans with num_range_data = 2, so submaps
  // roll over, finish and are evicted; the active submaps' grids, limits, boxes, counts,
  // finished flags and local poses, and the first submap's after its eviction, which
  // tests/test_gpu_adapter_active_submaps2d.py holds equal to scan_matching.ActiveSubmaps2D's ----
  {
    mapping::proto::SubmapsOptions2D so;
    so.set_num_range_data(2);
    so.mutable_grid_options_2d()->set_resolution(0.05f);
    auto* pgo = so.mutable_range_data_inserter_options()
                    ->mutable_probability_grid_range_data_inserter_options_2d();
    pgo->set_hit_probability(0.55);
    pgo->set_miss_probability(0.49);
    pgo->set_insert_free_space(true);
    mapping::ActiveSubmaps2D active(so, 0);
    std::shared_ptr<const mapping::DeviceSubmap2D> first;
    std::vector<std::shared_ptr<const mapping::DeviceSubmap2D>> subs;
    for (int k = 0; k < 7; ++k) {
      sensor::RangeData range_data;
      range_data.origin = {{0.3f * k, -0.2f * k, 0.f}};
      for (int i = 0; i < 180; ++i) {
        const double a = 0.035 * i + 0.1 * k;
        const float r = (i % 7 == 3) ? 5.f : 2.f + 0.01f * (i % 40);
        const sensor::RangefinderPoint p{{{range_data.origin.x() + r * static_cast<float>(std::cos(a)),
                                           range_data.origin.y() + r * static_cast<float>(std::sin(a)),
                                           0.f}}};
        (i % 7 == 3 ? range_data.misses : range_data.returns).push_back(p);
      }
      subs = active.InsertRangeData(range_data);
      if (!first) first = subs.front();
    }
    auto print = [](const char* name, const mapping::DeviceSubmap2D& s) {
      std::vector<uint16_t> cells;
      const csm_rt_grid2d_info info = s.grid().Read(&cells);
      std::printf("RESULT %s_grid %d %d %.17g %.17g %.17g %d %d %d %d %d", name, info.num_x_cells,
                  info.num_y_cells, info.resolution, info.max_x, info.max_y, info.known_empty,
                  info.known_min_x, info.known_min_y, info.known_max_x, info.known_max_y);
      for (uint16_t c : cells) std::printf(" %u", c);
      std::printf("\n");
      const transform::Rigid3d& p = s.local_pose();
      std::printf("RESULT %s_state %d %d %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", name,
                  s.num_range_data(), s.insertion_finished() ? 1 : 0, p.translation().x(),
                  p.translation().y(), p.translation().z(), p.rotation().w(), p.rotation().x(),
                  p.rotation().y(), p.rotation().z());
    };
    if (subs.size() != 2 || first == subs.front() || !first->insertion_finished()) return 1;
    print("active2d0", *subs[0]);
    print("active2d1", *subs[1]);
    print("evicted2d", *first);
    if (first->device_submap().grid != &first->grid()) return 1;
  }
  // ---- ActiveSubmaps3D over device grids: seven scans with num_range_data = 2, so submaps
  // roll over, finish and are evicted; the active submaps' handles and histograms, and the
  // first submap's after its eviction, which tests/test_gpu_adapter_active_submaps3d.py holds
  // equal to scan_matching.ActiveSubmaps3D's ----
  {
    mapping::proto::SubmapsOptions3D so;
    so.set_high_resolution(0.1);
    so.set_high_resolution_max_range(4.0);
    so.set_low_resolution(0.45);
    so.set_num_range_data(2);
    so.mutable_range_data_inserter_options()->set_hit_probability(0.55);
    so.mutable_range_data_inserter_options()->set_miss_probability(0.49);
    so.mutable_range_data_inserter_options()->set_num_free_space_voxels(2);
    so.mutable_range_data_inserter_options()->set_intensity_threshold(40.f);
    mapping::ActiveSubmaps3D active(so, 0);
    std::shared_ptr<const mapping::DeviceSubmap3D> first;
    std::vector<std::shared_ptr<const mapping::DeviceSubmap3D>> subs;
    for (int k = 0; k < 7; ++k) {
      sensor::RangeData range_data;
      range_data.origin = {{0.25f * k, -0.125f * k, 0.5f}};
      std::vector<sensor::RangefinderPoint> points;
      std::vector<float> intensities;
      for (int i = 0; i < 240; ++i) {
        points.push_back({{{-3.f + 0.125f * (i % 48) + 0.25f * k, 2.f - 0.5f * (i / 48),
                            1.5f - 0.25f * (i % 5)}}});
        intensities.push_back(static_cast<float>(i % 60));
      }
      range_data.returns = sensor::PointCloud(points, intensities);
      const transform::Quaterniond q{std::cos(0.05 * k), 0., 0., std::sin(0.05 * k)};
      std::vector<float> histogram(8);
      for (int i = 0; i < 8; ++i) histogram[i] = static_cast<float>(i + k);
      subs = active.InsertData(range_data, q, histogram);
      if (!first) first = subs.front();
    }
    auto print = [](const char* name, const mapping::DeviceSubmap3D& s) {
      int32_t lo[3], dims[3];
      for (const auto* g : {&s.high_resolution_hybrid_grid(), &s.low_resolution_hybrid_grid()}) {
        if (csm_grid3d_read(g->handle(), lo, dims, nullptr) != CSM_OK) return false;
        std::vector<uint16_t> v(static_cast<size_t>(dims[0]) * dims[1] * dims[2]);
        if (csm_grid3d_read(g->handle(), lo, dims, v.data()) != CSM_OK) return false;
        std::printf("RESULT %s_%s %d %d %d %d %d %d", name,
                    g == &s.high_resolution_hybrid_grid() ? "high" : "low", lo[0], lo[1], lo[2],
                    dims[0], dims[1], dims[2]);
        for (uint16_t x : v) std::printf(" %u", x);
        std::printf("\n");
      }
      std::printf("RESULT %s_state %d %d", name, s.num_range_data(), s.insertion_finished() ? 1 : 0);
      for (float h : s.rotational_scan_matcher_histogram()) std::printf(" %08x", Bits(h));
      std::printf("\n");
      std::printf("RESULT %s_intensity", name);
      if (const auto* ig = s.high_resolution_intensity_hybrid_grid()) {
        if (csm_intensity_grid3d_read(ig->handle(), lo, dims, nullptr, nullptr, nullptr) != CSM_OK)
          return false;
        const size_t vox = static_cast<size_t>(dims[0]) * dims[1] * dims[2];
        std::vector<float> mean(vox), sum(vox);
        std::vector<int32_t> count(vox);
        if (csm_intensity_grid3d_read(ig->handle(), lo, dims, mean.data(), sum.data(),
                                      count.data()) != CSM_OK)
          return false;
        std::printf(" %d %d %d %d %d %d", lo[0], lo[1], lo[2], dims[0], dims[1], dims[2]);
        for (size_t i = 0; i < vox; ++i)
          std::printf(" %08x:%08x:%d", Bits(mean[i]), Bits(sum[i]), count[i]);
      } else {
        std::printf(" forgotten");
      }
      std::printf("\n");
      return true;
    };
    if (subs.size() != 2 || first == subs.front()) return 1;
    if (!print("active0", *subs[0]) || !print("active1", *subs[1]) || !print("evicted", *first))
      return 1;
    if (subs[0]->device_submap().high_resolution_hybrid_grid != &subs[0]->high_resolution_hybrid_grid())
      return 1;
  }
  // ---- FastCorrelativeScanMatcher3D and ConstraintBuilder3D on inserted device grids: the
  // axis cloud inserted twice from its sensor position into empty grids; the same built from
  // host HybridGrids of the grids' non-zero voxels prints the *_host lines, which
  // tests/test_gpu_adapter_matcher3d_from_grid.py holds equal to the *_dev lines ----
  {
    mapping::proto::RangeDataInserterOptions3D io;
    io.set_hit_probability(0.7);
    io.set_miss_probability(0.4);
    io.set_num_free_space_voxels(2);
    io.set_intensity_threshold(100.f);
    const mapping::scan_matching::RangeDataInserter3D inserter(io);
    mapping::scan_matching::DeviceHybridGrid dhi(0.05f, 0), dlo(0.1f, 0);
    sensor::RangeData range_data;
    range_data.origin = {{tx, ty, tz}};
    for (const auto& p : cloud3.points())
      range_data.returns.push_back({{{p.position.x() + tx, p.position.y() + ty,
                                      p.position.z() + tz}}});
    for (int i = 0; i < 2; ++i) {
      inserter.Insert(range_data, &dhi, nullptr);
      inserter.Insert(range_data, &dlo, nullptr);
    }
    mapping::HybridGrid hhi(0.05f), hlo(0.1f);
    for (auto gp : {std::make_pair(&dhi, &hhi), std::make_pair(&dlo, &hlo)}) {
      int32_t lo[3], dims[3];
      if (csm_grid3d_read(gp.first->handle(), lo, dims, nullptr) != CSM_OK) return 1;
      std::vector<uint16_t> values(static_cast<size_t>(dims[0]) * dims[1] * dims[2]);
      if (csm_grid3d_read(gp.first->handle(), lo, dims, values.data()) != CSM_OK) return 1;
      for (int z = 0; z < dims[2]; ++z)
        for (int y = 0; y < dims[1]; ++y)
          for (int x = 0; x < dims[0]; ++x) {
            const uint16_t v = values[(static_cast<size_t>(z) * dims[1] + y) * dims[0] + x];
            if (v != 0) gp.second->Set(x + lo[0], y + lo[1], z + lo[2], v);
          }
    }
    using Matcher3D = mapping::scan_matching::FastCorrelativeScanMatcher3D;
    auto print = [](const char* name, const std::unique_ptr<Matcher3D::Result>& r) {
      std::printf("RESULT %s %d", name, r ? 1 : 0);
      if (r)
        std::printf(" %08x %.17g %.17g %.17g %.17g %.17g %.17g %.17g %08x %08x", Bits(r->score),
                    r->pose_estimate.translation().x(), r->pose_estimate.translation().y(),
                    r->pose_estimate.translation().z(), r->pose_estimate.rotation().w(),
                    r->pose_estimate.rotation().x(), r->pose_estimate.rotation().y(),
                    r->pose_estimate.rotation().z(), Bits(r->rotational_score),
                    Bits(r->low_resolution_score));
      std::printf("\n");
    };
    const Matcher3D mdev(dhi, &dlo, &histogram, o3);
    const Matcher3D mhost(hhi, &hlo, &histogram, o3);
    const transform::Quaterniond q{1., 0., 0., 0.};
    for (const Matcher3D* m : {&mdev, &mhost}) {
      const char* side = m == &mdev ? "dev" : "host";
      char name[64];
      std::snprintf(name, sizeof(name), "fast3d_grid_%s", side);
      const auto r = m->Match(transform::Rigid3d(), transform::Rigid3d(), data, 0.1f);
      if (!r) return 1;
      print(name, r);
      std::snprintf(name, sizeof(name), "fast3d_grid_full_%s", side);
      print(name, m->MatchFullSubmap(q, q, data, 0.1f));
    }
    using mapping::constraints::ConstraintBuilder3D;
    mapping::constraints::proto::ConstraintBuilderOptions bo;
    bo.sampling_ratio_ = 1.0;
    bo.min_score_ = 0.1;
    bo.global_localization_min_score_ = 0.1;
    bo.fast3d_ = o3;
    common::InlineThreadPool pool;
    const mapping::constraints::DeviceSubmap3D dsub{&dhi, &dlo, &histogram};
    const mapping::Submap3D hsub(&hhi, &hlo, &histogram);
    for (int side = 0; side < 2; ++side) {
      for (int refine = 0; refine < 2; ++refine) {
        ConstraintBuilder3D builder(bo, &pool);
        builder.set_device_refinement(refine == 1);
        const mapping::SubmapId sid{0, 0};
        if (side == 0) {
          builder.MaybeAddConstraint(sid, &dsub, mapping::NodeId{0, 0}, &data,
                                     transform::Rigid3d(), transform::Rigid3d());
          builder.MaybeAddGlobalConstraint(sid, &dsub, mapping::NodeId{0, 1}, &data, q, q);
        } else {
          builder.MaybeAddConstraint(sid, &hsub, mapping::NodeId{0, 0}, &data,
                                     transform::Rigid3d(), transform::Rigid3d());
          builder.MaybeAddGlobalConstraint(sid, &hsub, mapping::NodeId{0, 1}, &data, q, q);
        }
        builder.NotifyEndOfNode();
        ConstraintBuilder3D::Result got;
        builder.WhenDone([&](const ConstraintBuilder3D::Result& r) { got = r; });
        if (got.size() != 2) return 1;
        for (const auto& c : got) {
          const transform::Rigid3d& z = c.pose.zbar_ij;
          std::printf("RESULT cb3d_grid%s_%s %d %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n",
                      refine ? "_refined" : "", side == 0 ? "dev" : "host", c.node_id.node_index,
                      z.translation().x(), z.translation().y(), z.translation().z(),
                      z.rotation().w(), z.rotation().x(), z.rotation().y(), z.rotation().z());
        }
        builder.DeleteScanMatcher(sid);
      }
    }
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
      PrintBytes(g == &grid ? "grid_to_proto_insert2d" : "grid_to_proto_crop2d", g->ToProto());
      // Submap2D::ToResponseProto: the version, then the grid's texture with the local pose
      const transform::Rigid3d local_pose({{0.5, -0.25, 0.}},
                                          {0.96592582628906831, 0., 0., 0.25881904510252074});
      std::string texture;
      if (!g->DrawToSubmapTexture(&texture, local_pose)) return 1;
      PrintBytes(g == &grid ? "texture_response2d_insert" : "texture_response2d_crop", texture);
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
  // ---- ConstraintBuilder2D on device submaps: two submaps grown by the inserter in a 6 m x 4 m
  // room with a pillar, cropped, and driven through the reference's call cycle
  // (constraint_builder_2d_test.cc:58-112) as DeviceSubmap2Ds, unrefined and with the device
  // refinement.  The same queues on host Submap2Ds made from the cells read back print the
  // *_host lines, which tests/test_gpu_adapter_cb2d_device_submaps.py holds equal to the
  // *_dev lines ----
  {
    // a 1° scan of the room [-3, 3] x [-2, 2] with the pillar [1, 1.4] x [0.5, 0.9], from (x, y)
    const auto scan = [](double x, double y) {
      std::vector<sensor::RangefinderPoint> points;
      for (int k = 0; k < 360; ++k) {
        const double a = k * M_PI / 180. + 0.01, c = std::cos(a), s = std::sin(a);
        double t = 1e9;
        for (double wall : {3. - x, -3. - x})
          if (c * wall > 0) t = std::min(t, wall / c);
        for (double wall : {2. - y, -2. - y})
          if (s * wall > 0) t = std::min(t, wall / s);
        for (double px : {1. - x, 1.4 - x}) {   // the pillar's two x faces
          const double u = px / c;
          if (u > 0 && y + u * s >= 0.5 && y + u * s <= 0.9) t = std::min(t, u);
        }
        for (double py : {0.5 - y, 0.9 - y}) {   // and its two y faces
          const double u = py / s;
          if (u > 0 && x + u * c >= 1. && x + u * c <= 1.4) t = std::min(t, u);
        }
        points.push_back({{{static_cast<float>(t * c), static_cast<float>(t * s), 0.f}}});
      }
      return points;
    };
    mapping::proto::ProbabilityGridRangeDataInserterOptions2D io;
    io.set_hit_probability(0.55);
    io.set_miss_probability(0.49);
    io.set_insert_free_space(true);
    const mapping::scan_matching::ProbabilityGridRangeDataInserter2D inserter(io);
    const double origins[2][2] = {{-0.4, -0.3}, {0.6, 0.2}};
    std::vector<std::unique_ptr<mapping::scan_matching::DeviceGrid2D>> cropped;
    std::vector<std::unique_ptr<mapping::Grid2D>> host_grids;
    for (const auto& o : origins) {
      // ActiveSubmaps2D::CreateGrid(origin): 100 x 100 cells, max = origin + 50 * resolution
      mapping::scan_matching::DeviceGrid2D grid(
          mapping::MapLimits(0.05, o[0] + 2.5, o[1] + 2.5, mapping::CellLimits{100, 100}), 0);
      for (int k = 0; k < 4; ++k) {
        const double x = o[0] + 0.1 * k, y = o[1] - 0.05 * k;
        sensor::RangeData range_data;
        range_data.origin = {{static_cast<float>(x), static_cast<float>(y), 0.f}};
        for (const auto& p : scan(x, y))
          range_data.returns.push_back({{{p.position.x() + static_cast<float>(x),
                                          p.position.y() + static_cast<float>(y), 0.f}}});
        inserter.Insert(range_data, &grid);
      }
      cropped.push_back(grid.ComputeCroppedGrid());
      std::vector<uint16_t> cells;
      const csm_rt_grid2d_info info = cropped.back()->Read(&cells);
      if (info.is_tsdf != 0 || cropped.back()->device() != 0) return 1;
      host_grids.emplace_back(new mapping::Grid2D(
          mapping::MapLimits(info.resolution, info.max_x, info.max_y,
                             mapping::CellLimits{info.num_x_cells, info.num_y_cells}),
          1.f - 0.9f, 1.f - 0.1f, cells));   // kMin / kMaxCorrespondenceCost
    }
    const transform::Rigid2d local_poses[2] = {transform::Rigid2d({-0.4, -0.3}, 0.),
                                               transform::Rigid2d({0.6, 0.2}, 0.)};
    const mapping::constraints::DeviceSubmap2D dsubs[2] = {{cropped[0].get(), local_poses[0]},
                                                            {cropped[1].get(), local_poses[1]}};
    const mapping::Submap2D hsubs[2] = {{host_grids[0].get(), local_poses[0]},
                                        {host_grids[1].get(), local_poses[1]}};
    mapping::TrajectoryNodeData nodes[2];
    const double node_xy[2][2] = {{0.1, 0.3}, {-0.7, -0.5}};
    for (int n = 0; n < 2; ++n)
      for (const auto& p : scan(node_xy[n][0], node_xy[n][1]))
        nodes[n].filtered_gravity_aligned_point_cloud.push_back(p);
    using mapping::constraints::ConstraintBuilder2D;
    mapping::constraints::proto::ConstraintBuilderOptions bo;
    bo.sampling_ratio_ = 1.0;
    bo.max_constraint_distance_ = 10.0;
    bo.min_score_ = 0.3;
    bo.global_localization_min_score_ = 0.3;
    bo.fast2d_ = options;   // 1 m / 0.3 rad window, depth 4
    common::InlineThreadPool pool;
    for (int refine = 0; refine < 2; ++refine) {
      for (int side = 0; side < 2; ++side) {
        ConstraintBuilder2D builder(bo, &pool);
        builder.set_device_refinement(refine == 1);
        // two rounds, with DeleteScanMatcher in between: the second rebuilds both stacks
        for (int round = 0; round < 2; ++round) {
          for (int n = 0; n < 2; ++n) {
            for (int s = 0; s < 2; ++s) {
              const mapping::SubmapId sid{0, s};
              // a start 5 cm and 0.02 rad off the node's true pose
              const transform::Rigid2d relative =
                  local_poses[s].inverse() *
                  transform::Rigid2d({node_xy[n][0] + 0.05, node_xy[n][1] - 0.03}, 0.02);
              if (side == 0)
                builder.MaybeAddConstraint(sid, &dsubs[s], mapping::NodeId{0, n}, &nodes[n],
                                           relative);
              else
                builder.MaybeAddConstraint(sid, &hsubs[s], mapping::NodeId{0, n}, &nodes[n],
                                           relative);
            }
            const mapping::SubmapId gid{0, n};
            if (side == 0)
              builder.MaybeAddGlobalConstraint(gid, &dsubs[n], mapping::NodeId{0, n}, &nodes[n]);
            else
              builder.MaybeAddGlobalConstraint(gid, &hsubs[n], mapping::NodeId{0, n}, &nodes[n]);
            builder.NotifyEndOfNode();
          }
          int calls = 0;
          ConstraintBuilder2D::Result got;
          builder.WhenDone([&](const ConstraintBuilder2D::Result& r) { ++calls; got = r; });
          if (calls != 1 || got.empty() || builder.GetNumFinishedNodes() != 2 * (round + 1))
            return 1;
          for (const auto& c : got) {
            const transform::Rigid3d& z = c.pose.zbar_ij;
            std::printf("RESULT cb2d_device_submaps%s_%s %d %d %d %.17g %.17g %.17g %.17g %lld\n",
                        refine ? "_refined" : "", side == 0 ? "dev" : "host", round,
                        c.submap_id.submap_index, c.node_id.node_index, z.translation().x(),
                        z.translation().y(), z.rotation().w(), z.rotation().z(),
                        static_cast<long long>(builder.last_stats().candidates_scored));
          }
          for (int s = 0; s < 2; ++s) builder.DeleteScanMatcher(mapping::SubmapId{0, s});
        }
      }
    }
    // the handles outlive their builders and are still readable
    std::vector<uint16_t> after;
    cropped[0]->Read(&after);
    if (after != host_grids[0]->correspondence_cost_cells()) return 1;
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
    PrintBytes("grid_to_proto_insert_tsdf2d", grid.ToProto());
  }
  {
    // sensor::VoxelFilter's four overloads and AdaptiveVoxelFilter: every payload carries the
    // point's input index, so the RESULT lines list the kept indices
    const int n = 2000;
    sensor::PointCloud cloud;
    std::vector<float> intensities;
    std::vector<sensor::RangefinderPoint> points;
    sensor::TimedPointCloud timed;
    std::vector<sensor::TimedPointCloudOriginData::RangeMeasurement> measurements;
    for (int i = 0; i < n; ++i) {
      const sensor::RangefinderPoint p{{{float((i * 37) % 101) * 0.05f,
                                         float((i * 53) % 89) * 0.05f, float(i % 13) * 0.1f}}};
      cloud.push_back(p);
      intensities.push_back(float(i));
      points.push_back(p);
      timed.push_back({{{p.position.x(), p.position.y(), p.position.z()}}, float(i)});
      measurements.push_back({timed.back(), 0.f, size_t(i)});
    }
    const sensor::PointCloud with_intensities(cloud.points(), intensities);
    const sensor::PointCloud a = sensor::VoxelFilter(with_intensities, 0.3f);
    std::printf("RESULT vf_cloud");
    for (float v : a.intensities()) std::printf(" %d", int(v));
    std::printf("\n");
    std::printf("RESULT vf_points %zu\n", sensor::VoxelFilter(points, 0.3f).size());
    std::printf("RESULT vf_timed");
    for (const auto& p : sensor::VoxelFilter(timed, 0.2f)) std::printf(" %d", int(p.time));
    std::printf("\n");
    std::printf("RESULT vf_range");
    for (const auto& m : sensor::VoxelFilter(measurements, 0.5f))
      std::printf(" %zu", m.origin_index);
    std::printf("\n");
    sensor::proto::AdaptiveVoxelFilterOptions options;
    options.set_max_length(2.f);
    options.set_min_num_points(150.f);
    options.set_max_range(4.f);
    const sensor::PointCloud b = sensor::AdaptiveVoxelFilter(with_intensities, options);
    std::printf("RESULT vf_adaptive");
    for (float v : b.intensities()) std::printf(" %d", int(v));
    std::printf("\n");
  }
  {
    // io::OutlierRemovingPointsProcessor on three batches streamed three times (the fixture of
    // tests/test_gpu_adapter_outlier_removal.py): a wall at x = 5 and, per batch, a patch in front
    // of it that the other batches' rays cross.  Intensities carry each point's index and colors
    // its index and batch, so the RESULT lines show that the payloads follow the kept points.
    struct Sink : io::PointsProcessor {
      std::vector<std::unique_ptr<io::PointsBatch>> batches;
      void Process(std::unique_ptr<io::PointsBatch> b) override { batches.push_back(std::move(b)); }
      FlushResult Flush() override { return FlushResult::kFinished; }
    } sink;
    auto make = [](int b) {
      auto batch = std::make_unique<io::PointsBatch>();
      batch->origin.v[0] = float(b) * 0.3f;
      batch->origin.v[1] = float(b) * -0.2f;
      batch->origin.v[2] = 1.f;
      for (int i = 0; i < 600; ++i) {
        sensor::RangefinderPoint p;
        if (i < 400) {
          p = {{{5.f, float(i % 20) * 0.1f - 1.f, float(i / 20) * 0.1f}}};
        } else {
          p = {{{2.f + float(b), float(i % 10) * 0.1f - 0.5f, float((i / 10) % 10) * 0.1f}}};
        }
        batch->points.push_back(p);
        batch->intensities.push_back(float(i));
        batch->colors.push_back({float(i), float(b), 0.f});
      }
      return batch;
    };
    io::OutlierRemovingPointsProcessor processor(0.1, 3.0, &sink);
    std::printf("RESULT or_action %s\n",
                io::OutlierRemovingPointsProcessor::kConfigurationFileActionName);
    std::printf("RESULT or_flush");
    for (int pass = 0; pass < 3; ++pass) {
      for (int b = 0; b < 3; ++b) processor.Process(make(b));
      std::printf(" %d", processor.Flush() == io::PointsProcessor::FlushResult::kFinished);
    }
    std::printf("\n");
    for (const auto& batch : sink.batches) {
      std::printf("RESULT or_kept_%d", int(batch->colors.empty() ? -1 : batch->colors[0][1]));
      for (float v : batch->intensities) std::printf(" %d", int(v));
      std::printf("\nRESULT or_colors_%d", int(batch->colors.empty() ? -1 : batch->colors[0][1]));
      for (const auto& c : batch->colors) std::printf(" %d", int(c[0]));
      // 1 where a kept point is the input point its intensity names
      const int b = int(batch->colors.empty() ? 0 : batch->colors[0][1]);
      const auto input = make(b);
      std::printf("\nRESULT or_points_%d", b);
      for (size_t i = 0; i < batch->points.size(); ++i) {
        const auto& q = input->points[int(batch->intensities[i])].position;
        const auto& p = batch->points[i].position;
        std::printf(" %d", p.x() == q.x() && p.y() == q.y() && p.z() == q.z());
      }
      std::printf("\n");
    }
  }
  {
    // io::XRayPointsProcessor on three batches in three floors (the fixture of
    // tests/test_gpu_adapter_xray.py): batch b has start_time b, batch 1 has no colours, floor 0
    // holds times 0..1, floor 1 times 1..2 and floor 2 none.  The stand-in Image writes its
    // cairo words, so the RESULT lines list every floor's pixels.
    struct Writer : io::FileWriter {
      std::map<std::string, std::string>* files;
      std::string name, data;
      bool WriteHeader(const char* d, size_t n) override { data.insert(0, d, n); return true; }
      bool Write(const char* d, size_t n) override { data.append(d, n); return true; }
      bool Close() override { (*files)[name] = data; return true; }
      std::string GetFilename() override { return name; }
    };
    struct Sink : io::PointsProcessor {
      int batches = 0;
      void Process(std::unique_ptr<io::PointsBatch>) override { ++batches; }
      FlushResult Flush() override { return FlushResult::kFinished; }
    } sink;
    std::map<std::string, std::string> files;
    const io::FileWriterFactory factory = [&files](const std::string& name) {
      auto w = std::make_unique<Writer>();
      w->files = &files;
      w->name = name;
      return std::unique_ptr<io::FileWriter>(std::move(w));
    };
    std::vector<mapping::Floor> floors(3);
    floors[0].timespans = {{0, 1}};
    floors[1].timespans = {{1, 2}};
    floors[2].timespans = {{5, 6}};
    const transform::Rigid3f transform({0.5f, -0.25f, 0.125f}, {0.8f, 0.f, 0.6f, 0.f});
    io::XRayPointsProcessor processor(0.25, 1.5, transform, floors,
                                      io::XRayPointsProcessor::DrawTrajectories::kNo, "xray", {},
                                      factory, &sink);
    std::printf("RESULT xr_action %s\n", io::XRayPointsProcessor::kConfigurationFileActionName);
    for (int b = 0; b < 3; ++b) {
      auto batch = std::make_unique<io::PointsBatch>();
      batch->start_time = b;
      for (int i = 0; i < 300; ++i) {
        sensor::RangefinderPoint p{{{float((i * 7) % 23) * 0.1f,
                                     float((i * 11) % 17) * 0.1f - 0.8f,
                                     float(i % 9) * 0.15f + float(b) * 0.2f}}};
        batch->points.push_back(p);
        if (b != 1) {
          batch->colors.push_back(
              {float(i % 10) * 0.1f, float(b) * 0.3f, float((i * 3) % 7) / 7.f});
        }
      }
      processor.Process(std::move(batch));
    }
    std::printf("RESULT xr_flush %d %d\n",
                processor.Flush() == io::PointsProcessor::FlushResult::kFinished, sink.batches);
    const auto box = processor.bounding_box();
    std::printf("RESULT xr_box %d %d %d %d %d %d %d\n", int(box.empty), box.min[0], box.min[1],
                box.min[2], box.max[0], box.max[1], box.max[2]);
    for (const auto& file : files) {
      std::printf("RESULT xr_file_%s", file.first.c_str());
      for (size_t i = 0; i + 4 <= file.second.size(); i += 4) {
        uint32_t word;
        std::memcpy(&word, file.second.data() + i, 4);
        std::printf(" %u", word);
      }
      std::printf("\n");
    }
  }
  {
    // io::ProbabilityGridPointsProcessor (PNG and PB) and io::HybridGridPointsProcessor on the
    // three batches of tests/test_gpu_adapter_points_to_grid.py, which reach past the initial
    // 100 x 100 cells at 5 cm.  The stand-in Image writes its cairo words, so the RESULT lines
    // list the image's pixels and the serialised grids' bytes.
    struct Writer : io::FileWriter {
      std::map<std::string, std::string>* files;
      std::string name, data;
      bool WriteHeader(const char* d, size_t n) override { data.insert(0, d, n); return true; }
      bool Write(const char* d, size_t n) override { data.append(d, n); return true; }
      bool Close() override { (*files)[name] = data; return true; }
      std::string GetFilename() override { return name; }
    };
    struct Sink : io::PointsProcessor {
      int batches = 0;
      void Process(std::unique_ptr<io::PointsBatch>) override { ++batches; }
      FlushResult Flush() override { return FlushResult::kFinished; }
    } sink;
    std::map<std::string, std::string> files;
    const auto writer = [&files](const std::string& name) {
      auto w = std::make_unique<Writer>();
      w->files = &files;
      w->name = name;
      return std::unique_ptr<io::FileWriter>(std::move(w));
    };
    mapping::proto::ProbabilityGridRangeDataInserterOptions2D o2;
    o2.set_hit_probability(0.55);
    o2.set_miss_probability(0.49);
    o2.set_insert_free_space(true);
    mapping::proto::RangeDataInserterOptions3D o3;
    o3.set_hit_probability(0.55);
    o3.set_miss_probability(0.49);
    o3.set_num_free_space_voxels(2);
    o3.set_intensity_threshold(40.f);
    using PG = io::ProbabilityGridPointsProcessor;
    PG png(0.05, o2, PG::DrawTrajectories::kNo, PG::OutputType::kPng, writer("map.png"), {},
           &sink);
    PG pb(0.05, o2, PG::DrawTrajectories::kNo, PG::OutputType::kPb, writer("map.pb"), {}, &sink);
    io::HybridGridPointsProcessor hybrid(0.1, o3, writer("map_3d"), &sink);
    std::printf("RESULT pg_action %s %s\n", PG::kConfigurationFileActionName,
                io::HybridGridPointsProcessor::kConfigurationFileActionName);
    for (int b = 0; b < 3; ++b) {
      io::PointsProcessor* const stages[3] = {&png, &pb, &hybrid};
      for (io::PointsProcessor* stage : stages) {
        auto batch = std::make_unique<io::PointsBatch>();
        const float ox = float(b) * 0.7f - 0.5f, oy = float(b) * -0.4f + 0.2f;
        batch->origin.v[0] = ox;
        batch->origin.v[1] = oy;
        batch->origin.v[2] = 0.25f;
        for (int i = 0; i < 400; ++i) {
          sensor::RangefinderPoint p{{{float((i * 37) % 161 - 80) * 0.05f + ox,
                                       float((i * 53) % 149 - 74) * 0.05f + oy,
                                       float(i % 5) * 0.1f}}};
          batch->points.push_back(p);
        }
        stage->Process(std::move(batch));
      }
    }
    Eigen::Array2i offset;
    const std::unique_ptr<io::Image> image = io::DrawProbabilityGrid(png.probability_grid(),
                                                                     &offset);
    std::printf("RESULT pg_image %d %d %d %d\n", image->width(), image->height(), offset.x(),
                offset.y());
    int finished = 0;
    for (io::PointsProcessor* stage : {static_cast<io::PointsProcessor*>(&png),
                                       static_cast<io::PointsProcessor*>(&pb),
                                       static_cast<io::PointsProcessor*>(&hybrid)})
      finished += stage->Flush() == io::PointsProcessor::FlushResult::kFinished;
    std::printf("RESULT pg_flush %d %d\n", finished, sink.batches);
    std::printf("RESULT pg_file_map.png");
    const std::string& words = files["map.png"];
    for (size_t i = 0; i + 4 <= words.size(); i += 4) {
      uint32_t word;
      std::memcpy(&word, words.data() + i, 4);
      std::printf(" %u", word);
    }
    std::printf("\n");
    PrintBytes("pg_file_map.pb", files["map.pb"]);
    PrintBytes("pg_file_map_3d", files["map_3d"]);
    std::printf("RESULT pg_files %zu\n", files.size());
  }
  if (trimmer_cases::Run() != 0) return 1;
  return 0;
}
