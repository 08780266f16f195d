// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_common.h).
// Flat C entry points so tests/ and bench.py's cpu_baseline leg can drive the
// oracle through ctypes.  Not part of the product; libcsm_b200.so never sees it.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <thread>

#include "oracle_2d.h"
#include "oracle_3d.h"
#include "oracle_ceres2d.h"
#include "oracle_ceres3d.h"

using namespace oracle;

namespace {

ProbabilityGrid MakeGrid(const uint16_t* cells, int nx, int ny, double res, double max_x,
                         double max_y, float min_cost, float max_cost) {
  ProbabilityGrid grid(MapLimits{res, max_x, max_y, CellLimits{nx, ny}}, min_cost, max_cost);
  std::memcpy(grid.cells.data(), cells, sizeof(uint16_t) * static_cast<size_t>(nx) * ny);
  return grid;
}

PointCloud MakeCloud(const float* xyz, int n) {
  PointCloud cloud(n);
  for (int i = 0; i < n; ++i) cloud[i] = Vec3f{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
  return cloud;
}

void FillStats(const MatchStats& s, int64_t* out) {
  if (!out) return;
  out[0] = s.candidates_scored;
  out[1] = s.lowest_resolution_candidates;
  out[2] = s.nodes_expanded;
  out[3] = s.num_scans;
  out[4] = s.best_scan_index;
  out[5] = s.best_x_offset;
  out[6] = s.best_y_offset;
}

struct Fast2DHandle {
  ProbabilityGrid grid;
  FastOptions2D options;
  FastCorrelativeScanMatcher2D matcher;
  Fast2DHandle(ProbabilityGrid g, FastOptions2D o)
      : grid(std::move(g)), options(o), matcher(grid, o) {}
};

struct Frontend2D {
  SearchParameters sp;
  std::vector<DiscreteScan2D> scans;
  std::vector<PointCloud> rotated;
};

}  // namespace

extern "C" {

void orc_value_to_cost_table(float min_cost, float max_cost, float* out65536) {
  const std::vector<float> t = PrecomputeValueToBoundedFloat(0, max_cost, min_cost, max_cost);
  std::memcpy(out65536, t.data(), sizeof(float) * 65536);
}
uint16_t orc_probability_to_value(float p) { return ProbabilityToValue(p); }
uint16_t orc_correspondence_cost_to_value(float c) { return CorrespondenceCostToValue(c); }
float orc_constant(int which) {
  switch (which) {
    case 0: return kMinProbability;
    case 1: return kMaxProbability;
    case 2: return kMinCorrespondenceCost;
    case 3: return kMaxCorrespondenceCost;
  }
  return 0.f;
}

void orc_get_cell_index(double res, double max_x, double max_y, float px, float py, int32_t* out2) {
  const MapLimits l{res, max_x, max_y, CellLimits{1, 1}};
  const Array2i c = l.GetCellIndex(px, py);
  out2[0] = c.x;
  out2[1] = c.y;
}

// SearchParameters(linear, angular, cloud, resolution)
void orc_search_params(double lin, double ang, const float* xyz, int n, double res,
                       int32_t* num_angular, double* step, int32_t* num_scans,
                       int32_t* num_linear) {
  const SearchParameters sp(lin, ang, MakeCloud(xyz, n), res);
  *num_angular = sp.num_angular_perturbations;
  *step = sp.angular_perturbation_step_size;
  *num_scans = sp.num_scans;
  *num_linear = sp.linear_bounds.empty() ? 0 : sp.linear_bounds[0].max_x;
}

// Candidate2D(scan, xo, yo, SearchParameters(num_lin, num_ang, step, res)) -> x, y, orientation
void orc_candidate(int num_lin, int num_ang, double step, double res, int scan, int xo, int yo,
                   double* out3) {
  const SearchParameters sp(num_lin, num_ang, step, res);
  const Candidate2D c(scan, xo, yo, sp);
  out3[0] = c.x;
  out3[1] = c.y;
  out3[2] = c.orientation;
}

// GenerateRotatedScans with the "for testing" SearchParameters ctor.
void orc_generate_rotated_scans(const float* xyz, int n, int num_ang, double step,
                                float* out /* (2*num_ang+1) * n * 3 */) {
  const SearchParameters sp(0, num_ang, step, 0.);
  const std::vector<PointCloud> scans = GenerateRotatedScans(MakeCloud(xyz, n), sp);
  size_t k = 0;
  for (const PointCloud& s : scans)
    for (const Vec3f& p : s) {
      out[k++] = p.x;
      out[k++] = p.y;
      out[k++] = p.z;
    }
}

void orc_discretize_scans(double res, double max_x, double max_y, int nx, int ny,
                          const float* scans_xyz, int num_scans, int n, float tx, float ty,
                          int32_t* out /* S*n*2 */) {
  const MapLimits l{res, max_x, max_y, CellLimits{nx, ny}};
  std::vector<PointCloud> scans;
  for (int s = 0; s < num_scans; ++s) scans.push_back(MakeCloud(scans_xyz + 3 * size_t(s) * n, n));
  const std::vector<DiscreteScan2D> d = DiscretizeScans(l, scans, tx, ty);
  size_t k = 0;
  for (const DiscreteScan2D& s : d)
    for (const Array2i& c : s) {
      out[k++] = c.x;
      out[k++] = c.y;
    }
}

// The matcher front-end exactly as MatchWithSearchParameters runs it
// (fast...2d.cc:236-247): rotate by initial yaw, rotated scans, discretise,
// ShrinkToFit.  `full` selects the MatchFullSubmap window/centre (:210-225).
void* orc_frontend2d_create(double res, double max_x, double max_y, int nx, int ny,
                            const float* xyz, int n, const double* init_pose, int full,
                            double lin, double ang, int rt_mode) {
  const MapLimits l{res, max_x, max_y, CellLimits{nx, ny}};
  const PointCloud cloud = MakeCloud(xyz, n);
  Rigid2d init{init_pose[0], init_pose[1], init_pose[2]};
  if (full) {
    lin = 1e6 * res;
    ang = M_PI;
    init = Rigid2d{max_x - 0.5 * res * ny, max_y - 0.5 * res * nx, 0.};
  }
  const PointCloud rotated = TransformPointCloudRotZ(cloud, static_cast<float>(init.theta));
  // RT matcher builds SearchParameters from the rotated cloud (real_time...cc:128-130),
  // the fast matcher from the unrotated one (fast...cc:202-204).
  SearchParameters sp(lin, ang, rt_mode ? rotated : cloud, res);
  std::vector<PointCloud> rs = GenerateRotatedScans(rotated, sp);
  std::vector<DiscreteScan2D> ds =
      DiscretizeScans(l, rs, static_cast<float>(init.x), static_cast<float>(init.y));
  if (!rt_mode) sp.ShrinkToFit(ds, l.cell_limits);
  return new Frontend2D{std::move(sp), std::move(ds), std::move(rs)};
}
int orc_frontend2d_num_scans(void* h) { return static_cast<Frontend2D*>(h)->sp.num_scans; }
double orc_frontend2d_step(void* h) {
  return static_cast<Frontend2D*>(h)->sp.angular_perturbation_step_size;
}
void orc_frontend2d_get(void* h, int32_t* dscans /* S*n*2 */, int32_t* bounds /* S*4 */,
                        float* rotated_xyz /* S*n*3 or null */) {
  Frontend2D* f = static_cast<Frontend2D*>(h);
  size_t k = 0;
  for (const DiscreteScan2D& s : f->scans)
    for (const Array2i& c : s) {
      dscans[k++] = c.x;
      dscans[k++] = c.y;
    }
  for (int i = 0; i < f->sp.num_scans; ++i) {
    bounds[4 * i + 0] = f->sp.linear_bounds[i].min_x;
    bounds[4 * i + 1] = f->sp.linear_bounds[i].max_x;
    bounds[4 * i + 2] = f->sp.linear_bounds[i].min_y;
    bounds[4 * i + 3] = f->sp.linear_bounds[i].max_y;
  }
  if (rotated_xyz) {
    k = 0;
    for (const PointCloud& s : f->rotated)
      for (const Vec3f& p : s) {
        rotated_xyz[k++] = p.x;
        rotated_xyz[k++] = p.y;
        rotated_xyz[k++] = p.z;
      }
  }
}
void orc_frontend2d_destroy(void* h) { delete static_cast<Frontend2D*>(h); }

// PrecomputationGrid2D of one width; out has (nx+w-1)*(ny+w-1) bytes.
void orc_precompute_grid2d(const uint16_t* cells, int nx, int ny, float min_cost, float max_cost,
                           int width, uint8_t* out) {
  const ProbabilityGrid grid = MakeGrid(cells, nx, ny, 0.05, 0., 0., min_cost, max_cost);
  std::vector<float> tmp;
  const PrecomputationGrid2D pg(grid, grid.limits.cell_limits, width, &tmp);
  std::memcpy(out, pg.cells().data(), pg.cells().size());
}

void* orc_fast2d_create(const uint16_t* cells, int nx, int ny, double res, double max_x,
                        double max_y, float min_cost, float max_cost, double lin, double ang,
                        int depth) {
  return new Fast2DHandle(MakeGrid(cells, nx, ny, res, max_x, max_y, min_cost, max_cost),
                          FastOptions2D{lin, ang, depth});
}
void orc_fast2d_destroy(void* h) { delete static_cast<Fast2DHandle*>(h); }

int orc_fast2d_match(void* h, const float* xyz, int n, const double* init_pose, int full,
                     float min_score, float* score, double* pose_out, int64_t* stats_out) {
  Fast2DHandle* m = static_cast<Fast2DHandle*>(h);
  const PointCloud cloud = MakeCloud(xyz, n);
  MatchStats stats;
  Rigid2d pose{0, 0, 0};
  float s = 0.f;
  bool found;
  if (full) {
    found = m->matcher.MatchFullSubmap(cloud, min_score, &s, &pose, &stats);
  } else {
    found = m->matcher.Match(Rigid2d{init_pose[0], init_pose[1], init_pose[2]}, cloud,
                             min_score, &s, &pose, &stats);
  }
  if (found) {
    *score = s;
    pose_out[0] = pose.x;
    pose_out[1] = pose.y;
    pose_out[2] = pose.theta;
  }
  FillStats(stats, stats_out);
  return found ? 1 : 0;
}

// ScoreCandidates at one stack level, unsorted, plus the raw integer sums.
void orc_fast2d_score_candidates(void* h, int level, const int32_t* dscans, int num_scans, int n,
                                 const int32_t* cand /* C*3: scan, xo, yo */, int num_cand,
                                 float* scores, int32_t* sums) {
  Fast2DHandle* m = static_cast<Fast2DHandle*>(h);
  const PrecomputationGrid2D& pg = m->matcher.stack().Get(level);
  for (int c = 0; c < num_cand; ++c) {
    const int32_t* d = dscans + 2 * size_t(cand[3 * c]) * n;
    int sum = 0;
    for (int p = 0; p < n; ++p)
      sum += pg.GetValue(Array2i{d[2 * p] + cand[3 * c + 1], d[2 * p + 1] + cand[3 * c + 2]});
    if (sums) sums[c] = sum;
    scores[c] = pg.ToScore(sum / static_cast<float>(n));
  }
  (void)num_scans;
}

void orc_fast2d_level(void* h, int level, uint8_t* out, int32_t* wide_nx, int32_t* wide_ny) {
  Fast2DHandle* m = static_cast<Fast2DHandle*>(h);
  const PrecomputationGrid2D& pg = m->matcher.stack().Get(level);
  *wide_nx = pg.wide_limits().num_x_cells;
  *wide_ny = pg.wide_limits().num_y_cells;
  if (out) std::memcpy(out, pg.cells().data(), pg.cells().size());
}

double orc_rt2d_match(const uint16_t* cells, int nx, int ny, double res, double max_x,
                      double max_y, const float* xyz, int n, const double* init_pose, double lin,
                      double ang, double w_t, double w_r, double* pose_out, int64_t* stats_out) {
  const ProbabilityGrid grid =
      MakeGrid(cells, nx, ny, res, max_x, max_y, kMinCorrespondenceCost, kMaxCorrespondenceCost);
  const RealTimeCorrelativeScanMatcher2D matcher(RealTimeOptions{lin, ang, w_t, w_r});
  MatchStats stats;
  Rigid2d pose{0, 0, 0};
  const double score = matcher.Match(Rigid2d{init_pose[0], init_pose[1], init_pose[2]},
                                     MakeCloud(xyz, n), grid, &pose, &stats);
  pose_out[0] = pose.x;
  pose_out[1] = pose.y;
  pose_out[2] = pose.theta;
  FillStats(stats, stats_out);
  return score;
}

double orc_rt2d_match_tsdf(const uint16_t* tsd, const uint16_t* weight, int nx, int ny,
                           double res, double max_x, double max_y, float truncation,
                           float max_weight, const float* xyz, int n, const double* init_pose,
                           double lin, double ang, double w_t, double w_r, double* pose_out,
                           int64_t* stats_out) {
  TSDF2D grid(MapLimits{res, max_x, max_y, CellLimits{nx, ny}}, truncation, max_weight);
  std::memcpy(grid.tsd_cells.data(), tsd, sizeof(uint16_t) * size_t(nx) * ny);
  std::memcpy(grid.weight_cells.data(), weight, sizeof(uint16_t) * size_t(nx) * ny);
  const RealTimeCorrelativeScanMatcher2D matcher(RealTimeOptions{lin, ang, w_t, w_r});
  MatchStats stats;
  Rigid2d pose{0, 0, 0};
  const double score = matcher.Match(Rigid2d{init_pose[0], init_pose[1], init_pose[2]},
                                     MakeCloud(xyz, n), grid, &pose, &stats);
  pose_out[0] = pose.x;
  pose_out[1] = pose.y;
  pose_out[2] = pose.theta;
  FillStats(stats, stats_out);
  return score;
}
// Every candidate's score of the same matches, in generation order, as max_element sees them:
// the first min(cap, count) are written to `scores`; returns the count.
int64_t orc_rt2d_scores(const uint16_t* cells, int nx, int ny, double res, double max_x,
                        double max_y, const float* xyz, int n, const double* init_pose,
                        double lin, double ang, double w_t, double w_r, float* scores,
                        int64_t cap) {
  const ProbabilityGrid grid =
      MakeGrid(cells, nx, ny, res, max_x, max_y, kMinCorrespondenceCost, kMaxCorrespondenceCost);
  const RealTimeCorrelativeScanMatcher2D matcher(RealTimeOptions{lin, ang, w_t, w_r});
  Rigid2d pose{0, 0, 0};
  std::vector<float> all;
  matcher.Match(Rigid2d{init_pose[0], init_pose[1], init_pose[2]}, MakeCloud(xyz, n), grid,
                &pose, nullptr, &all);
  const int64_t count = static_cast<int64_t>(all.size());
  if (scores) std::memcpy(scores, all.data(), sizeof(float) * std::min(cap, count));
  return count;
}

int64_t orc_rt2d_scores_tsdf(const uint16_t* tsd, const uint16_t* weight, int nx, int ny,
                             double res, double max_x, double max_y, float truncation,
                             float max_weight, const float* xyz, int n, const double* init_pose,
                             double lin, double ang, double w_t, double w_r, float* scores,
                             int64_t cap) {
  TSDF2D grid(MapLimits{res, max_x, max_y, CellLimits{nx, ny}}, truncation, max_weight);
  std::memcpy(grid.tsd_cells.data(), tsd, sizeof(uint16_t) * size_t(nx) * ny);
  std::memcpy(grid.weight_cells.data(), weight, sizeof(uint16_t) * size_t(nx) * ny);
  const RealTimeCorrelativeScanMatcher2D matcher(RealTimeOptions{lin, ang, w_t, w_r});
  Rigid2d pose{0, 0, 0};
  std::vector<float> all;
  matcher.Match(Rigid2d{init_pose[0], init_pose[1], init_pose[2]}, MakeCloud(xyz, n), grid,
                &pose, nullptr, &all);
  const int64_t count = static_cast<int64_t>(all.size());
  if (scores) std::memcpy(scores, all.data(), sizeof(float) * std::min(cap, count));
  return count;
}

void orc_tsdf_values(float truncation, float max_weight, float tsd, float w, uint16_t* out2) {
  const TSDF2D g(MapLimits{1., 0., 0., CellLimits{1, 1}}, truncation, max_weight);
  out2[0] = g.TSDToValue(tsd);
  out2[1] = g.WeightToValue(w);
}

// RT ScoreCandidates over an explicit candidate list (test hook,
// real_time_correlative_scan_matcher_2d_test.cc:125-198).
void orc_rt2d_score_candidates(const uint16_t* cells, int nx, int ny, double res, double max_x,
                               double max_y, const int32_t* dscans, int n, int num_lin,
                               int num_ang, double step, double w_t, double w_r,
                               const int32_t* cand, int num_cand, float* scores) {
  const ProbabilityGrid grid =
      MakeGrid(cells, nx, ny, res, max_x, max_y, kMinCorrespondenceCost, kMaxCorrespondenceCost);
  const SearchParameters sp(num_lin, num_ang, step, res);
  std::vector<DiscreteScan2D> ds(sp.num_scans);
  for (int s = 0; s < sp.num_scans; ++s)
    for (int p = 0; p < n; ++p)
      ds[s].push_back(Array2i{dscans[2 * (size_t(s) * n + p)], dscans[2 * (size_t(s) * n + p) + 1]});
  std::vector<Candidate2D> cs;
  for (int c = 0; c < num_cand; ++c)
    cs.emplace_back(cand[3 * c], cand[3 * c + 1], cand[3 * c + 2], sp);
  const RealTimeCorrelativeScanMatcher2D matcher(RealTimeOptions{0., 0., w_t, w_r});
  matcher.ScoreCandidates(grid, ds, sp, &cs);
  for (int c = 0; c < num_cand; ++c) scores[c] = cs[c].score;
}

// CPU baseline: run `num_jobs` fast matches on `threads` worker threads
// (one matcher per job's stack handle, jobs pulled from an atomic counter —
// the oracle-side stand-in for ThreadPool, constraints/constraint_builder_2d.cc:102-111).
// jobs: per job {stack index, cloud index}; returns wall seconds.
double orc_fast2d_batch(void** matchers, const int32_t* job_matcher, const int32_t* job_cloud,
                        const double* job_init_pose /* J*3 */, int num_jobs,
                        const float* const* clouds_xyz, const int32_t* cloud_n, int full,
                        float min_score, int threads, int32_t* found, float* scores,
                        double* poses /* J*3 */, int64_t* cand_scored /* J */) {
  std::atomic<int> next(0);
  auto worker = [&]() {
    for (;;) {
      const int j = next.fetch_add(1);
      if (j >= num_jobs) return;
      int64_t st[8] = {0};
      float s = 0.f;
      double p[3] = {0, 0, 0};
      const int ci = job_cloud[j];
      found[j] = orc_fast2d_match(matchers[job_matcher[j]], clouds_xyz[ci], cloud_n[ci],
                                  job_init_pose + 3 * j, full, min_score, &s, p, st);
      scores[j] = s;
      poses[3 * j] = p[0];
      poses[3 * j + 1] = p[1];
      poses[3 * j + 2] = p[2];
      cand_scored[j] = st[0];
    }
  };
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) pool.emplace_back(worker);
  for (std::thread& t : pool) t.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}


// ===========================================================================
// 3D
// ===========================================================================
namespace {
struct Fast3DHandle {
  const HybridGrid* hi;
  const HybridGrid* lo;
  std::vector<float> histogram;
  FastOptions3D options;
  std::unique_ptr<FastCorrelativeScanMatcher3D> matcher;
};
Rigid3d MakeRigid3d(const double* p) {  // {tx,ty,tz, qw,qx,qy,qz}
  return Rigid3d{Vec3d{p[0], p[1], p[2]}, Quatd{p[3], p[4], p[5], p[6]}};
}
NodeData3D MakeNode(const double* gravity, const float* hi_xyz, int n_hi, const float* lo_xyz,
                    int n_lo, const float* hist, int hist_n) {
  NodeData3D d;
  d.gravity_alignment = Quatd{gravity[0], gravity[1], gravity[2], gravity[3]};
  d.high_resolution_point_cloud = MakeCloud(hi_xyz, n_hi);
  d.low_resolution_point_cloud = MakeCloud(lo_xyz, n_lo);
  d.rotational_scan_matcher_histogram.assign(hist, hist + hist_n);
  return d;
}
}  // namespace

void* orc_hybrid_create(float resolution, const int32_t* idx, const uint16_t* values, int64_t n) {
  HybridGrid* g = new HybridGrid(resolution);
  for (int64_t i = 0; i < n; ++i)
    *g->mutable_value(Array3i{idx[3 * i], idx[3 * i + 1], idx[3 * i + 2]}) = values[i];
  return g;
}
void orc_hybrid_destroy(void* h) { delete static_cast<HybridGrid*>(h); }
int orc_hybrid_grid_size(void* h) { return static_cast<HybridGrid*>(h)->grid_size(); }
void orc_hybrid_get_cell_index(float resolution, const float* p, int32_t* out) {
  const HybridGrid g(resolution);
  const Array3i c = g.GetCellIndex(Vec3f{p[0], p[1], p[2]});
  out[0] = c.x; out[1] = c.y; out[2] = c.z;
}
float orc_hybrid_get_probability(void* h, int x, int y, int z) {
  return static_cast<HybridGrid*>(h)->GetProbability(Array3i{x, y, z});
}

// RealTimeCorrelativeScanMatcher3D::Match (real_time_correlative_scan_matcher_3d.cc:34-53).
// pose in / out = {tx,ty,tz, qw,qx,qy,qz}; stats_out = {num_candidates, best_index}.
float orc_rt3d_match(void* hybrid, const float* xyz, int n, const double* initial_pose,
                     double lin, double ang, double w_t, double w_r, double* pose_out,
                     int64_t* stats_out) {
  const HybridGrid* g = static_cast<HybridGrid*>(hybrid);
  const RealTimeCorrelativeScanMatcher3D matcher(RealTimeOptions3D{lin, ang, w_t, w_r});
  Rigid3d pose{Vec3d{0., 0., 0.}, Quatd{1., 0., 0., 0.}};
  int64_t num = 0, best = -1;
  const float score =
      matcher.Match(MakeRigid3d(initial_pose), MakeCloud(xyz, n), *g, &pose, &num, &best);
  pose_out[0] = pose.t.x; pose_out[1] = pose.t.y; pose_out[2] = pose.t.z;
  pose_out[3] = pose.q.w; pose_out[4] = pose.q.x; pose_out[5] = pose.q.y; pose_out[6] = pose.q.z;
  if (stats_out) { stats_out[0] = num; stats_out[1] = best; }
  return score;
}

// Every candidate's score of the same match in generation order (translations z, y, x, then
// rotations rz, ry, rx): the first min(cap, count) are written to `scores`; returns the count.
int64_t orc_rt3d_scores(void* hybrid, const float* xyz, int n, const double* initial_pose,
                        double lin, double ang, double w_t, double w_r, float* scores,
                        int64_t cap) {
  const HybridGrid* g = static_cast<HybridGrid*>(hybrid);
  const RealTimeCorrelativeScanMatcher3D matcher(RealTimeOptions3D{lin, ang, w_t, w_r});
  Rigid3d pose{Vec3d{0., 0., 0.}, Quatd{1., 0., 0., 0.}};
  std::vector<float> all;
  matcher.Match(MakeRigid3d(initial_pose), MakeCloud(xyz, n), *g, &pose, nullptr, nullptr, &all);
  const int64_t count = static_cast<int64_t>(all.size());
  if (scores) std::memcpy(scores, all.data(), sizeof(float) * std::min(cap, count));
  return count;
}

void* orc_fast3d_create(void* hi, void* lo, const float* hist, int hist_n, int bb_depth,
                        int full_res_depth, double min_rot, double min_low, double lin_xy,
                        double lin_z, double ang) {
  Fast3DHandle* f = new Fast3DHandle;
  f->hi = static_cast<HybridGrid*>(hi);
  f->lo = static_cast<HybridGrid*>(lo);
  f->histogram.assign(hist, hist + hist_n);
  f->options = FastOptions3D{bb_depth, full_res_depth, min_rot, min_low, lin_xy, lin_z, ang};
  f->matcher.reset(new FastCorrelativeScanMatcher3D(*f->hi, f->lo, &f->histogram, f->options));
  return f;
}
void orc_fast3d_destroy(void* h) { delete static_cast<Fast3DHandle*>(h); }

// Dense dump of one precomputation level over its bounding box.  out may be null
// (query lo/dims first).  Layout: ((z - lo.z) * dims.y + (y - lo.y)) * dims.x + (x - lo.x).
void orc_fast3d_level(void* h, int depth, int32_t* lo, int32_t* dims, uint8_t* out) {
  Fast3DHandle* f = static_cast<Fast3DHandle*>(h);
  const PrecomputationGrid3D& g = f->matcher->stack().Get(depth);
  int mn[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, mx[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  g.ForEach([&](const Array3i& c, uint8_t) {
    mn[0] = std::min(mn[0], c.x); mn[1] = std::min(mn[1], c.y); mn[2] = std::min(mn[2], c.z);
    mx[0] = std::max(mx[0], c.x); mx[1] = std::max(mx[1], c.y); mx[2] = std::max(mx[2], c.z);
  });
  if (mn[0] > mx[0]) { for (int i = 0; i < 3; ++i) { lo[i] = 0; dims[i] = 0; } return; }
  if (!out) {
    for (int i = 0; i < 3; ++i) { lo[i] = mn[i]; dims[i] = mx[i] - mn[i] + 1; }
    return;
  }
  // caller passes the lo/dims it wants dumped (may be larger than the bbox)
  const int64_t nx = dims[0], ny = dims[1];
  std::memset(out, 0, static_cast<size_t>(dims[0]) * dims[1] * dims[2]);
  g.ForEach([&](const Array3i& c, uint8_t v) {
    const int64_t x = c.x - lo[0], y = c.y - lo[1], z = c.z - lo[2];
    if (x >= 0 && y >= 0 && z >= 0 && x < dims[0] && y < dims[1] && z < dims[2])
      out[(z * ny + y) * nx + x] = v;
  });
}

int orc_fast3d_match(void* h, int full, const double* node_pose, const double* submap_pose,
                     const double* gravity, const float* hi_xyz, int n_hi, const float* lo_xyz,
                     int n_lo, const float* hist, int hist_n, float min_score, float* score,
                     double* pose_out, float* rot_score, float* low_score, int64_t* stats_out) {
  Fast3DHandle* f = static_cast<Fast3DHandle*>(h);
  const NodeData3D data = MakeNode(gravity, hi_xyz, n_hi, lo_xyz, n_lo, hist, hist_n);
  MatchStats3D st;
  std::unique_ptr<Result3D> r;
  if (full) {
    const Rigid3d n = MakeRigid3d(node_pose), s = MakeRigid3d(submap_pose);
    r = f->matcher->MatchFullSubmap(n.q, s.q, data, min_score, &st);
  } else {
    r = f->matcher->Match(MakeRigid3d(node_pose), MakeRigid3d(submap_pose), data, min_score, &st);
  }
  if (stats_out) {
    stats_out[0] = st.candidates_scored;
    stats_out[1] = st.lowest_resolution_candidates;
    stats_out[2] = st.nodes_expanded;
    stats_out[3] = st.low_resolution_evaluations;
    stats_out[4] = st.num_scans;
    stats_out[5] = st.num_angles;
    stats_out[6] = st.best_scan_index;
    stats_out[7] = st.best_x;
    stats_out[8] = st.best_y;
    stats_out[9] = st.best_z;
  }
  if (!r) return 0;
  *score = r->score;
  pose_out[0] = r->pose_estimate.t.x; pose_out[1] = r->pose_estimate.t.y;
  pose_out[2] = r->pose_estimate.t.z; pose_out[3] = r->pose_estimate.q.w;
  pose_out[4] = r->pose_estimate.q.x; pose_out[5] = r->pose_estimate.q.y;
  pose_out[6] = r->pose_estimate.q.z;
  *rot_score = r->rotational_score;
  *low_score = r->low_resolution_score;
  return 1;
}

// Discrete scans of a match (test hook).  cells may be null to query num_scans.
int orc_fast3d_discrete_scans(void* h, int full, const double* node_pose,
                              const double* submap_pose, const double* gravity,
                              const float* hi_xyz, int n_hi, const float* hist, int hist_n,
                              int32_t* cells /* S*n*3 */, float* poses /* S*7 */,
                              float* rot_scores /* S */) {
  Fast3DHandle* f = static_cast<Fast3DHandle*>(h);
  const NodeData3D data = MakeNode(gravity, hi_xyz, n_hi, hi_xyz, 0, hist, hist_n);
  const auto scans = f->matcher->GenerateDiscreteScansForTest(
      full != 0, MakeRigid3d(node_pose), MakeRigid3d(submap_pose), data);
  if (cells) {
    size_t k = 0;
    for (size_t s = 0; s < scans.size(); ++s) {
      for (const Array3i& c : scans[s].cell_indices_per_depth[0]) {
        cells[k++] = c.x; cells[k++] = c.y; cells[k++] = c.z;
      }
      const Rigid3f& p = scans[s].pose;
      const float v[7] = {p.t.x, p.t.y, p.t.z, p.q.w, p.q.x, p.q.y, p.q.z};
      std::memcpy(poses + 7 * s, v, sizeof(v));
      rot_scores[s] = scans[s].rotational_score;
    }
  }
  return static_cast<int>(scans.size());
}

// ScoreCandidates of caller-given candidates (n x {scan, x, y, z}) at `depth` on the same
// discrete scans (test hook): sums, scores and, at depth 0, low-resolution scores (may be null).
void orc_fast3d_score_candidates(void* h, int full, const double* node_pose,
                                 const double* submap_pose, const double* gravity,
                                 const float* hi_xyz, int n_hi, const float* lo_xyz, int n_lo,
                                 const float* hist, int hist_n, int depth,
                                 const int32_t* candidates, int n, int32_t* sums, float* scores,
                                 float* low_scores) {
  Fast3DHandle* f = static_cast<Fast3DHandle*>(h);
  const NodeData3D data = MakeNode(gravity, hi_xyz, n_hi, lo_xyz, n_lo, hist, hist_n);
  std::vector<std::array<int, 4>> c(n);
  for (int i = 0; i < n; ++i)
    c[i] = {candidates[4 * i], candidates[4 * i + 1], candidates[4 * i + 2], candidates[4 * i + 3]};
  std::vector<int> s(n);
  f->matcher->ScoreCandidatesForTest(full != 0, MakeRigid3d(node_pose), MakeRigid3d(submap_pose),
                                     data, depth, c, s.data(), scores, low_scores);
  std::copy(s.begin(), s.end(), sums);
}

void orc_rotational_match(const float* submap_hist, const float* hist, int n, float initial_angle,
                          const float* angles, int m, float* out) {
  const std::vector<float> a(submap_hist, submap_hist + n), b(hist, hist + n);
  const std::vector<float> r =
      RotationalMatch(a, b, initial_angle, std::vector<float>(angles, angles + m));
  std::memcpy(out, r.data(), sizeof(float) * m);
}

// ---- CeresScanMatcher2D restatement (oracle_ceres2d.h) ---------------------------
// opts = {occupied_space_weight, translation_weight, rotation_weight,
//         use_nonmonotonic_steps, max_num_iterations}
static CeresScanMatcherOptions2D CeresOpts(const double* o) {
  CeresScanMatcherOptions2D opt;
  opt.occupied_space_weight = o[0];
  opt.translation_weight = o[1];
  opt.rotation_weight = o[2];
  opt.use_nonmonotonic_steps = o[3] != 0.;
  opt.max_num_iterations = static_cast<int>(o[4]);
  return opt;
}

// residuals: n + 3; jacobian: (n + 3) x 3 row-major, or NULL for the plain-double path
void orc_ceres2d_evaluate(const uint16_t* cells, int nx, int ny, double res, double max_x,
                          double max_y, const float* xyz, int n, const double* opts,
                          const double* target_xy, double target_angle, const double* pose,
                          double* residuals, double* jacobian) {
  const ProbabilityGrid grid =
      MakeGrid(cells, nx, ny, res, max_x, max_y, kMinCorrespondenceCost, kMaxCorrespondenceCost);
  std::vector<double> r, j;
  EvaluateCeresResiduals2D(grid, MakeCloud(xyz, n), CeresOpts(opts), target_xy, target_angle,
                           pose, &r, jacobian ? &j : nullptr);
  std::memcpy(residuals, r.data(), sizeof(double) * r.size());
  if (jacobian) std::memcpy(jacobian, j.data(), sizeof(double) * j.size());
}

// summary_out = {initial_cost, final_cost, iterations, num_successful_steps, termination}
void orc_ceres2d_match(const uint16_t* cells, int nx, int ny, double res, double max_x,
                       double max_y, const float* xyz, int n, const double* opts,
                       const double* target_xy, const double* init_pose, double* pose_out,
                       double* summary_out) {
  const ProbabilityGrid grid =
      MakeGrid(cells, nx, ny, res, max_x, max_y, kMinCorrespondenceCost, kMaxCorrespondenceCost);
  CeresSummary2D sum;
  CeresMatch2D(grid, MakeCloud(xyz, n), CeresOpts(opts), target_xy, init_pose, pose_out, &sum);
  summary_out[0] = sum.initial_cost;
  summary_out[1] = sum.final_cost;
  summary_out[2] = sum.iterations;
  summary_out[3] = sum.num_successful_steps;
  summary_out[4] = sum.termination;
}

// orc_ceres2d_match with the per-iteration trace: returns the number of records and writes
// at most `cap` of them (kCeresTraceDoubles doubles each, PackCeresTrace's order) to `trace`.
int orc_ceres2d_match_traced(const uint16_t* cells, int nx, int ny, double res, double max_x,
                             double max_y, const float* xyz, int n, const double* opts,
                             const double* target_xy, const double* init_pose, double* pose_out,
                             double* summary_out, double* trace, int cap) {
  const ProbabilityGrid grid =
      MakeGrid(cells, nx, ny, res, max_x, max_y, kMinCorrespondenceCost, kMaxCorrespondenceCost);
  CeresSummary2D sum;
  std::vector<CeresIterationTrace> records;
  CeresMatch2D(grid, MakeCloud(xyz, n), CeresOpts(opts), target_xy, init_pose, pose_out, &sum,
               &records);
  summary_out[0] = sum.initial_cost;
  summary_out[1] = sum.final_cost;
  summary_out[2] = sum.iterations;
  summary_out[3] = sum.num_successful_steps;
  summary_out[4] = sum.termination;
  if (static_cast<int>(records.size()) <= cap) PackCeresTrace(records, trace);
  return static_cast<int>(records.size());
}

// ---- CeresScanMatcher3D restatement (oracle_ceres3d.h) ---------------------------
// opts = {translation_weight, rotation_weight, use_nonmonotonic_steps, max_num_iterations,
//         occupied_space_weight_0, occupied_space_weight_1, ...}
static CeresScanMatcherOptions3D CeresOpts3(const double* o, int num_clouds) {
  CeresScanMatcherOptions3D opt;
  opt.translation_weight = o[0];
  opt.rotation_weight = o[1];
  opt.use_nonmonotonic_steps = o[2] != 0.;
  opt.max_num_iterations = static_cast<int>(o[3]);
  opt.occupied_space_weight.assign(o + 4, o + 4 + num_clouds);
  return opt;
}

double orc_interpolated_probability(void* hybrid, double x, double y, double z, double* gradient) {
  return InterpolatedProbability(*static_cast<HybridGrid*>(hybrid), x, y, z, gradient);
}

namespace {
struct Clouds3 {
  std::vector<PointCloud> clouds;
  std::vector<PointCloudAndHybridGrid> pairs;
  Clouds3(void** hybrids, const float* const* xyz, const int32_t* n, int num) {
    clouds.reserve(num);
    for (int b = 0; b < num; ++b) clouds.push_back(MakeCloud(xyz[b], n[b]));
    for (int b = 0; b < num; ++b)
      pairs.push_back(PointCloudAndHybridGrid{&clouds[b], static_cast<HybridGrid*>(hybrids[b])});
  }
};
}  // namespace

// residuals: sum(n) + 6; jacobian: rows x 6 (tangent space) or NULL
void orc_ceres3d_evaluate(void** hybrids, const float* const* xyz, const int32_t* n,
                          int num_clouds, const double* opts, const double* target_t,
                          const double* target_q, const double* pose, double* residuals,
                          double* jacobian) {
  const Clouds3 c(hybrids, xyz, n, num_clouds);
  std::vector<double> r, j;
  EvaluateCeresResiduals3D(c.pairs, CeresOpts3(opts, num_clouds), target_t, target_q, pose, &r,
                           jacobian ? &j : nullptr);
  std::memcpy(residuals, r.data(), sizeof(double) * r.size());
  if (jacobian) std::memcpy(jacobian, j.data(), sizeof(double) * j.size());
}

void orc_ceres3d_match(void** hybrids, const float* const* xyz, const int32_t* n, int num_clouds,
                       const double* opts, const double* target_t, const double* init_pose,
                       double* pose_out, double* summary_out) {
  const Clouds3 c(hybrids, xyz, n, num_clouds);
  CeresSummary2D sum;
  CeresMatch3D(c.pairs, CeresOpts3(opts, num_clouds), target_t, init_pose, pose_out, &sum);
  summary_out[0] = sum.initial_cost;
  summary_out[1] = sum.final_cost;
  summary_out[2] = sum.iterations;
  summary_out[3] = sum.num_successful_steps;
  summary_out[4] = sum.termination;
}

// as orc_ceres2d_match_traced
int orc_ceres3d_match_traced(void** hybrids, const float* const* xyz, const int32_t* n,
                             int num_clouds, const double* opts, const double* target_t,
                             const double* init_pose, double* pose_out, double* summary_out,
                             double* trace, int cap) {
  const Clouds3 c(hybrids, xyz, n, num_clouds);
  CeresSummary2D sum;
  std::vector<CeresIterationTrace> records;
  CeresMatch3D(c.pairs, CeresOpts3(opts, num_clouds), target_t, init_pose, pose_out, &sum,
               &records);
  summary_out[0] = sum.initial_cost;
  summary_out[1] = sum.final_cost;
  summary_out[2] = sum.iterations;
  summary_out[3] = sum.num_successful_steps;
  summary_out[4] = sum.termination;
  if (static_cast<int>(records.size()) <= cap) PackCeresTrace(records, trace);
  return static_cast<int>(records.size());
}

}  // extern "C"
