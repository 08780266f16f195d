/* csm_abi.h — C ABI of the H100 correlative scan-matching engine (libcsm_b200.so).
 *
 * This is the drop-in boundary: the entry points a maintainer of
 * cartographer-project/cartographer binds behind the existing C++ classes
 *   cartographer::mapping::scan_matching::FastCorrelativeScanMatcher2D
 *   cartographer::mapping::scan_matching::RealTimeCorrelativeScanMatcher2D
 *   cartographer::mapping::scan_matching::FastCorrelativeScanMatcher3D
 *   cartographer::mapping::constraints::ConstraintBuilder2D / 3D
 * (see INTEGRATION.md for the adapter code).  Plain pointers and sizes only;
 * no C++ / torch / CUDA types cross the boundary.
 *
 * Conventions
 *  - every function returns a csm_status (0 == CSM_OK); nothing aborts or
 *    throws across the ABI (the reference CHECK-aborts on programmer errors,
 *    e.g. fast_correlative_scan_matcher_2d.cc:232-233; here they become
 *    CSM_E_INVALID);  csm_last_error_string() describes the last failure of
 *    the calling thread.
 *  - "no pose above min_score" is NOT an error: *found == 0 and the outputs
 *    are left untouched (fast_correlative_scan_matcher_2d.cc:253-261).
 *  - opaque handles own device memory; the caller owns every host buffer and
 *    may free it as soon as the call returns.
 *  - all entry points are thread-safe (per-device serialisation inside);
 *    Match* may be called concurrently on one stack, as the reference's pool
 *    threads do (constraints/constraint_builder_2d.cc:102-111).
 *  - there is no CPU fallback: without a usable CUDA device every call
 *    returns CSM_E_CUDA.
 *
 * File:line citations are relative to the reference repository's cartographer/ .
 */
#ifndef CSM_ABI_H_
#define CSM_ABI_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t csm_status;
enum {
  CSM_OK = 0,
  CSM_E_INVALID = 1,      /* bad argument (reference: glog CHECK) */
  CSM_E_CUDA = 2,         /* CUDA runtime / no device */
  CSM_E_CAPACITY = 3,     /* internal capacity exceeded (e.g. > 2^20 exactly tied optima) */
  CSM_E_INTERNAL = 4
};

/* Per-call counters.  `candidates_scored` counts one per candidate whose score
 * the engine computed (all levels) — the unit of BASELINE.json's metric. */
typedef struct csm_stats {
  int64_t candidates_scored;
  int64_t lowest_resolution_candidates; /* == reference's top-level list size */
  int64_t nodes_expanded;               /* B&B parents whose children were scored */
  int64_t leaves_tied;                  /* leaves sharing the best score (1 == unique) */
  int32_t num_scans;                    /* SearchParameters::num_scans */
  int32_t best_scan_index;              /* winning Candidate2D identity (integers) */
  int32_t best_x_offset;
  int32_t best_y_offset;
  int32_t host_tie_resolves;            /* top-level std::sort replays (see DESIGN.md) */
  int32_t host_syncs;                   /* stream synchronisations inside the call (2D batch: 1 + ties) */
  float device_ms;                      /* CUDA-event time of the device work of this call */
  float collective_ms;                  /* host wall time inside the ncclAllGather step (csm_cb_batch*_run) */
} csm_stats;

/* ---- device / context ---------------------------------------------------- */
csm_status csm_device_count(int32_t* count);
const char* csm_last_error_string(void);
/* Number of kernel launches issued by this process so far (bench `gpu_launches`). */
int64_t csm_kernel_launch_count(void);

/* Per-kernel device timing for bench.py's roofline block: CUDA events on the
 * engine's stream around every kernel launch (adds a sync per launch; off by
 * default).  csm_profile_read writes "<kernel> <launches> <total_ms> <units>"
 * lines, units = scored candidates (or cells) the launches processed. */
csm_status csm_profile_enable(int32_t on);
csm_status csm_profile_read(char* buf, int32_t capacity);

/* ---- 2D precomputation grid stack ---------------------------------------- */
/* Replaces FastCorrelativeScanMatcher2D's ctor
 * (internal/2d/scan_matching/fast_correlative_scan_matcher_2d.cc:188-194), i.e.
 * PrecomputationGridStack2D (:171-186) over a Grid2D.  `cells` is
 * Grid2D::correspondence_cost_cells() (uint16, flat index num_x*y + x,
 * 2d/grid_2d.h:113-116); min/max_cost are Grid2D::Get{Min,Max}CorrespondenceCost().
 * Like the reference ctor it copies what it needs; `cells` is not retained. */
typedef struct csm_stack2d csm_stack2d;
csm_status csm_stack2d_create(const uint16_t* cells, int32_t num_x_cells, int32_t num_y_cells,
                              double resolution, double max_x, double max_y,
                              float min_correspondence_cost, float max_correspondence_cost,
                              int32_t branch_and_bound_depth, int32_t device,
                              csm_stack2d** out);
csm_status csm_stack2d_destroy(csm_stack2d* stack);
/* Test hook: PrecomputationGrid2D::cells_ of one level, row-major
 * (x + y * wide_num_x), fast_correlative_scan_matcher_2d.h:56-71,92.
 * `out` may be NULL to query the dimensions only. */
csm_status csm_stack2d_read_level(const csm_stack2d* stack, int32_t level, uint8_t* out,
                                  int32_t* wide_num_x, int32_t* wide_num_y);

/* Incremental refresh of a stack whose submap grid received new range data (same cell
 * limits and cost bounds): rebuilds every device layout in place.  No match may be in
 * flight on the stack. */
csm_status csm_stack2d_update(csm_stack2d* stack, const uint16_t* cells);

/* ---- ingest from Cartographer's serialized forms ---------------------------- */
/* Builds the stack straight from a serialized cartographer.mapping.proto.Grid2D
 * (mapping/proto/grid_2d.proto:23-42; what Submap2D::ToProto / a .pbstream holds), with
 * the semantics of Grid2D::Grid2D(const proto::Grid2D&) (mapping/2d/grid_2d.cc:75-96,
 * legacy default bounds :24-44).  No protobuf runtime is involved. */
csm_status csm_stack2d_create_from_proto(const uint8_t* serialized_grid2d, int64_t size,
                                         int32_t branch_and_bound_depth, int32_t device,
                                         csm_stack2d** out);
/* Host-only decode of the same message (usable without a GPU; cells may be NULL). */
typedef struct csm_grid2d_info {
  int32_t num_x_cells, num_y_cells;
  double resolution, max_x, max_y;
  float min_correspondence_cost, max_correspondence_cost;
  int32_t is_tsdf;
  int32_t reserved;
} csm_grid2d_info;
csm_status csm_grid2d_proto_decode(const uint8_t* serialized_grid2d, int64_t size,
                                   csm_grid2d_info* info, uint16_t* cells,
                                   int64_t cells_capacity);
/* Walks a .pbstream (io/proto_stream.cc:27-110: magic, then [u64 size, gzip blob]*; the
 * blobs after the header are proto::SerializedData, mapping/proto/serialization.proto) and
 * builds one stack per 2D submap in file order.  submap_ids (may be NULL) receives
 * {trajectory_id, submap_index} pairs.  *num_loaded is the number of 2D submaps in the
 * file; if it exceeds max_stacks only the first max_stacks were built. */
csm_status csm_pbstream_load_stacks2d(const char* path, int32_t branch_and_bound_depth,
                                      int32_t device, int32_t max_stacks, csm_stack2d** stacks,
                                      int32_t* submap_ids, int32_t* num_loaded);

/* ---- device-resident scan (sensor::PointCloud) --------------------------- */
/* A PointCloud (sensor/point_cloud.h:33-92: N x {x,y,z} float32) copied to the
 * device once so that many matches can borrow it (ConstraintBuilder matches one
 * node scan against many submaps). */
typedef struct csm_cloud csm_cloud;
csm_status csm_cloud_create(const float* xyz, int32_t num_points, int32_t device,
                            csm_cloud** out);
csm_status csm_cloud_destroy(csm_cloud* cloud);

/* ---- FastCorrelativeScanMatcher2D::Match / MatchFullSubmap ---------------- */
/* fast_correlative_scan_matcher_2d.cc:198-262.  full_submap != 0 ignores
 * initial_pose and the two windows (MatchFullSubmap, :210-225).
 * initial_pose / pose_estimate = {x, y, yaw} of a transform::Rigid2d. */
csm_status csm_match2d(const csm_stack2d* stack, const float* xyz, int32_t num_points,
                       const double initial_pose[3], int32_t full_submap,
                       double linear_search_window, double angular_search_window,
                       float min_score, int32_t* found, float* score,
                       double pose_estimate[3], csm_stats* stats /* may be NULL */);

/* One (submap, node) search of ConstraintBuilder2D::ComputeConstraint
 * (constraints/constraint_builder_2d.cc:188-277, the part before Ceres). */
typedef struct csm_job2d {
  int32_t stack_index;   /* into stacks[] */
  int32_t cloud_index;   /* into clouds[] */
  int32_t full_submap;   /* MaybeAddGlobalConstraint (:114-137) vs MaybeAddConstraint */
  int32_t reserved;
  double initial_pose[3];
  float min_score;       /* options.min_score() / global_localization_min_score() */
  float reserved_f;
} csm_job2d;

typedef struct csm_result2d {
  int32_t found;
  float score;
  double pose_estimate[3];
  int32_t best_scan_index, best_x_offset, best_y_offset;
  int32_t leaves_tied;
} csm_result2d;

/* Batched form: every job is an independent FastCorrelativeScanMatcher2D match;
 * all stacks and clouds must live on the same device.  Results are written in
 * job order.  This is the entry ConstraintBuilder2D's queue drains into. */
csm_status csm_match2d_batch(const csm_stack2d* const* stacks, int32_t num_stacks,
                             const csm_cloud* const* clouds, int32_t num_clouds,
                             const csm_job2d* jobs, int32_t num_jobs,
                             double linear_search_window, double angular_search_window,
                             csm_result2d* results, csm_stats* total /* may be NULL */);

/* Limits of the batched 2D branch-and-bound sweep.  csm_sweep_limits2d_default gives the
 * values csm_match2d_batch runs with (lattice_min and unroll follow CSM_NO_LATTICE and
 * CSM_LAT_UNROLL).  Smaller limits change only the control flow: every buffer keeps its
 * default size, and a limit too small for a search ends in CSM_E_CAPACITY. */
typedef struct csm_sweep_limits2d {
  int32_t chunk;        /* nodes per level chunk, 1 .. 1 << 23 */
  int32_t leaf_cap;     /* leaf buffer capacity, 2 .. 1 << 22 */
  int32_t inline_best;  /* optimal leaves read back with the first sync, 0 .. 4096 */
  int32_t lattice_min;  /* smallest chunk k_expand_lattice takes; INT32_MAX = never */
  int32_t unroll;       /* 4 | 8 | 16 */
  float dive_ratio;     /* >= 0, finite; > 1 disables the dives */
  int64_t max_points;   /* discrete-scan points per sub-batch, >= 1 */
} csm_sweep_limits2d;
void csm_sweep_limits2d_default(csm_sweep_limits2d* out);
/* csm_match2d_batch under `limits` (NULL: the defaults).  trace (may be NULL) receives
 * {collects, i.e. 1 + continuation sweeps, summed over sub-batches; leaf compactions between
 * sweeps, summed; most leaves held at any collect; optimal leaves, summed}. */
csm_status csm_match2d_batch_limits(const csm_stack2d* const* stacks, int32_t num_stacks,
                                    const csm_cloud* const* clouds, int32_t num_clouds,
                                    const csm_job2d* jobs, int32_t num_jobs,
                                    double linear_search_window, double angular_search_window,
                                    const csm_sweep_limits2d* limits, csm_result2d* results,
                                    csm_stats* total /* may be NULL */, int32_t trace[4]);

/* ---- test hooks ("visible for testing" in the reference) ------------------ */
/* FastCorrelativeScanMatcher2D::ScoreCandidates (fast...2d.cc:314-333) without
 * the sort: candidates are {scan_index, x_index_offset, y_index_offset} triples,
 * discrete_scans is num_scans x num_points x {x, y} int32 (DiscreteScan2D,
 * correlative_scan_matcher_2d.h:32).  sums may be NULL. */
csm_status csm_score_candidates2d(const csm_stack2d* stack, int32_t level,
                                  const int32_t* discrete_scans, int32_t num_scans,
                                  int32_t num_points, const int32_t* candidates,
                                  int32_t num_candidates, float* scores, int32_t* sums);
/* GenerateRotatedScans + DiscretizeScans + ShrinkToFit exactly as
 * MatchWithSearchParameters runs them (fast...2d.cc:236-247).  Call with
 * discrete_scans == NULL to get *num_scans first.  bounds is num_scans x
 * {min_x, max_x, min_y, max_y} (SearchParameters::LinearBounds). */
csm_status csm_discretize2d(const csm_stack2d* stack, const float* xyz, int32_t num_points,
                            const double initial_pose[3], int32_t full_submap,
                            double linear_search_window, double angular_search_window,
                            int32_t* num_scans, int32_t* discrete_scans, int32_t* bounds);
/* The lowest-resolution pass of the same match (ScoreCandidates at depth - 1 over every
 * candidate GenerateLowestResolutionCandidates makes, fast...2d.cc:281-312), run by the
 * batch's own launch code.  form: 0 = the size-based choice a match makes, 1 = small,
 * 2 = gather, 3 = tile, 4 = dense; a form that cannot serve the shape returns
 * CSM_E_INVALID.  Call with sums == NULL to get *num_scans and *slots_per_scan first.
 * sums is num_scans x slots_per_scan: the integer sum of candidate
 * (min_x + i * 2^(depth-1), min_y + j * 2^(depth-1)) at slot i * nyc + j, slots past
 * nxc * nyc unspecified.  lattices (may be NULL) is num_scans x
 * {min_x, max_x, min_y, max_y, nxc, nyc}.  kernel (may be NULL) receives the form that
 * ran (1 .. 4 as above) and, for the tile form, K of k_score_top_tile<K> (else 0). */
csm_status csm_score_top2d(const csm_stack2d* stack, const float* xyz, int32_t num_points,
                           const double initial_pose[3], int32_t full_submap,
                           double linear_search_window, double angular_search_window,
                           int32_t form, int32_t* num_scans, int32_t* slots_per_scan,
                           int32_t* sums, int32_t* lattices, int32_t* kernel);
/* A node of the branch-and-bound frontier: Candidate2D identity and score. */
typedef struct csm_node2d {
  int32_t scan_index, x_index_offset, y_index_offset;
  float score;
} csm_node2d;
/* One branch step of the same match (the children loop of BranchAndBound,
 * fast...2d.cc:335-376) over caller-given parents of level `level` (1 .. depth-1, on
 * their scan's lattice of stride 2^level), with the job's bound set to `bound` first,
 * run by the batch's own launch code.  form: 0 = one warp per parent, 1 = scan-grouped
 * lattice kernel with `unroll` 4, 8 or 16.  children (4 * num_parents records) receives
 * the pushed children in queue order (level >= 2) or the recorded leaves (level 1);
 * final_bound the job's bound afterwards, counters {candidates scored, parents expanded}. */
csm_status csm_branch_step2d(const csm_stack2d* stack, const float* xyz, int32_t num_points,
                             const double initial_pose[3], int32_t full_submap,
                             double linear_search_window, double angular_search_window,
                             float min_score, int32_t level, const csm_node2d* parents,
                             int32_t num_parents, float bound, int32_t form, int32_t unroll,
                             csm_node2d* children, int32_t* num_children, float* final_bound,
                             int64_t counters[2]);
/* The same match's phases between the lowest-resolution pass and the level loop, run by
 * the batch's own launch code with k_dive's gate at `dive_ratio`: job_best is the largest
 * lowest-resolution sum; bounds = {the job's bound after the dives, after the top-queue
 * filter} (they differ only at depth 1, where every queued candidate is a leaf);
 * counters = {candidates the dives scored, dives run}.  top_queue receives the first
 * top_capacity records of the top queue in queue order (at depth 1, of the leaves, which
 * are the queue's copy) and *top_count the queue's length. */
csm_status csm_dives2d(const csm_stack2d* stack, const float* xyz, int32_t num_points,
                       const double initial_pose[3], int32_t full_submap,
                       double linear_search_window, double angular_search_window,
                       float min_score, float dive_ratio, int32_t* job_best, float bounds[2],
                       int64_t counters[2], csm_node2d* top_queue, int32_t top_capacity,
                       int32_t* top_count);

/* ---- RealTimeCorrelativeScanMatcher2D::Match ------------------------------ */
/* real_time_correlative_scan_matcher_2d.cc:117-149 on a ProbabilityGrid (the
 * grid is passed per call, as in the reference signature).  Returns the best
 * score (the reference's return value) in *score. */
csm_status csm_rt_match2d(const uint16_t* cells, int32_t num_x_cells, int32_t num_y_cells,
                          double resolution, double max_x, double max_y, const float* xyz,
                          int32_t num_points, const double initial_pose[3],
                          double linear_search_window, double angular_search_window,
                          double translation_delta_cost_weight,
                          double rotation_delta_cost_weight, int32_t device, double* score,
                          double pose_estimate[3], csm_stats* stats /* may be NULL */);

/* Same for a TSDF2D grid (real_time_correlative_scan_matcher_2d.cc:38-59,160-166):
 * tsd_cells = Grid2D::correspondence_cost_cells(), weight_cells = TSDF2D::weight_cells_
 * (mapping/internal/2d/tsdf_2d.h), both uint16 with flat index num_x*y + x;
 * truncation_distance / max_weight are the TSDValueConverter parameters. */
csm_status csm_rt_match2d_tsdf(const uint16_t* tsd_cells, const uint16_t* weight_cells,
                               int32_t num_x_cells, int32_t num_y_cells, double resolution,
                               double max_x, double max_y, float truncation_distance,
                               float max_weight, const float* xyz, int32_t num_points,
                               const double initial_pose[3], double linear_search_window,
                               double angular_search_window,
                               double translation_delta_cost_weight,
                               double rotation_delta_cost_weight, int32_t device, double* score,
                               double pose_estimate[3], csm_stats* stats /* may be NULL */);

/* ---- grid-resident / batched real-time matcher ------------------------------ */
/* LocalTrajectoryBuilder2D::ScanMatch (internal/2d/local_trajectory_builder_2d.cc:77-82)
 * matches every incoming scan against the active submap's grid.  A csm_rt_grid2d keeps
 * that ProbabilityGrid on the device (refresh it with csm_rt_grid2d_update after a scan
 * was inserted; same cell limits), and csm_rt_match2d_batch scores many scans against it
 * in ONE launch: job j is exactly RealTimeCorrelativeScanMatcher2D::Match
 * (real_time_correlative_scan_matcher_2d.cc:117-149) of jobs[j] — same score, same pose. */
typedef struct csm_rt_grid2d csm_rt_grid2d;
csm_status csm_rt_grid2d_create(const uint16_t* cells, int32_t num_x_cells, int32_t num_y_cells,
                                double resolution, double max_x, double max_y, int32_t device,
                                csm_rt_grid2d** out);
csm_status csm_rt_grid2d_update(csm_rt_grid2d* grid, const uint16_t* cells);
/* The same handle for a TSDF2D (mapping/internal/2d/tsdf_2d.h): tsd cells and weight cells
 * (uint16, num_y x num_x, the proto's correspondence_cost_cells and tsdf_2d.weight_cells) and
 * the TSDValueConverter parameters.  csm_rt_match2d_batch then scores with the TSDF form of
 * csm_rt_match2d_tsdf, and csm_ceres_match2d_batch refines with TSDFMatchCostFunction2D. */
csm_status csm_rt_grid2d_create_tsdf(const uint16_t* tsd_cells, const uint16_t* weight_cells,
                                     int32_t num_x_cells, int32_t num_y_cells,
                                     double resolution, double max_x, double max_y,
                                     float truncation_distance, float max_weight,
                                     int32_t device, csm_rt_grid2d** out);
csm_status csm_rt_grid2d_update_tsdf(csm_rt_grid2d* grid, const uint16_t* tsd_cells,
                                     const uint16_t* weight_cells);
csm_status csm_rt_grid2d_destroy(csm_rt_grid2d* grid);

typedef struct csm_rt_job2d {
  const float* xyz;          /* sensor::PointCloud, num_points x {x, y, z} (host memory) */
  int32_t num_points;
  int32_t reserved;
  double initial_pose[3];    /* initial_pose_estimate {x, y, yaw} */
} csm_rt_job2d;

typedef struct csm_rt_result2d {
  double score;              /* Match's return value (best_candidate.score) */
  double pose_estimate[3];
  int32_t best_scan_index, best_x_offset, best_y_offset;
  int32_t num_scans;
  int64_t candidates_scored; /* num_scans * (2 * num_linear_perturbations + 1)^2 */
} csm_rt_result2d;

csm_status csm_rt_match2d_batch(const csm_rt_grid2d* grid, const csm_rt_job2d* jobs,
                                int32_t num_jobs, double linear_search_window,
                                double angular_search_window,
                                double translation_delta_cost_weight,
                                double rotation_delta_cost_weight, csm_rt_result2d* results,
                                csm_stats* stats /* may be NULL */);

/* Test hook: csm_rt_match2d_batch run exactly (same planning, kernel form and launches), and
 * every candidate's final weighted score: job-major, then scan, x offset, y offset
 * (generation order, real_time_correlative_scan_matcher_2d.cc:83-115); job j has
 * results[j].candidates_scored of them.  Call with scores == NULL to get the sizes first. */
csm_status csm_rt_scores2d(const csm_rt_grid2d* grid, const csm_rt_job2d* jobs, int32_t num_jobs,
                           double linear_search_window, double angular_search_window,
                           double translation_delta_cost_weight,
                           double rotation_delta_cost_weight, csm_rt_result2d* results,
                           float* scores);

/* RealTimeCorrelativeScanMatcher2D::ScoreCandidates — public in the reference
 * (real_time_correlative_scan_matcher_2d.h:75, .cc:151-176): scores caller-supplied
 * candidates {scan_index, x_index_offset, y_index_offset} against caller-supplied
 * discrete scans (num_scans x num_points x {x, y} int32).  The two SearchParameters
 * fields give Candidate2D::orientation = (scan_index - num_angular_perturbations) *
 * angular_perturbation_step_size (correlative_scan_matcher_2d.h:77-86). */
csm_status csm_rt_score_candidates2d(const uint16_t* cells, int32_t num_x_cells,
                                     int32_t num_y_cells, double resolution, double max_x,
                                     double max_y, const int32_t* discrete_scans,
                                     int32_t num_scans, int32_t num_points,
                                     int32_t num_angular_perturbations,
                                     double angular_perturbation_step_size,
                                     const int32_t* candidates, int32_t num_candidates,
                                     double translation_delta_cost_weight,
                                     double rotation_delta_cost_weight, int32_t device,
                                     float* scores);

/* ---- post-match refinement: CeresScanMatcher2D ------------------------------- */
/* ConstraintBuilder2D refines every found match with CeresScanMatcher2D::Match
 * (internal/constraints/constraint_builder_2d.cc:245-249 ->
 * internal/2d/scan_matching/ceres_scan_matcher_2d.cc:62-107): minimise over {x, y, theta}
 * the occupied-space residuals of the scan in the submap's ProbabilityGrid
 * (occupied_space_cost_function_2d.cc:42-69, bicubic interpolation of the correspondence
 * costs) plus the translation / rotation priors (translation_delta_cost_functor_2d.h:41-45,
 * rotation_delta_cost_functor_2d.h:40-43).  csm_ceres_match2d_batch solves many such
 * problems in ONE launch (one CTA per match, the trust-region loop on the device).  Ceres
 * itself is not linked: the solver follows Ceres' documented Levenberg-Marquardt
 * trust-region algorithm with the Solver::Options the reference sets (DENSE_QR,
 * use_nonmonotonic_steps, max_num_iterations; everything else default) — see DESIGN.md for
 * what that restatement is pinned to.  Grids are csm_rt_grid2d handles; the handle's grid
 * type selects the cost function as Grid2D::GetGridType() does (ceres_scan_matcher_2d.cc:
 * 74-91): a TSDF2D handle (csm_rt_grid2d_create_tsdf) gets TSDFMatchCostFunction2D
 * (tsdf_match_cost_function_2d.cc), bilinear interpolation of the correspondence costs
 * weighted by the interpolated weights.  One batch may mix both grid types. */
typedef struct csm_ceres_options2d {
  double occupied_space_weight;   /* proto/scan_matching/ceres_scan_matcher_options_2d.proto */
  double translation_weight;
  double rotation_weight;
  int32_t use_nonmonotonic_steps; /* common/proto/ceres_solver_options.proto */
  int32_t max_num_iterations;
} csm_ceres_options2d;

typedef struct csm_ceres_job2d {
  const csm_rt_grid2d* grid;      /* `grid` argument of Match */
  const float* xyz;               /* point_cloud, num_points x {x, y, z} (host memory) */
  int32_t num_points;
  int32_t reserved;
  double target_translation[2];
  double initial_pose[3];         /* initial_pose_estimate {x, y, rotation().angle()} */
} csm_ceres_job2d;

/* termination: 0 max_num_iterations reached (NO_CONVERGENCE), 1 function tolerance,
 * 2 gradient tolerance, 3 parameter tolerance, 4 minimum trust-region radius,
 * 5 too many consecutive invalid steps (FAILURE), 6 the cost function failed where Ceres
 * stops (FAILURE; TSDF2D only: the scan sees no weight, summed_weight == 0, at the initial
 * estimate or at an accepted step) — pose_estimate is then the initial estimate, and if it
 * failed at the initial estimate initial_cost = final_cost = -1 and iterations = 0.  A trial
 * step where the cost function fails counts as a step of infinite cost and is rejected.  Like
 * Ceres, 1 and 3 stop BEFORE taking the step that triggered them, and the lowest-cost iterate
 * visited is what is returned.
 *
 * Every csm_ceres_* entry point (2D and 3D, the batches and the test hooks) returns
 * CSM_E_INVALID, with the results untouched and nothing launched, when a cloud coordinate, an
 * intensity, a pose, a target translation or a target angle is NaN or infinite: such a value
 * would reach a float -> int conversion (floor, lround) whose result the reference leaves
 * undefined.  One such job refuses its whole batch. */
typedef struct csm_ceres_result2d {
  double pose_estimate[3];
  double initial_cost, final_cost; /* Solver::Summary::initial_cost / final_cost */
  int32_t iterations;              /* trust-region iterations after the initial evaluation */
  int32_t num_successful_steps;
  int32_t termination;
  int32_t reserved;
} csm_ceres_result2d;

csm_status csm_ceres_match2d_batch(const csm_ceres_job2d* jobs, int32_t num_jobs,
                                   const csm_ceres_options2d* options,
                                   csm_ceres_result2d* results,
                                   csm_stats* stats /* may be NULL */);

/* Test hook: the n + 3 residuals (and, if `jacobian` is not NULL, the (n + 3) x 3 row-major
 * Jacobian) of the three residual blocks at `pose`; max_num_iterations etc. are ignored. */
csm_status csm_ceres_evaluate2d(const csm_rt_grid2d* grid, const float* xyz, int32_t num_points,
                                const csm_ceres_options2d* options,
                                const double target_translation[2], double target_angle,
                                const double pose[3], double* residuals, double* jacobian);

/* Test hook for either grid type: as csm_ceres_evaluate2d, plus *valid = 0 where the cost
 * function returns false (TSDF2D, summed_weight == 0; the scan's residuals and Jacobian rows
 * are then 0, the priors' are still written).  ProbabilityGrid handles always give 1. */
csm_status csm_ceres_evaluate2d_checked(const csm_rt_grid2d* grid, const float* xyz,
                                        int32_t num_points, const csm_ceres_options2d* options,
                                        const double target_translation[2], double target_angle,
                                        const double pose[3], double* residuals,
                                        double* jacobian, int32_t* valid);

/* ==== 3D: FastCorrelativeScanMatcher3D ====================================== */
/* A HybridGrid crosses the ABI in the flat form of proto::HybridGrid
 * (mapping/proto/hybrid_grid.proto:19-28): voxel indices (n x {x,y,z} int32, origin
 * centred as in mapping/3d/hybrid_grid.h:263-264) and their uint16 values. */

/* proto/scan_matching/fast_correlative_scan_matcher_options_3d.proto */
typedef struct csm_options3d {
  int32_t branch_and_bound_depth;
  int32_t full_resolution_depth;
  double min_rotational_score;
  double min_low_resolution_score;
  double linear_xy_search_window;
  double linear_z_search_window;
  double angular_search_window;
} csm_options3d;

/* The matcher object: PrecomputationGridStack3D of the high-resolution grid
 * (fast_correlative_scan_matcher_3d.cc:57-77, precomputation_grid_3d.cc:49-81), the
 * low-resolution HybridGrid and the submap's rotational histogram — what
 * FastCorrelativeScanMatcher3D's ctor takes (:112-123).  Unlike the reference
 * (which keeps raw pointers to the low-res grid and histogram, :122-123) the
 * device copies are owned by the handle.  grid_size_in_voxels is
 * HybridGrid::grid_size() of the high-resolution grid (used by MatchFullSubmap,
 * :151-152); pass 0 to derive it from the voxel extents. */
typedef struct csm_matcher3d csm_matcher3d;
csm_status csm_matcher3d_create(const int32_t* hi_indices, const uint16_t* hi_values,
                                int64_t hi_num_voxels, float hi_resolution,
                                int32_t hi_grid_size_in_voxels, const int32_t* lo_indices,
                                const uint16_t* lo_values, int64_t lo_num_voxels,
                                float lo_resolution, const float* submap_histogram,
                                int32_t histogram_size, const csm_options3d* options,
                                int32_t device, csm_matcher3d** out);
csm_status csm_matcher3d_destroy(csm_matcher3d* matcher);
/* Same from two serialized cartographer.mapping.proto.HybridGrid messages
 * (mapping/proto/hybrid_grid.proto:19-28; Submap3D::ToProto), with the semantics of
 * HybridGrid(const proto::HybridGrid&) (mapping/3d/hybrid_grid.h:473-484). */
csm_status csm_matcher3d_create_from_proto(const uint8_t* hi_grid, int64_t hi_size,
                                           const uint8_t* lo_grid, int64_t lo_size,
                                           const float* submap_histogram, int32_t histogram_size,
                                           const csm_options3d* options, int32_t device,
                                           csm_matcher3d** out);
/* Test hook: one precomputation level as a dense box.  With out == NULL it
 * returns the level's bounding box (lo, dims); otherwise it fills `out`
 * (((z-lo.z)*dims.y + (y-lo.y))*dims.x + (x-lo.x)) for the box passed in. */
csm_status csm_matcher3d_read_level(const csm_matcher3d* matcher, int32_t depth, int32_t lo[3],
                                    int32_t dims[3], uint8_t* out);

/* TrajectoryNode::Data (mapping/trajectory_node.h:45-63), the fields the matcher reads. */
typedef struct csm_node3d {
  const float* high_resolution_point_cloud;   /* n x 3 */
  int32_t num_high;
  const float* low_resolution_point_cloud;    /* n x 3 */
  int32_t num_low;
  const float* rotational_scan_matcher_histogram;
  int32_t histogram_size;
  double gravity_alignment[4];                /* Quaterniond w, x, y, z */
} csm_node3d;

/* FastCorrelativeScanMatcher3D::Result (fast_correlative_scan_matcher_3d.h:68-73);
 * pose_estimate = {tx, ty, tz, qw, qx, qy, qz}.  found == 0 <=> nullptr. */
typedef struct csm_result3d {
  int32_t found;
  float score;
  double pose_estimate[7];
  float rotational_score;
  float low_resolution_score;
  int32_t best_scan_index;       /* index among the scans that passed the rotational filter */
  int32_t best_offset[3];
  int32_t leaves_tied;
  int32_t reserved;
} csm_result3d;

/* Match (full_submap == 0, fast_correlative_scan_matcher_3d.cc:127-144; poses are
 * Rigid3d {tx,ty,tz,qw,qx,qy,qz}) or MatchFullSubmap (full_submap != 0, :146-170;
 * only the rotation parts of the two poses are used). */
csm_status csm_match3d(const csm_matcher3d* matcher, const csm_node3d* node,
                       const double global_node_pose[7], const double global_submap_pose[7],
                       int32_t full_submap, float min_score, csm_result3d* result,
                       csm_stats* stats /* may be NULL */);

/* A queue of ConstraintBuilder3D::ComputeConstraint searches
 * (constraints/constraint_builder_3d.cc:220-223 global, :239-241 local) in one call:
 * job j matches nodes[node_index] against matchers[matcher_index].  The reference
 * runs these from its thread pool, one Match per task (:107-116); here the library
 * keeps up to max_concurrency (0 = default 8) matches in flight on separate CUDA
 * streams.  results[j] is exactly what csm_match3d returns for job j.  `stats`
 * (may be NULL) sums candidates_scored / nodes_expanded over the jobs. */
typedef struct csm_job3d {
  int32_t matcher_index;
  int32_t node_index;
  int32_t full_submap;
  float min_score;
  double global_node_pose[7];
  double global_submap_pose[7];
} csm_job3d;
csm_status csm_match3d_batch(const csm_matcher3d* const* matchers, int32_t num_matchers,
                             const csm_node3d* nodes, int32_t num_nodes, const csm_job3d* jobs,
                             int32_t num_jobs, int32_t max_concurrency, csm_result3d* results,
                             csm_stats* stats /* may be NULL */);

/* Limits of the 3D branch-and-bound sweep.  csm_sweep_limits3d_default gives the values
 * csm_match3d and csm_match3d_batch run with.  Smaller limits change only the control flow:
 * every buffer keeps its default size, and a limit too small for a search ends in
 * CSM_E_CAPACITY. */
typedef struct csm_sweep_limits3d {
  int32_t chunk;        /* nodes per level chunk, 1 .. 1 << 16 */
  int32_t leaf_cap;     /* leaves a match may record, 1 .. 1 << 20 */
  int32_t inline_best;  /* optimal leaves read back with each collect, 0 .. 256 */
  float dive_ratio;     /* >= 0, finite; > 1 disables the dives */
} csm_sweep_limits3d;
void csm_sweep_limits3d_default(csm_sweep_limits3d* out);
/* csm_match3d_batch under `limits` (NULL: the defaults), validated before any device is
 * used.  trace (may be NULL) receives {collects, i.e. 1 + continuation sweeps, summed over
 * the jobs; most leaves recorded by one match at a collect; optimal leaves, summed}. */
csm_status csm_match3d_batch_limits(const csm_matcher3d* const* matchers, int32_t num_matchers,
                                    const csm_node3d* nodes, int32_t num_nodes,
                                    const csm_job3d* jobs, int32_t num_jobs,
                                    int32_t max_concurrency, const csm_sweep_limits3d* limits,
                                    csm_result3d* results, csm_stats* stats /* may be NULL */,
                                    int32_t trace[3]);

/* Test hooks: RotationalScanMatcher::Match (rotational_scan_matcher.cc:178-189) and
 * the discrete scans of a match (GenerateDiscreteScans, :246-295): full-resolution
 * cell indices (num_scans x n x 3), scan poses (num_scans x 7 float: t, q wxyz) and
 * rotational scores.  Call with cells == NULL to get *num_scans. */
csm_status csm_rotational_match3d(const float* submap_histogram, const float* histogram,
                                  int32_t histogram_size, float initial_angle,
                                  const float* angles, int32_t num_angles, int32_t device,
                                  float* scores);
csm_status csm_discretize3d(const csm_matcher3d* matcher, const csm_node3d* node,
                            const double global_node_pose[7],
                            const double global_submap_pose[7], int32_t full_submap,
                            int32_t* num_scans, int32_t* cells, float* poses,
                            float* rotational_scores);
/* A candidate of ScoreCandidates (:332-355): a discrete scan (index after the rotational
 * filter), a linear offset in voxels and the precomputation depth it is scored at. */
typedef struct csm_candidate3d {
  int32_t scan_index, x, y, z, depth;
} csm_candidate3d;
/* ScoreCandidates of the same match's discrete scans over a caller-given list (no sort),
 * run by the match's own scoring kernel: sums and scores receive num_candidates values,
 * the integer sum and ToProbability(sum / n). */
csm_status csm_score_candidates3d(const csm_matcher3d* matcher, const csm_node3d* node,
                                  const double global_node_pose[7],
                                  const double global_submap_pose[7], int32_t full_submap,
                                  const csm_candidate3d* candidates, int32_t num_candidates,
                                  int32_t* sums, float* scores);
/* The same match up to and including its greedy dives: *num_scans after the rotational
 * filter and lattice = {nxc, nzc} (lowest-resolution candidates per axis, x == y).  The
 * other outputs may be NULL (call with sums == NULL to size them first): the angle index
 * and rotational score of each kept scan, every lowest-resolution sum (scan-major, then
 * z, y, x), the largest of them, the bound after the dives and
 * counters {candidates scored by the dives, low-resolution gate evaluations}. */
csm_status csm_score_top3d(const csm_matcher3d* matcher, const csm_node3d* node,
                           const double global_node_pose[7], const double global_submap_pose[7],
                           int32_t full_submap, float min_score, int32_t* num_scans,
                           int32_t lattice[2], int32_t* angle_index, float* rotational_scores,
                           int32_t* sums, int32_t* top_best, float* bound, int64_t counters[2]);
/* A node of the 3D branch-and-bound frontier, and a recorded leaf with its low-resolution
 * (gate) score. */
typedef struct csm_bnb_node3d {
  int32_t scan_index, x, y, z;
  float score;
} csm_bnb_node3d;
typedef struct csm_bnb_leaf3d {
  int32_t scan_index, x, y, z;
  float score, low_resolution_score;
} csm_bnb_leaf3d;
/* One level of the same match's branch step (BranchAndBound's children loop, :403-437)
 * over caller-given parents of `level` (1 .. depth-1, nodes of that level's lattice), with
 * the bound set to `bound` first, run by the match's own launch code until the level's
 * queue is drained (in chunks, from its end).  Level >= 2: children (8 * num_parents
 * records) receives the pushed children in queue order; level 1: leaves (8 * num_parents
 * records) the recorded gate-passing leaves.  *num_out is their number, *final_bound the
 * bound afterwards, counters {candidates scored, parents expanded, gate evaluations}.  A
 * full queue or leaf list returns CSM_E_CAPACITY, as in a match. */
csm_status csm_branch_step3d(const csm_matcher3d* matcher, const csm_node3d* node,
                             const double global_node_pose[7],
                             const double global_submap_pose[7], int32_t full_submap,
                             float min_score, int32_t level, const csm_bnb_node3d* parents,
                             int32_t num_parents, float bound, csm_bnb_node3d* children,
                             csm_bnb_leaf3d* leaves, int32_t* num_out, float* final_bound,
                             int64_t counters[3]);
/* The same match through its dives (k3_dive's gate at `dive_ratio`) and its top-queue filter:
 * *bound is the bound the level loop starts from, *count the length of the top queue (the
 * lowest-resolution candidates with score > min_score and score >= *bound) and queue its
 * first `capacity` records.  The queue is filled by atomic appends, so its order is not
 * deterministic: compare it as a set. */
csm_status csm_top_queue3d(const csm_matcher3d* matcher, const csm_node3d* node,
                           const double global_node_pose[7], const double global_submap_pose[7],
                           int32_t full_submap, float min_score, float dive_ratio, float* bound,
                           csm_bnb_node3d* queue, int32_t capacity, int32_t* count);

/* ==== RealTimeCorrelativeScanMatcher3D ======================================== */
/* A HybridGrid resident on the device (dense uint16 box over its non-zero voxels; reads
 * outside the box return 0 = unknown, as HybridGrid::value does for unallocated cells,
 * mapping/3d/hybrid_grid.h:263-279).  Same flat form as csm_matcher3d_create. */
typedef struct csm_grid3d csm_grid3d;
csm_status csm_grid3d_create(const int32_t* indices, const uint16_t* values, int64_t num_voxels,
                             float resolution, int32_t device, csm_grid3d** out);
csm_status csm_grid3d_destroy(csm_grid3d* grid);
/* RealTimeCorrelativeScanMatcher3D::Match
 * (internal/3d/scan_matching/real_time_correlative_scan_matcher_3d.cc:34-53): exhaustive
 * (2L+1)^3 x (2A+1)^3 window; *score is the return value, pose_estimate the best
 * candidate.cast<double>() ({tx,ty,tz, qw,qx,qy,qz}).  stats->num_scans = rotations. */
csm_status csm_rt_match3d(const csm_grid3d* grid, const float* xyz, int32_t num_points,
                          const double initial_pose[7], double linear_search_window,
                          double angular_search_window, double translation_delta_cost_weight,
                          double rotation_delta_cost_weight, float* score,
                          double pose_estimate[7], csm_stats* stats /* may be NULL */);
/* Test hook: the same match run by its own launch code; *num_candidates = T * R, and unless
 * scores is NULL (sizes only) scores receives every candidate's weighted score in generation
 * order (translations z, y, x outermost, then rotations rz, ry, rx; :55-98). */
csm_status csm_rt_scores3d(const csm_grid3d* grid, const float* xyz, int32_t num_points,
                           const double initial_pose[7], double linear_search_window,
                           double angular_search_window, double translation_delta_cost_weight,
                           double rotation_delta_cost_weight, float* scores,
                           int64_t* num_candidates);

/* ---- post-match refinement in 3D: CeresScanMatcher3D --------------------------- */
/* ConstraintBuilder3D refines every found match with CeresScanMatcher3D::Match
 * (internal/constraints/constraint_builder_3d.cc:265-275 ->
 * internal/3d/scan_matching/ceres_scan_matcher_3d.cc:95-157): occupied-space residuals of
 * up to two (point cloud, HybridGrid) pairs — high and low resolution — through the
 * smoothstep-interpolated grid (occupied_space_cost_function_3d.h:68-78,
 * interpolated_grid.h:49-96), a translation prior and a rotation prior
 * (translation_delta_cost_functor_3d.h, rotation_delta_cost_functor_3d.h:42-53), minimised over
 * {translation[3], rotation[4]} with ceres::QuaternionParameterization.  Intensity grids
 * (which the constraint builder does not pass): csm_ceres_match3d_intensity_batch below.
 * only_optimize_yaw must be 0.  Same solver notes as
 * csm_ceres_match2d_batch; grids are csm_grid3d handles.  Poses are {t xyz, q wxyz}. */
typedef struct csm_ceres_options3d {
  double occupied_space_weight[2]; /* occupied_space_weight_0 / _1 */
  double translation_weight;
  double rotation_weight;
  int32_t only_optimize_yaw;       /* must be 0 */
  int32_t use_nonmonotonic_steps;
  int32_t max_num_iterations;
  int32_t reserved;
} csm_ceres_options3d;

typedef struct csm_ceres_job3d {
  const csm_grid3d* grid[2];       /* PointCloudAndHybridGridsPointers::hybrid_grid */
  const float* xyz[2];             /* ::point_cloud, num_points x {x, y, z} (host memory) */
  int32_t num_points[2];
  int32_t num_clouds;              /* 1 or 2 */
  int32_t reserved;
  double target_translation[3];
  double initial_pose[7];          /* initial_pose_estimate; its rotation is the rotation prior's target */
} csm_ceres_job3d;

typedef struct csm_ceres_result3d {
  double pose_estimate[7];
  double initial_cost, final_cost;
  int32_t iterations, num_successful_steps, termination, reserved;  /* as csm_ceres_result2d */
} csm_ceres_result3d;

csm_status csm_ceres_match3d_batch(const csm_ceres_job3d* jobs, int32_t num_jobs,
                                   const csm_ceres_options3d* options,
                                   csm_ceres_result3d* results,
                                   csm_stats* stats /* may be NULL */);

/* Test hook: all residuals (clouds in order, 3 translation, 3 rotation) at `pose` and, if
 * `jacobian` is not NULL, the row-major (rows x 6) Jacobian by the tangent-space parameters
 * {dt[3], dq[3]}; the rotation prior's target is job->initial_pose's rotation. */
csm_status csm_ceres_evaluate3d(const csm_ceres_job3d* job, const csm_ceres_options3d* options,
                                const double pose[7], double* residuals, double* jacobian);

/* ---- intensity residuals in 3D: IntensityCostFunction3D under HuberLoss ---------- */
/* An IntensityHybridGrid resident on the device (mapping/3d/hybrid_grid.h:547-570), from the
 * flat form HybridGridBase<AverageIntensityData>::Iterator gives: voxel indices (n x 3, as
 * csm_grid3d_create), sum[n] and count[n] of each voxel's AverageIntensityData, no index
 * twice.  Each voxel holds GetIntensity (sum / count in float, 0 where count == 0); reads
 * outside the voxels' bounding box return 0, and a grid of no voxels reads 0 everywhere. */
typedef struct csm_intensity_grid3d csm_intensity_grid3d;
csm_status csm_intensity_grid3d_create(const int32_t* indices, const float* sum,
                                       const int32_t* count, int64_t num_voxels,
                                       float resolution, int32_t device,
                                       csm_intensity_grid3d** out);
csm_status csm_intensity_grid3d_destroy(csm_intensity_grid3d* grid);

/* Per csm_ceres_job3d: PointCloudAndHybridGridsPointers::intensity_hybrid_grid of each cloud
 * (NULL: that cloud has no intensity block) and its PointCloud::intensities()
 * (num_points[b] floats, host memory; required where the grid is set). */
typedef struct csm_ceres_intensity_job3d {
  const csm_intensity_grid3d* intensity_grid[2];
  const float* intensities[2];
} csm_ceres_intensity_job3d;

/* intensity_cost_function_options_0 / _1 (ceres_scan_matcher_options_3d.proto:24-25,42-43);
 * each must be positive for a cloud that has an intensity block in the batch. */
typedef struct csm_ceres_intensity_options3d {
  double weight[2];
  double huber_scale[2];
  float intensity_threshold[2];    /* returns brighter than this are left out */
} csm_ceres_intensity_options3d;

/* csm_ceres_match3d_batch where cloud b of job j may carry an intensity block
 * (ceres_scan_matcher_3d.cc:123-139): IntensityCostFunction3D with scaling weight / sqrt(n)
 * under ceres::HuberLoss(huber_scale), after that cloud's occupied-space block.  Jobs with
 * and without intensity blocks may share a batch; a job without one gives what
 * csm_ceres_match3d_batch gives, bit for bit. */
csm_status csm_ceres_match3d_intensity_batch(
    const csm_ceres_job3d* jobs, const csm_ceres_intensity_job3d* intensity_jobs,
    int32_t num_jobs, const csm_ceres_options3d* options,
    const csm_ceres_intensity_options3d* intensity_options, csm_ceres_result3d* results,
    csm_stats* stats /* may be NULL */);

/* ---- map writing in 3D: RangeDataInserter3D on device grids --------------------------- */
/* RangeDataInserter3D (mapping/3d/range_data_inserter_3d.cc:71-114) applied in place to a
 * csm_grid3d and, optionally, a csm_intensity_grid3d, so that the handles the 3D matchers read
 * follow the submap without a rebuild.  Every voxel ends bit-equal to what the reference's
 * Insert + FinishUpdate leaves: hits apply the hit table, misses (the last
 * num_free_space_voxels samples of each ray) the miss table, each cell at most once per insert
 * and hits first; intensities (returns not brighter than intensity_threshold) are added per
 * voxel in return order.  A handle's dense box grows as an insert reaches past it (DESIGN §9).
 * No match may be in flight on a handle being inserted into. */
typedef struct csm_range_inserter_options3d {   /* proto RangeDataInserterOptions3D */
  double hit_probability;                       /* in (0.5, 1) */
  double miss_probability;                      /* in [0, 0.5) */
  int32_t num_free_space_voxels;                /* >= 0 */
  float intensity_threshold;
} csm_range_inserter_options3d;
/* Owns the hit and miss tables (ComputeLookupTableToApplyOdds, probability_values.cc:76-87)
 * on one device. */
typedef struct csm_range_inserter3d csm_range_inserter3d;
csm_status csm_range_inserter3d_create(const csm_range_inserter_options3d* options,
                                       int32_t device, csm_range_inserter3d** out);
csm_status csm_range_inserter3d_destroy(csm_range_inserter3d* inserter);
/* RangeDataInserter3D::Insert.  origin and returns (num_returns x {x, y, z}) are in the grid's
 * frame; intensities (num_returns floats) may be NULL, and intensity_grid may be NULL.
 * CSM_E_INVALID, with every handle unchanged, for an origin, hit or intensity cell outside
 * [-8192, 8192)^3 or grids on another device than the inserter.  stats (may be NULL) gets
 * host_syncs and device_ms. */
csm_status csm_range_inserter3d_insert(const csm_range_inserter3d* inserter,
                                       const float origin[3], const float* returns,
                                       const float* intensities, int32_t num_returns,
                                       csm_grid3d* grid, csm_intensity_grid3d* intensity_grid,
                                       csm_stats* stats /* may be NULL */);
/* Submap3D::InsertData (mapping/3d/submap_3d.cc:271-294) into every entry of `submaps`, in
 * order, in one call: the range data (origin, num_returns x {x, y, z} returns and, may be NULL,
 * num_returns intensities) is in the local frame; each entry transforms it by
 * local_pose().inverse().cast<float>(), inserts the returns within high_resolution_max_range
 * of the transformed origin into high_resolution and, with intensities, intensity (may be NULL:
 * ForgetIntensityHybridGrid), and every return into low_resolution.  Every handle ends
 * bit-equal to what csm_range_inserter3d_insert leaves when it is given the transformed and
 * filtered data of each entry in turn: voxels, intensity sums, counts and means, dense and
 * tight boxes (the origin cell joins a handle's box only when that handle receives a return).
 * With no returns every handle keeps its contents and boxes; the origin is still checked.
 * CSM_E_INVALID, with every handle unchanged, for a null pointer, num_submaps outside
 * [1, 65535], a handle that appears twice, a handle on another device than the inserter, or
 * what csm_range_inserter3d_insert refuses for any entry: a non-finite point or an origin, hit
 * or intensity cell outside [-8192, 8192)^3, or num_samples >= 2^15.  Two stream
 * synchronisations however many entries; stats (may be NULL) gets host_syncs and device_ms. */
typedef struct csm_submap_insert3d {
  double local_pose[7];                 /* the submap's local_pose(): t xyz, q wxyz */
  csm_grid3d* high_resolution;
  csm_grid3d* low_resolution;
  csm_intensity_grid3d* intensity;      /* may be NULL */
} csm_submap_insert3d;
csm_status csm_range_inserter3d_insert_submaps(const csm_range_inserter3d* inserter,
                                               const csm_submap_insert3d* submaps,
                                               int32_t num_submaps, const float origin[3],
                                               const float* returns, const float* intensities,
                                               int32_t num_returns,
                                               float high_resolution_max_range,
                                               csm_stats* stats /* may be NULL */);
/* Test hooks: a handle's current dense box.  With out / mean == NULL only lo and dims are
 * written; otherwise the box is copied out (((z - lo.z) * dims.y + (y - lo.y)) * dims.x +
 * (x - lo.x)).  For an intensity grid, sum and count (each may be NULL) are every voxel's
 * AverageIntensityData and mean its GetIntensity. */
csm_status csm_grid3d_read(const csm_grid3d* grid, int32_t lo[3], int32_t dims[3], uint16_t* out);
/* FastCorrelativeScanMatcher3D's ctor over device-resident grids: what csm_matcher3d_create
 * builds from the NON-ZERO voxels of `hybrid_grid` and `low_resolution_hybrid_grid` (HybridGrid's
 * iterator skips value 0, hybrid_grid.h:57) and their resolutions, device to device, without a
 * host copy: every level, the low-resolution box, the derived grid size and every match result
 * are the same.  The matcher lives on the handles' device and owns its copies: later inserts
 * into, or destruction of, the handles do not change it.  No insert may be in flight on either
 * handle during the call.  grid_size_in_voxels as in csm_matcher3d_create (0 = derive it from
 * the high-resolution grid's non-zero voxels).  CSM_E_INVALID, with *out unwritten and nothing
 * allocated, for a null handle, options or out, handles on different devices, or options
 * csm_matcher3d_create refuses.  Two stream synchronisations. */
csm_status csm_matcher3d_create_from_grid3d(const csm_grid3d* hybrid_grid,
                                            int32_t grid_size_in_voxels,
                                            const csm_grid3d* low_resolution_hybrid_grid,
                                            const float* submap_histogram, int32_t histogram_size,
                                            const csm_options3d* options, csm_matcher3d** out);
csm_status csm_intensity_grid3d_read(const csm_intensity_grid3d* grid, int32_t lo[3],
                                     int32_t dims[3], float* mean, float* sum, int32_t* count);

/* ---- saving device grids: HybridGrid::ToProto and Grid2D::ToProto --------------------------- */
/* What Submap3D::ToProto / Submap2D::ToProto serialise (and MapBuilder::SerializeState saves),
 * straight from the device handles.  Encoding: fields in field-number order; implicit-presence
 * scalars omitted when zero, including a MapLimits max.x of 0.0 and a known-cells box coordinate of
 * 0; a float or double is omitted only when its bit pattern is all zeros, so -0.0 IS written (the
 * bit-pattern test of protobuf C++'s generated serialisers); repeated scalars packed, and omitted
 * when empty; a present empty sub-message written with length 0.  No protobuf runtime is involved.
 * A handle carries no update marker between calls (the inserters finish every update), as
 * ToProto's CHECK(update_indices_.empty()) requires; no insert may be in flight on it, and the
 * handle is left unchanged.  With buf == NULL only *size is written; a capacity below *size returns
 * CSM_E_CAPACITY with *size the needed size and nothing written, and so does a message of 2^31
 * bytes or more (protobuf's limit), whatever the capacity. */

/* The non-zero voxels of a csm_grid3d in HybridGrid's iteration order, which ToProto writes
 * (hybrid_grid.h:528-540, iterator :300-340): n x {x, y, z} indices and n values as the handle
 * holds them, the flat form csm_grid3d_create and csm_matcher3d_create take.  With
 * indices == values == NULL only *num_voxels is written; a capacity (in voxels) below it returns
 * CSM_E_CAPACITY with *num_voxels set and nothing written.  Three stream synchronisations (the
 * non-zero box, the count, the copy; one when the grid has no non-zero voxel, two without a list). */
csm_status csm_grid3d_voxels(const csm_grid3d* grid, int32_t* indices, uint16_t* values,
                             int64_t capacity, int64_t* num_voxels);
/* A serialised cartographer.mapping.proto.HybridGrid (hybrid_grid.proto): resolution, then the
 * csm_grid3d_voxels list as packed sint32 x / y / z indices and packed int32 values.  A grid with
 * no non-zero voxel gives the resolution field alone.  The stream synchronisations of
 * csm_grid3d_voxels; the encoding runs on the host. */
csm_status csm_grid3d_to_proto(const csm_grid3d* grid, uint8_t* buf, int64_t capacity,
                               int64_t* size);
/* A serialised cartographer.mapping.proto.Grid2D, as ProbabilityGrid::ToProto or TSDF2D::ToProto
 * writes it (grid_2d.cc:166-183, probability_grid.cc:84-89, tsdf_2d.cc:107-116): limits, every
 * cell (num_y x num_x, row-major), the known-cells box unless it is empty, probability_grid_2d {}
 * or tsdf_2d {truncation_distance, max_weight, weight_cells} from the handle's own converter, and
 * the min / max correspondence cost (ProbabilityGrid: kMin/kMaxCorrespondenceCost; TSDF2D:
 * -/+ truncation_distance).  One or two stream synchronisations (the known-cells box of a handle
 * made from cells, the cell copy). */
csm_status csm_rt_grid2d_to_proto(const csm_rt_grid2d* grid, uint8_t* buf, int64_t capacity,
                                  int64_t* size);

/* ---- drawing submaps for display: Submap2D / Submap3D::ToResponseProto ------------------------ */
/* A serialised cartographer.mapping.proto.SubmapQuery.Response.SubmapTexture, the texture
 * MapBuilder::SubmapToProto serves and io::FetchSubmapTextures paints, straight from a device
 * handle: cells = 1 (the value / alpha byte pairs, x fastest, gzip'd as common::FastGzipString
 * does: boost's gzip header with XFL 4 and OS 255, raw deflate at level 1, window 15, memLevel 8,
 * then CRC-32 and ISIZE), width = 2, height = 3, resolution = 4 and slice_pose = 5 (Rigid3d
 * {translation {x, y, z}, rotation {x, y, z, w}}), with the encoding rules of the *_to_proto
 * entry points above.  Poses are {tx, ty, tz, qw, qx, qy, qz}; a non-finite component returns
 * CSM_E_INVALID.  The pixel values are bit for bit the reference's; the step function
 * ProbabilityToLogOddsInteger is a table of its 254 steps, built on the host with the reference's
 * expression on the host's logf.  Every call, including one with buf == NULL, does the whole
 * work (the size of a gzip member is known only after compressing): *size is always the exact
 * size; a capacity below it returns CSM_E_CAPACITY with *size set and nothing written, and so
 * does a message of 2^31 bytes or more.  The handle is left unchanged, and no insert may be in
 * flight on it. */

/* ProbabilityGrid::DrawToSubmapTexture or TSDF2D::DrawToSubmapTexture (probability_grid.cc:109-147,
 * internal/2d/tsdf_2d.cc:137-181) with the submap's local pose, as Submap2D::ToResponseProto
 * calls it: the cells of Grid2D::ComputeCroppedLimits (the known-cells box, or 1 x 1 at offset 0
 * when it is empty).  ProbabilityGrid: delta = 128 - ProbabilityToLogOddsInteger(probability);
 * TSDF2D: delta = round(weight / max_weight * (pow(|tsd| / max_tsd, 0.5f) * 255. - 128.)), the
 * powers from the host's powf.  One or two stream synchronisations (the known-cells box of a
 * handle made from cells, the cells). */
csm_status csm_rt_grid2d_to_texture(const csm_rt_grid2d* grid, const double local_pose[7],
                                    uint8_t* buf, int64_t capacity, int64_t* size);
/* io::DrawProbabilityGrid (io/probability_grid_points_processor.cc:175-196), the image the
 * assets writer's write_probability_grid stage saves: the cells of Grid2D::ComputeCroppedLimits
 * (the known-cells box, or 1 x 1 at offset (0, 0) when it is empty, which draws one pixel of
 * 128), width = num_x_cells and height = num_y_cells of those limits, offset = their first cell.
 * Pixel (x, y) is cell (offset[0] + x, offset[1] + y) at pixels[y * width + x], a cairo ARGB32
 * grey word 0xFF << 24 | v << 16 | v << 8 | v: v = 128 for an unknown cell, else
 * ProbabilityToColor(GetProbability(cell)) with the reference's float steps, bit for bit (a
 * table of every cell value built on the host).  With pixels == NULL only the size and offset
 * are written; a capacity below width * height returns CSM_E_CAPACITY with the size and offset
 * set and no pixel written.  A TSDF2D handle returns CSM_E_INVALID.  The handle is left
 * unchanged, and no insert may be in flight on it.  One or two stream synchronisations (the
 * known-cells box of a handle made from cells, the pixels); stats (may be NULL) gets host_syncs
 * and device_ms. */
csm_status csm_rt_grid2d_draw(const csm_rt_grid2d* grid, uint32_t* pixels, int64_t capacity,
                              int32_t* width, int32_t* height, int32_t offset[2],
                              csm_stats* stats /* may be NULL */);
/* Test hook, no device needed: the 32768 grey levels csm_rt_grid2d_draw looks cell values up in
 * (grey[0] = 128, the unknown cell). */
csm_status csm_rt_grid2d_draw_table(uint8_t* grey /* 32768 */);
/* AddToTextureProto (mapping/3d/submap_3d.cc:51-176) with the global submap pose, as
 * Submap3D::ToResponseProto calls it for the high- and then the low-resolution grid: an X-ray
 * view of the voxels with probability >= 0.501f, transformed by the pose cast to float, rounded
 * to pixels and accumulated per pixel in HybridGrid's iteration order.  A grid with no such
 * voxel gives what x86-64 gives the reference: the pixel box stays (INT_MAX, INT_MIN), its
 * width and height wrap to 2, the 2 x 2 pixels are (0, 0) and the slice pose is built from
 * INT_MIN * resolution.  A pixel box of 2^30 pixels or more returns CSM_E_CAPACITY (the
 * reference would allocate 20 bytes per pixel).  Four stream synchronisations (the non-zero box,
 * the voxel count, the pixel box, the pixels; one when the grid has no non-zero voxel). */
csm_status csm_grid3d_to_texture(const csm_grid3d* grid, const double global_submap_pose[7],
                                 uint8_t* buf, int64_t capacity, int64_t* size);

/* ---- lifelong mapping in 2D: OverlappingSubmapsTrimmer2D's coverage pass ------------------- */
/* One finished submap with a freshness (overlapping_submaps_trimmer_2d.cc:62-64: the caller
 * leaves out unfinished submaps and submaps without one).  grid: the submap's ProbabilityGrid or
 * TSDF2D handle (IsKnown reads the cell alone); translation and rotation (w, x, y, z):
 * global_frame_from_local_frame = global_pose * local_pose().inverse(), composed by the caller;
 * freshness: the common::Time ticks of the submap's latest intra-submap node. */
typedef struct csm_coverage_submap2d {
  const csm_rt_grid2d* grid;
  double translation[3];
  double rotation[4];
  int64_t freshness;
} csm_coverage_submap2d;
typedef struct csm_coverage_stats2d {
  int64_t entries;             /* (submap, known cell) entries of the coverage grid */
  int64_t coverage_cells;      /* distinct global cells */
  int64_t device_tie_cells;    /* cells of <= 16 entries with a tie between submaps across the
                                  cut, settled in list order (libstdc++'s insertion sort) */
  int64_t host_sorted_cells;   /* cells of > 16 entries with such a tie, std::sort'ed on the host */
  int32_t host_syncs;          /* stream synchronisations */
  int32_t reserved;
} csm_coverage_stats2d;
/* AddSubmapsToSubmapCoverageGrid2D + FindSubmapIdsToTrim (overlapping_submaps_trimmer_2d.cc:55-102,
 * 145-182) over the submaps' device grids: every known cell of each submap's cropped limits (the
 * known-cells box, 1 x 1 at offset 0 when it is empty), x fastest, its centre moved into the
 * global frame in double (no FMA) and keyed by lround((first_max - p) / first_resolution) per
 * axis; per global cell the fresh_submaps_count freshest entries, chosen as the reference's
 * std::sort chooses them, count for their submaps.  trim[i] = 1 iff submap i gets no covered
 * entry or uint16(covered_entries[i]) < min_covered_cells_count (the reference's
 * std::map<SubmapId, uint16>, whose counts wrap at 65536); covered_entries[i] is the count before
 * the wrap.  The handles are read and left unchanged; no insert may be in flight on them.
 * CSM_E_INVALID for null pointers, a null grid, non-finite poses or limits, a resolution <= 0 or
 * handles on more than one device; CSM_E_CAPACITY, with nothing written, for a global cell key
 * outside int32 or entries that do not fit the device.  n == 0 does nothing.  At most three stream
 * synchronisations (the entry total; the counts; the cells left to the host, if any). */
csm_status csm_trim_overlapping_submaps2d(const csm_coverage_submap2d* submaps, int32_t n,
                                          double first_max_x, double first_max_y,
                                          double first_resolution, uint16_t fresh_submaps_count,
                                          uint16_t min_covered_cells_count,
                                          uint8_t* trim /* n */,
                                          uint32_t* covered_entries /* n */,
                                          csm_coverage_stats2d* stats /* may be NULL */);

/* ---- map writing in 2D: ProbabilityGridRangeDataInserter2D on device grids ------------ */
/* ProbabilityGridRangeDataInserter2D (mapping/2d/probability_grid_range_data_inserter_2d.cc)
 * applied in place to a ProbabilityGrid csm_rt_grid2d, so that a 2D submap lives on the device
 * from its first scan to the stack it becomes.  After every insert, every cell, the limits and
 * the known-cells box are bit-equal to what the reference's Insert + FinishUpdate leaves:
 * returns apply the hit table, every pixel of each return's and each miss's RayToPixelMask the
 * miss table (insert_free_space only), each cell at most once per insert and hits first.  The
 * handle grows as Grid2D::GrowLimits does (doubling, old cells at the doubling offset).  A
 * handle's cells must carry no kUpdateMarker, as the reference's FinishUpdate leaves them.  No
 * match may be in flight on a handle being inserted into. */
typedef struct csm_range_inserter_options2d {   /* proto ProbabilityGridRangeDataInserterOptions2D */
  double hit_probability;                       /* in (0.5, 1) */
  double miss_probability;                      /* in [0, 0.5) */
  int32_t insert_free_space;                    /* bool */
  int32_t reserved;
} csm_range_inserter_options2d;
/* Owns the hit and miss tables (ComputeLookupTableToApplyCorrespondenceCostOdds,
 * probability_values.cc:89-105) on one device. */
typedef struct csm_range_inserter2d csm_range_inserter2d;
csm_status csm_range_inserter2d_create(const csm_range_inserter_options2d* options,
                                       int32_t device, csm_range_inserter2d** out);
csm_status csm_range_inserter2d_destroy(csm_range_inserter2d* inserter);
/* ProbabilityGridRangeDataInserter2D::Insert(range_data, grid).  origin, returns (num_returns x
 * {x, y, z}) and misses (num_misses x {x, y, z}) are in the grid's frame; z is ignored.
 * CSM_E_INVALID, with the handle unchanged, for a TSDF2D handle, a null or non-finite input, a
 * grid on another device, or an insert that would grow the grid to 30000 cells or more per
 * axis.  One stream synchronisation; stats (may be NULL) gets host_syncs and device_ms. */
csm_status csm_range_inserter2d_insert(const csm_range_inserter2d* inserter,
                                       const float origin[3], const float* returns,
                                       int32_t num_returns, const float* misses,
                                       int32_t num_misses, csm_rt_grid2d* grid,
                                       csm_stats* stats /* may be NULL */);
/* ActiveSubmaps2D::InsertRangeData's inserts (mapping/2d/submap_2d.cc:162-175): the range data
 * into every handle of `grids`, in one call.  Every handle ends bit-equal to what num_grids
 * csm_range_inserter2d_insert calls in order would leave it: cells, limits and known-cells box.
 * CSM_E_INVALID, with every handle unchanged, for a null pointer (the list or an entry),
 * num_grids outside [1, 65535], a handle that appears twice, or what csm_range_inserter2d_insert
 * refuses for any handle: a TSDF2D handle, a handle on another device than the inserter, a
 * non-finite input, or an insert that would grow a grid to 30000 cells or more per axis.  One
 * stream synchronisation however many handles; stats (may be NULL) gets host_syncs and
 * device_ms, which spans the whole call. */
csm_status csm_range_inserter2d_insert_submaps(const csm_range_inserter2d* inserter,
                                               const float origin[3], const float* returns,
                                               int32_t num_returns, const float* misses,
                                               int32_t num_misses, csm_rt_grid2d* const* grids,
                                               int32_t num_grids, csm_stats* stats /* may be NULL */);
/* ActiveSubmaps2D::CreateGrid (mapping/2d/submap_2d.cc): an all-unknown ProbabilityGrid of the
 * given limits with an empty known-cells box. */
csm_status csm_rt_grid2d_create_empty(double resolution, double max_x, double max_y,
                                      int32_t num_x_cells, int32_t num_y_cells, int32_t device,
                                      csm_rt_grid2d** out);
/* ProbabilityGrid::ComputeCroppedGrid (probability_grid.cc:91-107) from device to device: a
 * new handle over the known-cells box (1 x 1 if it is empty) whose known cells went through
 * SetProbability(GetProbability(v)).  ProbabilityGrid handles only. */
csm_status csm_rt_grid2d_crop(const csm_rt_grid2d* grid, csm_rt_grid2d** out);
/* The PrecomputationGridStack2D constructor over a ProbabilityGrid handle: as csm_stack2d_create
 * on the handle's cells and limits, with kMin/kMaxCorrespondenceCost, without a host copy. */
csm_status csm_stack2d_create_from_rt_grid2d(const csm_rt_grid2d* grid,
                                             int32_t branch_and_bound_depth, csm_stack2d** out);
/* A handle's limits, its known-cells box (inclusive cell bounds; known_empty when there is
 * none) and, with cells != NULL, its cells (num_y x num_x, row-major; capacity in cells).  A
 * handle made by csm_rt_grid2d_create or refreshed by an update takes the bounding box of its
 * non-zero cells as its known-cells box. */
typedef struct csm_rt_grid2d_info {
  int32_t num_x_cells, num_y_cells;
  double resolution, max_x, max_y;
  int32_t known_min_x, known_min_y, known_max_x, known_max_y;
  int32_t known_empty;
  int32_t is_tsdf;
} csm_rt_grid2d_info;
csm_status csm_rt_grid2d_read(const csm_rt_grid2d* grid, csm_rt_grid2d_info* info,
                              uint16_t* cells, int64_t capacity);
/* A handle's MapLimits alone (resolution, max and cell counts; any pointer but grid may be NULL),
 * read on the host: no stream synchronisation, even when the known-cells box of a handle made from
 * cells has not been computed yet. */
csm_status csm_rt_grid2d_limits(const csm_rt_grid2d* grid, double* resolution, double* max_x,
                                double* max_y, int32_t* num_x_cells, int32_t* num_y_cells);

/* ---- map writing in 2D: TSDFRangeDataInserter2D on device grids ----------------------- */
/* TSDFRangeDataInserter2D (mapping/internal/2d/tsdf_range_data_inserter_2d.cc) applied in place
 * to a TSDF2D csm_rt_grid2d, so that a TSDF submap lives on the device as a ProbabilityGrid
 * submap does.  After every insert, every tsd and weight cell, the limits and the known-cells box
 * are bit-equal to what the reference's Insert + FinishUpdate leaves.  Each cell is written at
 * most once per insert, from its value before the insert, by the first ray in sorted order that
 * reaches it with a non-zero weight (DESIGN §9).  The handle grows as Grid2D::GrowLimits does,
 * both arrays alike.  The inserter's truncation distance and maximum weight drive the update; the
 * handle's own ones encode and decode its cells.  No match may be in flight on a handle being
 * inserted into. */
typedef struct csm_tsdf_inserter_options2d {   /* proto TSDFRangeDataInserterOptions2D */
  double truncation_distance;                  /* > 0 */
  double maximum_weight;                       /* > 0 */
  int32_t update_free_space;                   /* bool */
  int32_t num_normal_samples;                  /* normal_estimation_options, > 0 */
  double sample_radius;                        /* normal_estimation_options, > 0 */
  int32_t project_sdf_distance_to_scan_normal; /* bool */
  int32_t update_weight_range_exponent;
  double update_weight_angle_scan_normal_to_ray_kernel_bandwidth;
  double update_weight_distance_cell_to_hit_kernel_bandwidth;
} csm_tsdf_inserter_options2d;
typedef struct csm_tsdf_inserter2d csm_tsdf_inserter2d;
csm_status csm_tsdf_inserter2d_create(const csm_tsdf_inserter_options2d* options, int32_t device,
                                      csm_tsdf_inserter2d** out);
csm_status csm_tsdf_inserter2d_destroy(csm_tsdf_inserter2d* inserter);
/* TSDFRangeDataInserter2D::Insert(range_data, grid) + FinishUpdate.  origin and returns
 * (num_returns x {x, y, z}) are in the grid's frame; z enters only the growth and the normals, as
 * in the reference.  CSM_E_INVALID, with the handle unchanged (cells, weights, limits and box),
 * for a ProbabilityGrid handle, a null or non-finite input, a grid on another device, an insert
 * that would grow the grid to 30000 cells or more per axis, a tsd cell on a ray that carries
 * kUpdateMarker, or a ray whose pixel mask leaves the grown grid (a return whose z differs from
 * the origin's can reach past the growth the reference computes).  One stream synchronisation;
 * stats (may be NULL) gets host_syncs and device_ms. */
csm_status csm_tsdf_inserter2d_insert(const csm_tsdf_inserter2d* inserter, const float origin[3],
                                      const float* returns, int32_t num_returns,
                                      csm_rt_grid2d* grid, csm_stats* stats /* may be NULL */);
/* ActiveSubmaps2D::CreateGrid for GridType::TSDF: an all-unknown TSDF2D (tsd 0, weight 0) of the
 * given limits and converter, with an empty known-cells box. */
csm_status csm_rt_grid2d_create_empty_tsdf(double resolution, double max_x, double max_y,
                                           int32_t num_x_cells, int32_t num_y_cells,
                                           float truncation_distance, float max_weight,
                                           int32_t device, csm_rt_grid2d** out);
/* The weight cells of a TSDF2D handle (num_y x num_x, row-major; capacity in cells).
 * csm_rt_grid2d_read gives its tsd cells, limits and known-cells box. */
csm_status csm_rt_grid2d_read_weights(const csm_rt_grid2d* grid, uint16_t* weight_cells,
                                      int64_t capacity);

/* ---- scan filtering: VoxelFilter and AdaptiveVoxelFilter ------------------------------- */
/* sensor::VoxelFilter (sensor/internal/voxel_filter.cc:88-180) on many clouds at once: per
 * cloud, the input indices the reference's reservoir sampling keeps (one std::minstd_rand0 of
 * seed 1 per cloud, libstdc++'s uniform_int_distribution), bit for bit, in input order.
 * xyz[c] holds num_points[c] x {x, y, z}.  kept_indices (capacity sum of num_points) receives
 * the clouds' kept indices one cloud after another, each index into its own cloud; num_kept[c]
 * their count.  The four VoxelFilter overloads differ only in the payload that follows the
 * kept points.  CSM_E_INVALID, writing no output, for a negative count, a null pointer where
 * data is required, a non-finite coordinate, a resolution that is not finite and > 0, or more
 * than 2^30 points in one call.  One stream synchronisation; stats (may be NULL) gets
 * host_syncs and device_ms. */
csm_status csm_voxel_filter_batch(const float* const* xyz, const int32_t* num_points,
                                  const float* resolution, int32_t num_clouds, int32_t device,
                                  int32_t* kept_indices, int32_t* num_kept,
                                  csm_stats* stats /* may be NULL */);
typedef struct csm_adaptive_voxel_filter_options {   /* proto AdaptiveVoxelFilterOptions */
  float max_length;                                  /* finite, > 0 */
  float min_num_points;                              /* a float field: compared as float */
  float max_range;                                   /* not NaN; may be +infinity */
  int32_t reserved;
} csm_adaptive_voxel_filter_options;
/* sensor::AdaptiveVoxelFilter (voxel_filter.cc:31-75, 192-197) per cloud with its own options:
 * the points within max_range, then, unless there are at most min_num_points of them, the
 * VoxelFilter of those points at the length the reference's halving and bisection settle on
 * (the last halving length when none leaves min_num_points).  The search runs on the device;
 * whatever the number of lengths tried, one stream synchronisation.  Output, refusals and stats
 * as csm_voxel_filter_batch (indices into the unfiltered input cloud); a NaN min_num_points or
 * max_range is refused too.  CSM_E_INTERNAL if a bisection does not settle within 8 steps. */
csm_status csm_adaptive_voxel_filter_batch(const float* const* xyz, const int32_t* num_points,
                                           const csm_adaptive_voxel_filter_options* options,
                                           int32_t num_clouds, int32_t device,
                                           int32_t* kept_indices, int32_t* num_kept,
                                           csm_stats* stats /* may be NULL */);

/* ---- map assets: OutlierRemovingPointsProcessor ------------------------------------------ */
/* io::OutlierRemovingPointsProcessor (io/outlier_removing_points_processor.cc:53-129), the
 * assets writer's voxel_filter_and_remove_moving_objects stage, with its voxel map on one
 * device.  Three phases, each over every batch of the stream: add_hits counts hits per voxel
 * (GetCellIndex = lround(p / (float)voxel_size), narrowed to int); count_rays samples every ray
 * from its batch's origin at x = 0, x += voxel_size (x a float, voxel_size a double) while
 * x < |point - origin|, and counts a ray in each sampled voxel that has hits; filter keeps a point
 * iff rays < miss_per_hit_limit * hits of its voxel (in double; a voxel never hit reads {0, 0}).
 * Every count and kept index is bit for bit the reference's, however the batches are grouped
 * into calls.  Phases only move forward: a call of an earlier phase than one already begun
 * returns CSM_E_INVALID.  Batch b has num_points[b] x {x, y, z} in xyz[b]; a call takes any
 * number of batches.  Every call checks all its input first, and a refused call changes nothing:
 * CSM_E_INVALID for a null pointer where data is required, a negative count, a non-finite
 * coordinate or origin, more than 2^30 points in one call, a hit outside the [-8192, 8192)^3
 * voxels the reference's grid can grow to (its CHECK), or a ray longer than the point where
 * x += voxel_size stops growing (the reference would loop forever).  One stream synchronisation
 * per call with points (none without); stats (may be NULL) gets host_syncs and device_ms.
 * Counts are int32, as in the reference, whose overflow is undefined behaviour. */
typedef struct csm_outlier_remover csm_outlier_remover;
/* CSM_E_INVALID for a voxel_size that is not finite and > 0, or a non-finite limit. */
csm_status csm_outlier_remover_create(double voxel_size, double miss_per_hit_limit, int32_t device,
                                      csm_outlier_remover** out);
csm_status csm_outlier_remover_destroy(csm_outlier_remover* remover);
/* Phase 1 (ProcessInPhaseOne).  The voxel map grows (a device rehash) at the start of a call
 * that would fill it past one half; CSM_E_CAPACITY, with the map unchanged, when the device has
 * not the memory for that. */
csm_status csm_outlier_remover_add_hits(csm_outlier_remover* remover, const float* const* xyz,
                                        const int32_t* num_points, int32_t num_batches,
                                        csm_stats* stats /* may be NULL */);
/* Phase 2 (ProcessInPhaseTwo); origins holds num_batches x {x, y, z}. */
csm_status csm_outlier_remover_count_rays(csm_outlier_remover* remover, const float* origins,
                                          const float* const* xyz, const int32_t* num_points,
                                          int32_t num_batches, csm_stats* stats /* may be NULL */);
/* Phase 3 (ProcessInPhaseThree): kept_indices (capacity sum of num_points) receives the batches'
 * kept indices in input order, one batch after another, each index into its own batch;
 * num_kept[b] their count.  The removed points are the others (RemovePoints). */
csm_status csm_outlier_remover_filter(csm_outlier_remover* remover, const float* const* xyz,
                                      const int32_t* num_points, int32_t num_batches,
                                      int32_t* kept_indices, int32_t* num_kept,
                                      csm_stats* stats /* may be NULL */);
/* Test hook: every voxel with hits in ascending (z, y, x): indices (n x {x, y, z}), hits, rays
 * (each may be NULL).  With all three NULL only *num_voxels is written, without a stream
 * synchronisation; a capacity below it returns CSM_E_CAPACITY with *num_voxels set. */
csm_status csm_outlier_remover_voxels(const csm_outlier_remover* remover, int32_t* indices,
                                      int32_t* hits, int32_t* rays, int64_t capacity,
                                      int64_t* num_voxels);
/* The current phase (1, 2 or 3), the voxel count and the map's slot count (a power of two),
 * read on the host. */
csm_status csm_outlier_remover_info(const csm_outlier_remover* remover, int32_t* phase,
                                    int64_t* num_voxels, int64_t* slots);

/* ---- map assets: XRayPointsProcessor ----------------------------------------------------- */
/* io::XRayPointsProcessor (io/xray_points_processor.cc), the assets writer's write_xray_image
 * stage, with its aggregations on one device.  Each aggregation (one per floor, or one) holds the
 * voxels the points fall in and, per (y, z) column, the float sums of their colours and their
 * count; one bounding box of cell indices is shared by all aggregations.  A point p goes to cell
 * lround((transform * p) / (float)voxel_size) per axis, narrowed to int.  Every voxel, column sum
 * and count, the box and every pixel are bit for bit the reference's, however the batches are
 * grouped into calls.  Batch b has num_points[b] x {x, y, z} in xyz[b] and, unless rgb or rgb[b]
 * is NULL (black, as a batch without colours), num_points[b] x {r, g, b} in rgb[b].  Every call
 * checks its input first, and a refused call changes no voxel, column, count or box:
 * CSM_E_INVALID for a null handle or a null pointer where data is required, an aggregation out of
 * range, a negative count, a non-finite coordinate or colour, more than 2^30 points in one call,
 * or a cell outside the [-8192, 8192)^3 cells the reference's grid can grow to (its CHECK).
 * stats (may be NULL) gets host_syncs and device_ms. */
typedef struct csm_xray csm_xray;
/* transform = {t x, y, z, q w, x, y, z} (transform::Rigid3f).  CSM_E_INVALID for a voxel_size
 * that is not finite and > 0 in float, a non-finite saturation_factor or transform, or
 * num_aggregations < 1. */
csm_status csm_xray_create(double voxel_size, double saturation_factor, const float transform[7],
                           int32_t num_aggregations, int32_t device, csm_xray** out);
csm_status csm_xray_destroy(csm_xray* xray);
/* Insert (xray_points_processor.cc:221-239) of every batch, in order, into one aggregation.  The
 * aggregation's voxel set and column map grow (a device rehash) at the start of a call that could
 * fill them past one half; CSM_E_CAPACITY, with nothing changed, when the device has not the
 * memory for that.  One stream synchronisation per call with points (none without). */
csm_status csm_xray_insert(csm_xray* xray, int32_t aggregation, const float* const* xyz,
                           const float* const* rgb, const int32_t* num_points,
                           int32_t num_batches, csm_stats* stats /* may be NULL */);
/* The shared bounding box (the reference's bounding_box()), read on the host: *empty = 1 while
 * no point was inserted, and min and max are then {0, 0, 0}. */
csm_status csm_xray_bounding_box(const csm_xray* xray, int32_t min[3], int32_t max[3],
                                 int32_t* empty);
/* The aggregation's image (WriteVoxels and IntoImage, xray_points_processor.cc:65-104, 170-203):
 * width = max.y - min.y + 1 and height = max.z - min.z + 1 of the shared box, and pixel
 * (max.y - y, max.z - z) for column (y, z), each a cairo ARGB32 word 0xFF << 24 | r << 16 |
 * g << 8 | b, row-major with a stride of width.  An aggregation without points is all white.
 * With pixels == NULL only *width and *height are written, without a stream synchronisation;
 * an empty box writes 0 x 0 and returns CSM_OK (the reference writes no image); a capacity
 * below width * height returns CSM_E_CAPACITY with *width and *height set and nothing else
 * written.  One stream synchronisation otherwise. */
csm_status csm_xray_draw(csm_xray* xray, int32_t aggregation, uint32_t* pixels, int64_t capacity,
                         int32_t* width, int32_t* height, csm_stats* stats /* may be NULL */);
/* Test hook: the aggregation's voxels in ascending (z, y, x) as n x {x, y, z}.  With
 * indices == NULL only *num_voxels is written, without a stream synchronisation; a capacity
 * below it returns CSM_E_CAPACITY with *num_voxels set. */
csm_status csm_xray_voxels(const csm_xray* xray, int32_t aggregation, int32_t* indices,
                           int64_t capacity, int64_t* num_voxels);
/* Test hook: the aggregation's columns in ascending (y, z): yz (n x {y, z}), sums (n x {r, g, b})
 * and counts (each may be NULL).  With all three NULL only *num_columns is written, without a
 * stream synchronisation; a capacity below it returns CSM_E_CAPACITY with *num_columns set. */
csm_status csm_xray_columns(const csm_xray* xray, int32_t aggregation, int32_t* yz, float* sums,
                            uint32_t* counts, int64_t capacity, int64_t* num_columns);

/* Test hook: as csm_ceres_evaluate3d, in the problem's residual-block order — per cloud its
 * occupied-space residuals, then its intensity residuals if it has a grid; then 3
 * translation and 3 rotation residuals.  Residuals and rows are uncorrected by the loss, as
 * CostFunction::Evaluate returns them. */
csm_status csm_ceres_evaluate3d_intensity(const csm_ceres_job3d* job,
                                          const csm_ceres_intensity_job3d* intensity_job,
                                          const csm_ceres_options3d* options,
                                          const csm_ceres_intensity_options3d* intensity_options,
                                          const double pose[7], double* residuals,
                                          double* jacobian);

/* ==== multi-GPU: one process per GPU, the sharded ConstraintBuilder queue ==== */
/* Every (submap, node) search only depends on its submap's matcher
 * (constraints/constraint_builder_2d.cc:102-111), so the queue shards by submap with no
 * data-path exchange; RunWhenDoneCallback (:279-300) hands ONE vector of all constraints
 * to the caller, so the results are combined with exactly one ncclAllGather of fixed-size
 * records on the context's stream.  Bootstrap: rank 0 calls csm_comm_unique_id and the
 * application hands the 128 bytes to every rank by any means (file, socket, MPI, a
 * torch.distributed object broadcast); then every rank calls csm_ctx_create. */
#define CSM_COMM_ID_BYTES 128
typedef struct csm_ctx csm_ctx;
csm_status csm_comm_unique_id(uint8_t id[CSM_COMM_ID_BYTES]);
csm_status csm_ctx_create(int32_t world_size, int32_t rank, int32_t device,
                          const uint8_t id[CSM_COMM_ID_BYTES] /* NULL iff world_size == 1 */,
                          csm_ctx** out);
csm_status csm_ctx_destroy(csm_ctx* ctx);
csm_status csm_ctx_info(const csm_ctx* ctx, int32_t* world_size, int32_t* rank, int32_t* device);
/* recv = world_size x bytes, rank-major (host buffers; one ncclAllGather inside). */
csm_status csm_ctx_allgather(csm_ctx* ctx, const void* send, int64_t bytes, void* recv);

/* ConstraintBuilder2D's drained queue on all GPUs.  `jobs` is the WHOLE queue and must be
 * identical on every rank; job j runs on rank submap_owner[jobs[j].stack_index]
 * (submap_owner == NULL: stack_index % world_size).  stacks[s] may be NULL on ranks that
 * do not own submap s; clouds[] must exist on every rank that uses them (node scans are
 * replicated by H2D, 13 KB each).  On return EVERY rank holds results[0 .. num_jobs) in
 * job order.  `stats` counts this rank's searches. */
csm_status csm_cb_batch2d_run(csm_ctx* ctx, const csm_stack2d* const* stacks, int32_t num_stacks,
                              const csm_cloud* const* clouds, int32_t num_clouds,
                              const csm_job2d* jobs, int32_t num_jobs,
                              const int32_t* submap_owner, double linear_search_window,
                              double angular_search_window, csm_result2d* results,
                              csm_stats* stats /* may be NULL */);
/* Same for ConstraintBuilder3D (constraints/constraint_builder_3d.cc:107-116). */
csm_status csm_cb_batch3d_run(csm_ctx* ctx, const csm_matcher3d* const* matchers,
                              int32_t num_matchers, const csm_node3d* nodes, int32_t num_nodes,
                              const csm_job3d* jobs, int32_t num_jobs,
                              const int32_t* submap_owner, int32_t max_concurrency,
                              csm_result3d* results, csm_stats* stats /* may be NULL */);

/* ---- local SLAM in 2D: LocalTrajectoryBuilder2D on the device ------------------------------ */
/* LocalTrajectoryBuilder2D (mapping/internal/2d/local_trajectory_builder_2d.cc:65-300) from
 * synchronized range data to the submap insert, with the range data in device memory between the
 * stages.  The caller keeps the pose extrapolator, the range-data collator and the motion filter
 * (double precision and libm on the host) and the ActiveSubmaps2D lifecycle; the handle runs
 * every per-point stage.  Each stage equals the existing single-stage entry points on the same
 * data: csm_voxel_filter_batch, csm_adaptive_voxel_filter_batch, csm_rt_match2d_batch,
 * csm_ceres_match2d_batch and csm_range_inserter2d_insert_submaps.  Float options of the proto
 * are floats here and compare as floats. */
typedef struct csm_local_slam_options2d {   /* proto LocalTrajectoryBuilderOptions2D */
  float min_range, max_range;
  float min_z, max_z;
  float missing_data_ray_length;
  float voxel_filter_size;                   /* finite, > 0 */
  int32_t num_accumulated_range_data;        /* >= 1; the caller decides when to match */
  int32_t use_online_correlative_scan_matching;
  csm_adaptive_voxel_filter_options adaptive_voxel_filter;
  double linear_search_window;               /* real_time_correlative_scan_matcher */
  double angular_search_window;
  double translation_delta_cost_weight;
  double rotation_delta_cost_weight;
  csm_ceres_options2d ceres;                 /* ceres_scan_matcher */
  csm_range_inserter_options2d inserter;     /* submaps.range_data_inserter */
} csm_local_slam_options2d;
typedef struct csm_local_slam2d csm_local_slam2d;
csm_status csm_local_slam2d_create(const csm_local_slam_options2d* options, int32_t device,
                                   csm_local_slam2d** out);
csm_status csm_local_slam2d_destroy(csm_local_slam2d* handle);
/* AddRangeData's per-point loop (:163-186) on one synchronized scan: hit i (hits, num_hits x
 * {x, y, z}) and its origin origins[origin_index[i]] go through poses[pose_index[i]] (num_poses x
 * {tx, ty, tz, qw, qx, qy, qz}, the Rigid3f range_data_poses the host extrapolated, with the
 * backwards-time clamp applied); a hit at range >= min_range is a return if range <= max_range,
 * else a miss at missing_data_ray_length along its ray.  Returns and misses are appended in input
 * order to the accumulation, which the first call after a match starts afresh.  CSM_E_INVALID,
 * with nothing changed, for a null pointer, an empty input, a non-finite point or pose, or an
 * index out of range; CSM_E_CAPACITY, with nothing changed, when the grown accumulation does not
 * fit the device.  No stream synchronisation (device_ms is not measured and reads 0).  The input
 * is staged in one of two pinned buffers that alternate between calls: the call waits for the
 * copy out of its buffer from two calls earlier (an event wait, normally long complete), and a
 * staging buffer that has to grow is reallocated, which waits for the device. */
csm_status csm_local_slam2d_accumulate(csm_local_slam2d* handle, const float* hits,
                                       int32_t num_hits, const float* origins,
                                       int32_t num_origins, const int32_t* origin_index,
                                       const float* poses, int32_t num_poses,
                                       const int32_t* pose_index, csm_stats* stats /* may be NULL */);
enum {
  CSM_LOCAL_SLAM_MATCHED = 0,
  CSM_LOCAL_SLAM_DROPPED_EMPTY_RETURNS = 1,    /* :217-220, no return in [min_z, max_z] */
  CSM_LOCAL_SLAM_DROPPED_EMPTY_FILTERED = 2    /* :231-233 */
};
typedef struct csm_local_slam_match2d {
  int32_t status;             /* CSM_LOCAL_SLAM_* */
  int32_t matched_submap;     /* 1 when a grid was given: the pose is the scan matchers' */
  int32_t num_returns;        /* the voxel-filtered gravity-aligned range data */
  int32_t num_misses;
  int32_t num_filtered;       /* the adaptively filtered point cloud */
  int32_t reserved;
  double pose_estimate[3];    /* the 2D pose {x, y, angle} (the prediction without a grid) */
  double rt_score;            /* the real-time matcher's score, 0 when it did not run */
  csm_ceres_result2d ceres;   /* the refinement's summary, zero when it did not run */
} csm_local_slam_match2d;
/* TransformToGravityAlignedFrameAndFilter (:51-63) of the accumulation through to_gravity
 * (gravity_alignment.cast<float>() * range_data_poses.back().inverse(), {t, q wxyz}), then
 * AddAccumulatedRangeData up to the pose (:211-244): the adaptive voxel filter and ScanMatch
 * against `grid` (the front active submap's ProbabilityGrid; NULL when there is none) with the
 * prediction pose_prediction.  origin is the accumulated origin (range_data_poses.back()
 * .translation()).  The call ends the accumulation.  A dropped scan is not an error and leaves
 * every grid untouched.  CSM_E_INVALID, with nothing changed, for a null pointer, a non-finite
 * pose or origin, nothing accumulated, a TSDF2D grid or a grid on another device.  Stream
 * synchronisations: one when the cropped returns are empty, two when the filtered cloud is empty
 * or there is no grid, three with a grid, four with the online matcher. */
csm_status csm_local_slam2d_match(csm_local_slam2d* handle, const float to_gravity[7],
                                  const float origin[3], const double pose_prediction[3],
                                  const csm_rt_grid2d* grid, csm_local_slam_match2d* result,
                                  csm_stats* stats /* may be NULL */);
/* InsertIntoSubmap's insert (:245-252, 279-300) of the last matched scan: TransformRangeData of
 * its voxel-filtered gravity-aligned range data through pose (Embed3D(pose_estimate_2d
 * .cast<float>()), {t, q wxyz}) into the local frame, then what csm_range_inserter2d_insert_submaps
 * does with it on `grids` (the active submaps), without an upload.  local_origin (may be NULL)
 * receives range_data_in_local.origin.  CSM_E_INVALID, with every handle unchanged, for what
 * csm_range_inserter2d_insert_submaps refuses, a non-finite pose, or no matched scan since the
 * last insert.  Two stream synchronisations (the local range data's box and ray lengths, which
 * decide the grids' growth, then the insert). */
csm_status csm_local_slam2d_insert(csm_local_slam2d* handle, const float pose[7],
                                   csm_rt_grid2d* const* grids, int32_t num_grids,
                                   float local_origin[3], csm_stats* stats /* may be NULL */);
/* Read-back hooks: the points of one stage of the current scan (n x {x, y, z}).  *count gets
 * their number; with xyz != NULL they are copied (CSM_E_CAPACITY below it).  The filtered cloud is
 * the host copy the match made (no synchronisation); the others take one. */
enum {
  CSM_LOCAL_SLAM_ACCUMULATED_RETURNS = 0,
  CSM_LOCAL_SLAM_ACCUMULATED_MISSES = 1,
  CSM_LOCAL_SLAM_CROPPED_RETURNS = 2,   /* gravity-aligned and cropped */
  CSM_LOCAL_SLAM_CROPPED_MISSES = 3,
  CSM_LOCAL_SLAM_FILTERED_RETURNS = 4,  /* + VoxelFilter: the gravity-aligned range data */
  CSM_LOCAL_SLAM_FILTERED_MISSES = 5,
  CSM_LOCAL_SLAM_FILTERED = 6,          /* AdaptiveVoxelFilter of the returns */
  CSM_LOCAL_SLAM_LOCAL_RETURNS = 7,     /* range_data_in_local, after an insert */
  CSM_LOCAL_SLAM_LOCAL_MISSES = 8
};
csm_status csm_local_slam2d_read(const csm_local_slam2d* handle, int32_t which, float* xyz,
                                 int64_t capacity, int32_t* count);

#ifdef __cplusplus
}
#endif

#endif /* CSM_ABI_H_ */
