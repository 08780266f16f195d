// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_common.h).
// CeresScanMatcher2D (mapping/internal/2d/scan_matching/ceres_scan_matcher_2d.{h,cc}),
// the refinement ConstraintBuilder2D runs on every found match
// (mapping/internal/constraints/constraint_builder_2d.cc:245-249).
//
// PARITY UNPINNED AGAINST CERES ITSELF.  The solver is a third-party dependency that is
// absent from the reference source tree: Ceres Solver, pinned by the reference at
// commit 58c5edae2f7c4d2533fe8a975c1f5f0b892dfd3e (bazel/repositories.bzl:136-142;
// package.xml:48 libceres-dev).  What is restated here:
//   * the reference's own cost functors, line by line (occupied_space_cost_function_2d.cc:
//     31-106, translation_delta_cost_functor_2d.h:41-45, rotation_delta_cost_functor_2d.h:
//     40-43) including the kPadding = INT_MAX / 4 shift of the interpolation coordinates;
//   * Ceres' published algorithms for everything the reference's call reaches with
//     Solver::Options defaults + {DENSE_QR, use_nonmonotonic_steps, max_num_iterations}
//     (ceres_scan_matcher_2d.cc:52-57, common/internal/ceres_solver_options.cc:37-44):
//     BiCubicInterpolator / CubicHermiteSpline (Catmull-Rom, ceres/cubic_interpolation.h),
//     the forward-mode derivative of the functor, the trust-region loop with the
//     Levenberg-Marquardt strategy, Jacobi column scaling, the function / gradient / parameter
//     tolerances and the non-monotonic step acceptance of Conn, Gould & Toint, Alg. 10.1.2.
//     The 3-parameter damped least-squares step is solved through the normal equations
//     (Ceres: Householder QR of the stacked [J; D] — same minimiser, different rounding).
// Pinned to what the reference holds for this path: ceres_scan_matcher_2d_test.cc:40-97
// (four known-answer starts, pose within 1e-2, final cost within 1e-2 of 0) and
// occupied_space_cost_function_2d_test.cc:31-51 (residual == kMaxProbability exactly) —
// tests/test_oracle_golden_ceres2d.py.
#ifndef ORACLE_CERES2D_H_
#define ORACLE_CERES2D_H_

#include <vector>

#include "oracle_2d.h"

namespace oracle {

// proto/scan_matching/ceres_scan_matcher_options_2d.proto + common/proto/ceres_solver_options.proto
struct CeresScanMatcherOptions2D {
  double occupied_space_weight = 20.;  // configuration_files/pose_graph.lua:30-39
  double translation_weight = 10.;
  double rotation_weight = 1.;
  bool use_nonmonotonic_steps = true;
  int max_num_iterations = 10;
};

enum CeresTermination {
  kCeresNoConvergence = 0,        // max_num_iterations reached
  kCeresFunctionTolerance = 1,
  kCeresGradientTolerance = 2,
  kCeresParameterTolerance = 3,
  kCeresMinTrustRegionRadius = 4,
  kCeresInvalidSteps = 5,         // max_num_consecutive_invalid_steps reached (FAILURE)
};

struct CeresSummary2D {
  double initial_cost = 0., final_cost = 0.;
  int iterations = 0;              // trust-region iterations after the initial evaluation
  int num_successful_steps = 0;
  int termination = kCeresNoConvergence;
};

// One record per pass of the trust-region loop, for tests that must show which branch of the
// minimiser a case took.  Every deciding quantity is beside its threshold: step_quality
// against min_relative_decrease (1e-3), step_norm against step_norm_threshold (parameter
// tolerance), cost_change against cost_change_threshold (function tolerance),
// gradient_max_norm against 1e-10, and for an accepted step candidate_cost against the step
// evaluator's evaluator_minimum_cost (a lower cost resets the non-monotonic count) and, when
// it is not lower, against evaluator_candidate_cost (both as they were before the step).
// Fields a pass did not reach are NaN.
enum CeresStepOutcome {
  kStepAccepted = 0,
  kStepRejected = 1,
  kStepInvalid = 2,              // no valid trial step; the radius shrinks and the pass repeats
  kStepParameterTolerance = 3,   // stopped, the step is not taken
  kStepFunctionTolerance = 4,    // stopped, the step is not taken
  kStepLoopExit = 5,             // stopped before a trial step (see the summary's termination)
};

struct CeresIterationTrace {
  int outcome = kStepLoopExit;
  bool reused_diagonal = false;      // the damping diagonal was kept from the rejected pass before
  bool reference_switched = false;   // the step evaluator's reference cost was replaced
  double x_cost, gradient_max_norm, radius_before, radius_after;
  double candidate_cost, model_cost_change, step_quality;
  double step_norm, step_norm_threshold, cost_change, cost_change_threshold;
  double evaluator_minimum_cost, evaluator_candidate_cost;
  CeresIterationTrace();
};
constexpr int kCeresTraceDoubles = 16;
// {outcome, reused_diagonal, reference_switched, x_cost, ... cost_change_threshold}
void PackCeresTrace(const std::vector<CeresIterationTrace>& trace, double* out);

// residuals (n + 3) and the row-major (n + 3) x 3 Jacobian of the three residual blocks at
// `pose` = {x, y, theta}; `jacobian` may be null (then the plain-double evaluation path).
void EvaluateCeresResiduals2D(const ProbabilityGrid& grid, const PointCloud& cloud,
                              const CeresScanMatcherOptions2D& options,
                              const double target_translation[2], double target_angle,
                              const double pose[3], std::vector<double>* residuals,
                              std::vector<double>* jacobian);

// CeresScanMatcher2D::Match (ceres_scan_matcher_2d.cc:62-107)
void CeresMatch2D(const ProbabilityGrid& grid, const PointCloud& cloud,
                  const CeresScanMatcherOptions2D& options, const double target_translation[2],
                  const double initial_pose[3], double pose_estimate[3],
                  CeresSummary2D* summary, std::vector<CeresIterationTrace>* trace = nullptr);

}  // namespace oracle

#endif  // ORACLE_CERES2D_H_
