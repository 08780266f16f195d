// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_common.h).
// CeresScanMatcher3D (mapping/internal/3d/scan_matching/ceres_scan_matcher_3d.{h,cc}) as
// ConstraintBuilder3D calls it (mapping/internal/constraints/constraint_builder_3d.cc:
// 265-275): occupied-space blocks for (point cloud, HybridGrid) pairs — no intensity grid —
// plus the translation and rotation priors, over {translation[3], rotation[4]} with Ceres'
// QuaternionParameterization (only_optimize_yaw = false, configuration_files/
// pose_graph.lua:49-60).
//
// PARITY UNPINNED AGAINST CERES ITSELF, for the same reason and with the same split as
// oracle_ceres2d.h: the reference's own functors are restated line by line
// (occupied_space_cost_function_3d.h:46-80, interpolated_grid.h:41-141,
// translation_delta_cost_functor_3d.h, rotation_delta_cost_functor_3d.h:42-53,
// common/math.h:74-81), Ceres' published algorithms supply the rest (forward-mode
// derivatives, QuaternionParameterization::Plus / ComputeJacobian, the trust-region
// Levenberg-Marquardt loop of oracle_ceres2d.cc generalised to 6 tangent-space parameters).
// Pinned to ceres_scan_matcher_3d_test.cc:36-137 (five starts; the fixture's intensity block
// is left out, as the constraint builder passes no intensity grid) and
// interpolated_grid_test.cc:30-88 — tests/test_oracle_golden_ceres3d.py.
#ifndef ORACLE_CERES3D_H_
#define ORACLE_CERES3D_H_

#include <vector>

#include "oracle_3d.h"
#include "oracle_ceres2d.h"

namespace oracle {

struct CeresScanMatcherOptions3D {   // proto/scan_matching/ceres_scan_matcher_options_3d.proto
  std::vector<double> occupied_space_weight = {5., 30.};   // pose_graph.lua:49-60
  double translation_weight = 10.;
  double rotation_weight = 1.;
  bool use_nonmonotonic_steps = false;
  int max_num_iterations = 10;
};

struct PointCloudAndHybridGrid {     // ceres_scan_matcher_3d.h:38-42 without the intensity grid
  const PointCloud* point_cloud;
  const HybridGrid* hybrid_grid;
};

// InterpolatedGrid<HybridGrid>::GetInterpolatedValue (interpolated_grid.h:49-96); with
// `gradient` the derivative by (x, y, z) the dual-number evaluation carries.
double InterpolatedProbability(const HybridGrid& grid, double x, double y, double z,
                               double gradient[3]);

// All residuals at pose = {t xyz, q wxyz} (clouds in order, then 3 translation and 3
// rotation residuals) and, if `jacobian` is not null, the row-major (rows x 6) Jacobian by
// the tangent-space parameters {dt[3], dq[3]} (ambient Jacobian times the
// parameterisation's 4 x 3 plus-Jacobian).
void EvaluateCeresResiduals3D(const std::vector<PointCloudAndHybridGrid>& clouds,
                              const CeresScanMatcherOptions3D& options,
                              const double target_translation[3],
                              const double target_rotation[4], const double pose[7],
                              std::vector<double>* residuals, std::vector<double>* jacobian);

// CeresScanMatcher3D::Match (ceres_scan_matcher_3d.cc:95-157)
void CeresMatch3D(const std::vector<PointCloudAndHybridGrid>& clouds,
                  const CeresScanMatcherOptions3D& options, const double target_translation[3],
                  const double initial_pose[7], double pose_estimate[7],
                  CeresSummary2D* summary, std::vector<CeresIterationTrace>* trace = nullptr);

}  // namespace oracle

#endif  // ORACLE_CERES3D_H_
