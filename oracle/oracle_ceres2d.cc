// ORACLE — TEST INFRASTRUCTURE ONLY.  See oracle_ceres2d.h for what is restated from the
// reference and what from Ceres' published algorithms ("parity unpinned" against Ceres).
#include "oracle_ceres2d.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <limits>

namespace oracle {
namespace {

// occupied_space_cost_function_2d.cc:72 — the grid is presented to the interpolator shifted by
// kPadding cells so that cells outside it read kMaxCorrespondenceCost (:78-86).
constexpr int kPadding = INT_MAX / 4;

double PaddedValue(const ProbabilityGrid& grid, const int row, const int column) {
  const int num_rows = grid.limits.cell_limits.num_y_cells + 2 * kPadding;   // :89-91
  const int num_cols = grid.limits.cell_limits.num_x_cells + 2 * kPadding;   // :93-95
  if (row < kPadding || column < kPadding || row >= num_rows - kPadding ||
      column >= num_cols - kPadding) {
    return static_cast<double>(kMaxCorrespondenceCost);
  }
  return static_cast<double>(
      grid.GetCorrespondenceCost(Array2i{column - kPadding, row - kPadding}));
}

// Catmull-Rom spline through p1, p2 with tangents from p0, p3 (ceres/cubic_interpolation.h,
// CubicHermiteSpline): value and derivative at x in [0, 1].
void CubicHermiteSpline(const double p0, const double p1, const double p2, const double p3,
                        const double x, double* f, double* dfdx) {
  const double a = 0.5 * (-p0 + 3.0 * p1 - 3.0 * p2 + p3);
  const double b = 0.5 * (2.0 * p0 - 5.0 * p1 + 4.0 * p2 - p3);
  const double c = 0.5 * (-p0 + p2);
  const double d = p1;
  if (f != nullptr) *f = d + x * (c + x * (b + x * a));
  if (dfdx != nullptr) *dfdx = c + x * (2.0 * b + 3.0 * a * x);
}

// BiCubicInterpolator::Evaluate: four row splines along the columns, then one spline across
// the rows for the value and d/dr, and one across the row derivatives for d/dc.
void BiCubic(const ProbabilityGrid& grid, const double r, const double c, double* f,
             double* dfdr, double* dfdc) {
  const int row = static_cast<int>(std::floor(r));
  const int col = static_cast<int>(std::floor(c));
  double fr[4], dfr[4];
  for (int k = 0; k < 4; ++k) {
    const int rr = row - 1 + k;
    CubicHermiteSpline(PaddedValue(grid, rr, col - 1), PaddedValue(grid, rr, col),
                       PaddedValue(grid, rr, col + 1), PaddedValue(grid, rr, col + 2), c - col,
                       &fr[k], &dfr[k]);
  }
  CubicHermiteSpline(fr[0], fr[1], fr[2], fr[3], r - row, f, dfdr);
  if (dfdc != nullptr) CubicHermiteSpline(dfr[0], dfr[1], dfr[2], dfr[3], r - row, dfdc, nullptr);
}

}  // namespace

void EvaluateCeresResiduals2D(const ProbabilityGrid& grid, const PointCloud& cloud,
                              const CeresScanMatcherOptions2D& options,
                              const double target_translation[2], const double target_angle,
                              const double pose[3], std::vector<double>* residuals,
                              std::vector<double>* jacobian) {
  const size_t n = cloud.size();
  residuals->assign(n + 3, 0.);
  if (jacobian != nullptr) jacobian->assign(3 * (n + 3), 0.);
  // ceres_scan_matcher_2d.cc:76-78
  const double scaling = options.occupied_space_weight / std::sqrt(static_cast<double>(n));
  // occupied_space_cost_function_2d.cc:44-48: Rotation2D(pose[2]).toRotationMatrix()
  const double cs = std::cos(pose[2]), sn = std::sin(pose[2]);
  const double resolution = grid.limits.resolution;
  const double inverse_resolution = 1.0 / resolution;
  for (size_t i = 0; i < n; ++i) {
    const double px = static_cast<double>(cloud[i].x), py = static_cast<double>(cloud[i].y);
    // :56-60 — transform * (x, y, 1)
    const double wx = (cs * px + (-sn) * py) + pose[0] * 1.0;
    const double wy = (sn * px + cs * py) + pose[1] * 1.0;
    double f, dfdr, dfdc;
    if (jacobian == nullptr) {
      // :61-66, plain doubles
      const double r = (grid.limits.max_x - wx) / resolution - 0.5 + static_cast<double>(kPadding);
      const double c = (grid.limits.max_y - wy) / resolution - 0.5 + static_cast<double>(kPadding);
      BiCubic(grid, r, c, &f, nullptr, nullptr);
      (*residuals)[i] = scaling * f;
      continue;
    }
    // the same expression on dual numbers: a dual divided by a scalar multiplies value and
    // derivatives by the scalar's reciprocal
    const double r =
        (grid.limits.max_x - wx) * inverse_resolution - 0.5 + static_cast<double>(kPadding);
    const double c =
        (grid.limits.max_y - wy) * inverse_resolution - 0.5 + static_cast<double>(kPadding);
    BiCubic(grid, r, c, &f, &dfdr, &dfdc);
    (*residuals)[i] = scaling * f;
    // d(wx, wy) / d(x, y, theta)
    const double dwx[3] = {1.0, 0.0, (-sn) * px + (-cs) * py};
    const double dwy[3] = {0.0, 1.0, cs * px + (-sn) * py};
    for (int k = 0; k < 3; ++k) {
      const double dr = -dwx[k] * inverse_resolution, dc = -dwy[k] * inverse_resolution;
      (*jacobian)[3 * i + k] = scaling * (dfdr * dr + dfdc * dc);
    }
  }
  // translation_delta_cost_functor_2d.h:41-45
  (*residuals)[n] = options.translation_weight * (pose[0] - target_translation[0]);
  (*residuals)[n + 1] = options.translation_weight * (pose[1] - target_translation[1]);
  // rotation_delta_cost_functor_2d.h:40-43
  (*residuals)[n + 2] = options.rotation_weight * (pose[2] - target_angle);
  if (jacobian != nullptr) {
    (*jacobian)[3 * n + 0] = options.translation_weight;
    (*jacobian)[3 * (n + 1) + 1] = options.translation_weight;
    (*jacobian)[3 * (n + 2) + 2] = options.rotation_weight;
  }
}

namespace {

// What one evaluation leaves behind for the minimiser: cost = 1/2 |r|^2, g = J^T r and
// H = J^T J (xx, xy, xt, yy, yt, tt) of the unscaled Jacobian.
struct Normal {
  double cost = 0.;
  double g[3] = {0., 0., 0.};
  double h[6] = {0., 0., 0., 0., 0., 0.};
};

Normal Evaluate(const ProbabilityGrid& grid, const PointCloud& cloud,
                const CeresScanMatcherOptions2D& options, const double target[2],
                const double target_angle, const double x[3], const bool with_jacobian) {
  std::vector<double> r, j;
  EvaluateCeresResiduals2D(grid, cloud, options, target, target_angle, x, &r,
                           with_jacobian ? &j : nullptr);
  Normal nm;
  double sq = 0.;
  for (size_t i = 0; i < r.size(); ++i) {
    sq += r[i] * r[i];
    if (!with_jacobian) continue;
    const double* ji = &j[3 * i];
    nm.g[0] += ji[0] * r[i];
    nm.g[1] += ji[1] * r[i];
    nm.g[2] += ji[2] * r[i];
    nm.h[0] += ji[0] * ji[0];
    nm.h[1] += ji[0] * ji[1];
    nm.h[2] += ji[0] * ji[2];
    nm.h[3] += ji[1] * ji[1];
    nm.h[4] += ji[1] * ji[2];
    nm.h[5] += ji[2] * ji[2];
  }
  nm.cost = 0.5 * sq;
  return nm;
}

// Solves the symmetric positive definite 3x3 system A y = b (Cholesky); false if a pivot is
// not positive or the result is not finite.
bool SolveSpd3(const double a[6], const double b[3], double y[3]) {
  const double l00sq = a[0];
  if (!(l00sq > 0.)) return false;
  const double l00 = std::sqrt(l00sq);
  const double l10 = a[1] / l00, l20 = a[2] / l00;
  const double l11sq = a[3] - l10 * l10;
  if (!(l11sq > 0.)) return false;
  const double l11 = std::sqrt(l11sq);
  const double l21 = (a[4] - l20 * l10) / l11;
  const double l22sq = a[5] - l20 * l20 - l21 * l21;
  if (!(l22sq > 0.)) return false;
  const double l22 = std::sqrt(l22sq);
  const double z0 = b[0] / l00;
  const double z1 = (b[1] - l10 * z0) / l11;
  const double z2 = (b[2] - l20 * z0 - l21 * z1) / l22;
  y[2] = z2 / l22;
  y[1] = (z1 - l21 * y[2]) / l11;
  y[0] = (z0 - l10 * y[1] - l20 * y[2]) / l00;
  return std::isfinite(y[0]) && std::isfinite(y[1]) && std::isfinite(y[2]);
}

double Norm3(const double v[3]) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

}  // namespace

CeresIterationTrace::CeresIterationTrace() {
  const double nan = std::numeric_limits<double>::quiet_NaN();
  x_cost = gradient_max_norm = radius_before = radius_after = nan;
  candidate_cost = model_cost_change = step_quality = nan;
  step_norm = step_norm_threshold = cost_change = cost_change_threshold = nan;
  evaluator_minimum_cost = evaluator_candidate_cost = nan;
}

void PackCeresTrace(const std::vector<CeresIterationTrace>& trace, double* out) {
  for (const CeresIterationTrace& t : trace) {
    const double rec[kCeresTraceDoubles] = {
        static_cast<double>(t.outcome), t.reused_diagonal ? 1. : 0., t.reference_switched ? 1. : 0.,
        t.x_cost, t.gradient_max_norm, t.radius_before, t.radius_after, t.candidate_cost,
        t.model_cost_change, t.step_quality, t.step_norm, t.step_norm_threshold, t.cost_change,
        t.cost_change_threshold, t.evaluator_minimum_cost, t.evaluator_candidate_cost};
    out = std::copy(rec, rec + kCeresTraceDoubles, out);
  }
}

void CeresMatch2D(const ProbabilityGrid& grid, const PointCloud& cloud,
                  const CeresScanMatcherOptions2D& options, const double target_translation[2],
                  const double initial_pose[3], double pose_estimate[3],
                  CeresSummary2D* summary, std::vector<CeresIterationTrace>* trace) {
  // Solver::Options defaults the reference leaves untouched
  const double kInitialRadius = 1e4, kMaxRadius = 1e16, kMinRadius = 1e-32;
  const double kMinRelativeDecrease = 1e-3;
  const double kMinLmDiagonal = 1e-6, kMaxLmDiagonal = 1e32;
  const int kMaxConsecutiveInvalidSteps = 5;
  const double kFunctionTolerance = 1e-6, kGradientTolerance = 1e-10, kParameterTolerance = 1e-8;
  const int max_nonmonotonic = options.use_nonmonotonic_steps ? 5 : 0;

  // ceres_scan_matcher_2d.cc:68-70, :94-97 — the rotation prior is on the INITIAL angle
  double x[3] = {initial_pose[0], initial_pose[1], initial_pose[2]};
  const double target_angle = initial_pose[2];
  double best[3] = {x[0], x[1], x[2]};
  CeresSummary2D sum;

  Normal at_x = Evaluate(grid, cloud, options, target_translation, target_angle, x, true);
  double x_cost = at_x.cost;
  double x_norm = Norm3(x);
  sum.initial_cost = x_cost;
  double minimum_cost = x_cost;
  // Jacobi scaling, fixed at the first Jacobian
  double scale[3];
  scale[0] = 1.0 / (1.0 + std::sqrt(at_x.h[0]));
  scale[1] = 1.0 / (1.0 + std::sqrt(at_x.h[3]));
  scale[2] = 1.0 / (1.0 + std::sqrt(at_x.h[5]));
  // Levenberg-Marquardt strategy state
  double radius = kInitialRadius, decrease_factor = 2.0;
  bool reuse_diagonal = false;
  double diagonal[3] = {0., 0., 0.};
  // non-monotonic step evaluator (Conn, Gould & Toint, Algorithm 10.1.2)
  double current_cost = x_cost, reference_cost = x_cost, candidate_cost_ev = x_cost;
  double ev_minimum_cost = x_cost;
  double acc_reference = 0., acc_candidate = 0.;
  int num_nonmonotonic = 0;
  int num_invalid = 0;
  bool last_step_successful = false;
  int iteration = 0;

  while (true) {
    // bookkeeping of the previous iteration, then the loop's stopping tests
    if (last_step_successful) {
      ++sum.num_successful_steps;
      if (x_cost < minimum_cost) {
        minimum_cost = x_cost;
        best[0] = x[0];
        best[1] = x[1];
        best[2] = x[2];
      }
    }
    const double gmax = std::max(std::abs(at_x.g[0]), std::max(std::abs(at_x.g[1]), std::abs(at_x.g[2])));
    CeresIterationTrace rec;
    rec.x_cost = x_cost;
    rec.gradient_max_norm = gmax;
    rec.radius_before = rec.radius_after = radius;
    rec.reused_diagonal = reuse_diagonal;
    auto record = [&](int outcome) {
      rec.outcome = outcome;
      rec.radius_after = radius;
      if (trace != nullptr) trace->push_back(rec);
    };
    if (iteration >= options.max_num_iterations) {
      sum.termination = kCeresNoConvergence;
      record(kStepLoopExit);
      break;
    }
    if (gmax <= kGradientTolerance) {
      sum.termination = kCeresGradientTolerance;
      record(kStepLoopExit);
      break;
    }
    if (radius <= kMinRadius) {
      sum.termination = kCeresMinTrustRegionRadius;
      record(kStepLoopExit);
      break;
    }
    ++iteration;
    last_step_successful = false;

    // scaled normal equations: Js = J diag(scale)
    const double hs[6] = {at_x.h[0] * scale[0] * scale[0], at_x.h[1] * scale[0] * scale[1],
                          at_x.h[2] * scale[0] * scale[2], at_x.h[3] * scale[1] * scale[1],
                          at_x.h[4] * scale[1] * scale[2], at_x.h[5] * scale[2] * scale[2]};
    const double gs[3] = {at_x.g[0] * scale[0], at_x.g[1] * scale[1], at_x.g[2] * scale[2]};
    if (!reuse_diagonal) {
      diagonal[0] = std::min(std::max(hs[0], kMinLmDiagonal), kMaxLmDiagonal);
      diagonal[1] = std::min(std::max(hs[3], kMinLmDiagonal), kMaxLmDiagonal);
      diagonal[2] = std::min(std::max(hs[5], kMinLmDiagonal), kMaxLmDiagonal);
    }
    // min |Js y - r|^2 + |D y|^2 with D^2 = diagonal / radius; step = -y
    const double a[6] = {hs[0] + diagonal[0] / radius, hs[1], hs[2],
                         hs[3] + diagonal[1] / radius, hs[4], hs[5] + diagonal[2] / radius};
    double y[3];
    bool valid = SolveSpd3(a, gs, y);
    reuse_diagonal = true;
    double step[3] = {0., 0., 0.}, model_cost_change = 0.;
    if (valid) {
      step[0] = -y[0];
      step[1] = -y[1];
      step[2] = -y[2];
      // cost - model cost at the step = -(Js step)^T (r + Js step / 2)
      const double hs_step[3] = {hs[0] * step[0] + hs[1] * step[1] + hs[2] * step[2],
                                 hs[1] * step[0] + hs[3] * step[1] + hs[4] * step[2],
                                 hs[2] * step[0] + hs[4] * step[1] + hs[5] * step[2]};
      model_cost_change =
          -((step[0] * gs[0] + step[1] * gs[1] + step[2] * gs[2]) +
            0.5 * (step[0] * hs_step[0] + step[1] * hs_step[1] + step[2] * hs_step[2]));
      valid = !(model_cost_change < 0.0);
    }
    if (!valid) {
      if (++num_invalid >= kMaxConsecutiveInvalidSteps) {
        sum.termination = kCeresInvalidSteps;
        record(kStepInvalid);
        break;
      }
      // treated as a rejected step whose diagonal is recomputed
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = false;
      record(kStepInvalid);
      continue;
    }
    num_invalid = 0;

    const double delta[3] = {step[0] * scale[0], step[1] * scale[1], step[2] * scale[2]};
    const double cand[3] = {x[0] + delta[0], x[1] + delta[1], x[2] + delta[2]};
    const double candidate_cost =
        Evaluate(grid, cloud, options, target_translation, target_angle, cand, false).cost;

    const double diff[3] = {x[0] - cand[0], x[1] - cand[1], x[2] - cand[2]};
    rec.candidate_cost = candidate_cost;
    rec.model_cost_change = model_cost_change;
    rec.step_norm = Norm3(diff);
    rec.step_norm_threshold = kParameterTolerance * (x_norm + kParameterTolerance);
    if (Norm3(diff) <= kParameterTolerance * (x_norm + kParameterTolerance)) {
      sum.termination = kCeresParameterTolerance;   // the step is not taken
      record(kStepParameterTolerance);
      break;
    }
    rec.cost_change = std::abs(x_cost - candidate_cost);
    rec.cost_change_threshold = kFunctionTolerance * x_cost;
    if (std::abs(x_cost - candidate_cost) <= kFunctionTolerance * x_cost) {
      sum.termination = kCeresFunctionTolerance;    // the step is not taken
      record(kStepFunctionTolerance);
      break;
    }

    const double relative_decrease = (current_cost - candidate_cost) / model_cost_change;
    const double historical_decrease =
        (reference_cost - candidate_cost) / (acc_reference + model_cost_change);
    const double step_quality = std::max(relative_decrease, historical_decrease);
    rec.step_quality = step_quality;

    if (step_quality > kMinRelativeDecrease) {
      x[0] = cand[0];
      x[1] = cand[1];
      x[2] = cand[2];
      x_norm = Norm3(x);
      at_x = Evaluate(grid, cloud, options, target_translation, target_angle, x, true);
      x_cost = at_x.cost;
      last_step_successful = true;
      // LevenbergMarquardtStrategy::StepAccepted
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * step_quality - 1.0, 3));
      radius = std::min(kMaxRadius, radius);
      decrease_factor = 2.0;
      reuse_diagonal = false;
      // step evaluator: accepted
      current_cost = candidate_cost;
      rec.evaluator_minimum_cost = ev_minimum_cost;
      rec.evaluator_candidate_cost = candidate_cost_ev;
      acc_candidate += model_cost_change;
      acc_reference += model_cost_change;
      if (current_cost < ev_minimum_cost) {
        ev_minimum_cost = current_cost;
        num_nonmonotonic = 0;
        candidate_cost_ev = current_cost;
        acc_candidate = 0.;
      } else {
        ++num_nonmonotonic;
        if (current_cost > candidate_cost_ev) {
          candidate_cost_ev = current_cost;
          acc_candidate = 0.;
        }
      }
      if (num_nonmonotonic == max_nonmonotonic) {
        reference_cost = candidate_cost_ev;
        acc_reference = acc_candidate;
        rec.reference_switched = true;
      }
      record(kStepAccepted);
    } else {
      // LevenbergMarquardtStrategy::StepRejected
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = true;
      record(kStepRejected);
    }
  }
  sum.iterations = iteration;
  sum.final_cost = minimum_cost;
  pose_estimate[0] = best[0];
  pose_estimate[1] = best[1];
  pose_estimate[2] = best[2];
  if (summary != nullptr) *summary = sum;
}

}  // namespace oracle
