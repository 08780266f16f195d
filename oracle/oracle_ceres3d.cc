// ORACLE — TEST INFRASTRUCTURE ONLY.  See oracle_ceres3d.h ("parity unpinned" against Ceres).
#include "oracle_ceres3d.h"

#include <algorithm>
#include <cmath>

namespace oracle {
namespace {

// A dual number over (x, y, z) with Ceres' Jet arithmetic (ceres/jet.h): the value part of
// every operation is the plain-double operation, the derivative part the product / sum rule
// in the order jet.h writes it.
struct D3 {
  double a;
  double v[3];
};
D3 operator+(const D3& f, const D3& g) {
  return D3{f.a + g.a, {f.v[0] + g.v[0], f.v[1] + g.v[1], f.v[2] + g.v[2]}};
}
D3 operator-(const D3& f, const D3& g) {
  return D3{f.a - g.a, {f.v[0] - g.v[0], f.v[1] - g.v[1], f.v[2] - g.v[2]}};
}
D3 operator+(const D3& f, double s) { return D3{f.a + s, {f.v[0], f.v[1], f.v[2]}}; }
D3 operator*(const D3& f, const D3& g) {
  return D3{f.a * g.a, {f.a * g.v[0] + f.v[0] * g.a, f.a * g.v[1] + f.v[1] * g.a,
                        f.a * g.v[2] + f.v[2] * g.a}};
}
D3 operator*(const D3& f, double s) { return D3{f.a * s, {f.v[0] * s, f.v[1] * s, f.v[2] * s}}; }
D3 operator*(double s, const D3& f) { return f * s; }

// interpolated_grid.h:115-135: centre of the voxel whose centre is at most (x, y, z) per axis
void CenterOfLowerVoxel(const HybridGrid& grid, double x, double y, double z, float center[3]) {
  const Array3i index = grid.GetCellIndex(
      Vec3f{static_cast<float>(x), static_cast<float>(y), static_cast<float>(z)});
  // HybridGrid::GetCenterOfCell (mapping/3d/hybrid_grid.h:444-446)
  center[0] = static_cast<float>(index.x) * grid.resolution();
  center[1] = static_cast<float>(index.y) * grid.resolution();
  center[2] = static_cast<float>(index.z) * grid.resolution();
  if (center[0] > x) center[0] -= grid.resolution();
  if (center[1] > y) center[1] -= grid.resolution();
  if (center[2] > z) center[2] -= grid.resolution();
}

D3 Interpolate(const HybridGrid& grid, double x, double y, double z, bool dual) {
  float lower[3];
  CenterOfLowerVoxel(grid, x, y, z, lower);
  // :98-112
  const double x1 = lower[0], y1 = lower[1], z1 = lower[2];
  const double x2 = lower[0] + grid.resolution();
  const double y2 = lower[1] + grid.resolution();
  const double z2 = lower[2] + grid.resolution();
  const Array3i i1 = grid.GetCellIndex(
      Vec3f{static_cast<float>(x1), static_cast<float>(y1), static_cast<float>(z1)});
  auto value = [&](int dx, int dy, int dz) {
    return static_cast<double>(grid.GetProbability(Array3i{i1.x + dx, i1.y + dy, i1.z + dz}));
  };
  const double q111 = value(0, 0, 0), q112 = value(0, 0, 1), q121 = value(0, 1, 0);
  const double q122 = value(0, 1, 1), q211 = value(1, 0, 0), q212 = value(1, 0, 1);
  const double q221 = value(1, 1, 0), q222 = value(1, 1, 1);
  // :68-70 — on dual numbers the division multiplies value and derivative by the reciprocal
  D3 nx, ny, nz;
  if (dual) {
    const double ix = 1.0 / (x2 - x1), iy = 1.0 / (y2 - y1), iz = 1.0 / (z2 - z1);
    nx = D3{(x - x1) * ix, {1.0 * ix, 0.0 * ix, 0.0 * ix}};
    ny = D3{(y - y1) * iy, {0.0 * iy, 1.0 * iy, 0.0 * iy}};
    nz = D3{(z - z1) * iz, {0.0 * iz, 0.0 * iz, 1.0 * iz}};
  } else {
    nx = D3{(x - x1) / (x2 - x1), {0., 0., 0.}};
    ny = D3{(y - y1) / (y2 - y1), {0., 0., 0.}};
    nz = D3{(z - z1) / (z2 - z1), {0., 0., 0.}};
  }
  // :72-95 — smoothstep blends along z, then y, then x
  const D3 nxx = nx * nx, nxxx = nx * nxx;
  const D3 nyy = ny * ny, nyyy = ny * nyy;
  const D3 nzz = nz * nz, nzzz = nz * nzz;
  const D3 q11 = (q111 - q112) * nzzz * 2. + (q112 - q111) * nzz * 3. + q111;
  const D3 q12 = (q121 - q122) * nzzz * 2. + (q122 - q121) * nzz * 3. + q121;
  const D3 q21 = (q211 - q212) * nzzz * 2. + (q212 - q211) * nzz * 3. + q211;
  const D3 q22 = (q221 - q222) * nzzz * 2. + (q222 - q221) * nzz * 3. + q221;
  const D3 q1 = (q11 - q12) * nyyy * 2. + (q12 - q11) * nyy * 3. + q11;
  const D3 q2 = (q21 - q22) * nyyy * 2. + (q22 - q21) * nyy * 3. + q21;
  return (q1 - q2) * nxxx * 2. + (q2 - q1) * nxx * 3. + q1;
}

void Cross(const double a[3], const double b[3], double out[3]) {
  out[0] = a[1] * b[2] - a[2] * b[1];
  out[1] = a[2] * b[0] - a[0] * b[2];
  out[2] = a[0] * b[1] - a[1] * b[0];
}

// world = q * p + t with Eigen's quaternion-vector product (QuaternionBase::_transformVector,
// not normalising q) as transform/rigid_transform.h:192-196 applies it; dworld[k][c] =
// d world[c] / d param k for k = {tx, ty, tz, qw, qx, qy, qz}.
void TransformPoint(const double pose[7], const double p[3], double world[3],
                    double dworld[7][3]) {
  const double w = pose[3];
  const double qv[3] = {pose[4], pose[5], pose[6]};
  double uv[3];
  Cross(qv, p, uv);
  uv[0] += uv[0];
  uv[1] += uv[1];
  uv[2] += uv[2];
  double c[3];
  Cross(qv, uv, c);
  for (int k = 0; k < 3; ++k) world[k] = ((p[k] + w * uv[k]) + c[k]) + pose[k];
  if (dworld == nullptr) return;
  for (int k = 0; k < 3; ++k)
    for (int cc = 0; cc < 3; ++cc) dworld[k][cc] = k == cc ? 1.0 : 0.0;
  for (int cc = 0; cc < 3; ++cc) dworld[3][cc] = uv[cc];   // d/dw
  for (int k = 0; k < 3; ++k) {                            // d/d qv[k]
    double e[3] = {0., 0., 0.};
    e[k] = 1.0;
    double duv[3], t1[3], t2[3];
    Cross(e, p, duv);
    duv[0] += duv[0];
    duv[1] += duv[1];
    duv[2] += duv[2];
    Cross(e, uv, t1);
    Cross(qv, duv, t2);
    for (int cc = 0; cc < 3; ++cc) dworld[4 + k][cc] = (w * duv[cc] + t1[cc]) + t2[cc];
  }
}

// ceres::QuaternionParameterization::ComputeJacobian (4 x 3, row-major)
void PlusJacobian(const double q[4], double jac[12]) {
  jac[0] = -q[1]; jac[1] = -q[2]; jac[2] = -q[3];
  jac[3] = q[0];  jac[4] = q[3];  jac[5] = -q[2];
  jac[6] = -q[3]; jac[7] = q[0];  jac[8] = q[1];
  jac[9] = q[2];  jac[10] = -q[1]; jac[11] = q[0];
}

// x (+) delta: translation is Euclidean, the rotation block is
// ceres::QuaternionParameterization::Plus (q_delta * q, |delta| = half the rotation angle)
void Plus(const double x[7], const double delta[6], double out[7]) {
  for (int k = 0; k < 3; ++k) out[k] = x[k] + delta[k];
  const double* d = delta + 3;
  const double norm_delta = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (norm_delta > 0.0) {
    const double sin_delta_by_delta = std::sin(norm_delta) / norm_delta;
    const double z[4] = {std::cos(norm_delta), sin_delta_by_delta * d[0],
                         sin_delta_by_delta * d[1], sin_delta_by_delta * d[2]};
    const double* w = x + 3;
    out[3] = z[0] * w[0] - z[1] * w[1] - z[2] * w[2] - z[3] * w[3];
    out[4] = z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2];
    out[5] = z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1];
    out[6] = z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0];
  } else {
    for (int k = 3; k < 7; ++k) out[k] = x[k];
  }
}

}  // namespace

double InterpolatedProbability(const HybridGrid& grid, double x, double y, double z,
                               double gradient[3]) {
  const D3 f = Interpolate(grid, x, y, z, gradient != nullptr);
  if (gradient != nullptr) {
    gradient[0] = f.v[0];
    gradient[1] = f.v[1];
    gradient[2] = f.v[2];
  }
  return f.a;
}

void EvaluateCeresResiduals3D(const std::vector<PointCloudAndHybridGrid>& clouds,
                              const CeresScanMatcherOptions3D& options,
                              const double target_translation[3],
                              const double target_rotation[4], const double pose[7],
                              std::vector<double>* residuals, std::vector<double>* jacobian) {
  size_t rows = 6;
  for (const auto& c : clouds) rows += c.point_cloud->size();
  residuals->assign(rows, 0.);
  if (jacobian != nullptr) jacobian->assign(rows * 6, 0.);
  double plus_jacobian[12];
  PlusJacobian(pose + 3, plus_jacobian);
  auto to_local = [&](const double ambient[7], double* row) {
    row[0] = ambient[0];
    row[1] = ambient[1];
    row[2] = ambient[2];
    for (int k = 0; k < 3; ++k)
      row[3 + k] = ambient[3] * plus_jacobian[k] + ambient[4] * plus_jacobian[3 + k] +
                   ambient[5] * plus_jacobian[6 + k] + ambient[6] * plus_jacobian[9 + k];
  };
  size_t row = 0;
  for (size_t b = 0; b < clouds.size(); ++b) {
    const PointCloud& cloud = *clouds[b].point_cloud;
    const HybridGrid& grid = *clouds[b].hybrid_grid;
    // ceres_scan_matcher_3d.cc:119-121
    const double scaling =
        options.occupied_space_weight[b] / std::sqrt(static_cast<double>(cloud.size()));
    for (size_t i = 0; i < cloud.size(); ++i, ++row) {
      const double p[3] = {static_cast<double>(cloud[i].x), static_cast<double>(cloud[i].y),
                           static_cast<double>(cloud[i].z)};
      double world[3], dworld[7][3];
      TransformPoint(pose, p, world, jacobian != nullptr ? dworld : nullptr);
      double grad[3];
      const double probability = InterpolatedProbability(grid, world[0], world[1], world[2],
                                                         jacobian != nullptr ? grad : nullptr);
      (*residuals)[row] = scaling * (1. - probability);   // occupied_space_cost_function_3d.h:75
      if (jacobian == nullptr) continue;
      double ambient[7];
      for (int k = 0; k < 7; ++k) {
        const double dp = (grad[0] * dworld[k][0] + grad[1] * dworld[k][1]) + grad[2] * dworld[k][2];
        ambient[k] = scaling * (-dp);
      }
      to_local(ambient, &(*jacobian)[6 * row]);
    }
  }
  // translation_delta_cost_functor_3d.h: scaling * (translation - target)
  for (int k = 0; k < 3; ++k, ++row) {
    (*residuals)[row] = options.translation_weight * (pose[k] - target_translation[k]);
    if (jacobian != nullptr) (*jacobian)[6 * row + k] = options.translation_weight;
  }
  // rotation_delta_cost_functor_3d.h:42-53: vector part of target^-1 * rotation
  const double z[4] = {target_rotation[0], -target_rotation[1], -target_rotation[2],
                       -target_rotation[3]};
  const double* w = pose + 3;
  const double delta[3] = {z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2],
                           z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1],
                           z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0]};
  // d delta[k] / d (w0, w1, w2, w3)
  const double ddelta[3][4] = {{z[1], z[0], -z[3], z[2]},
                               {z[2], z[3], z[0], -z[1]},
                               {z[3], -z[2], z[1], z[0]}};
  for (int k = 0; k < 3; ++k, ++row) {
    (*residuals)[row] = options.rotation_weight * delta[k];
    if (jacobian == nullptr) continue;
    double ambient[7] = {0., 0., 0., 0., 0., 0., 0.};
    for (int c = 0; c < 4; ++c) ambient[3 + c] = options.rotation_weight * ddelta[k][c];
    to_local(ambient, &(*jacobian)[6 * row]);
  }
}

namespace {

constexpr int kN = 6;                       // tangent-space parameters
constexpr int kH = kN * (kN + 1) / 2;       // upper triangle, row-major

struct Normal {
  double cost = 0.;
  double g[kN] = {};
  double h[kH] = {};
};

inline int Tri(int i, int j) { return i * kN - i * (i - 1) / 2 + (j - i); }   // i <= j

Normal Evaluate(const std::vector<PointCloudAndHybridGrid>& clouds,
                const CeresScanMatcherOptions3D& options, const double target_t[3],
                const double target_q[4], const double x[7], bool with_jacobian) {
  std::vector<double> r, j;
  EvaluateCeresResiduals3D(clouds, options, target_t, target_q, x, &r,
                           with_jacobian ? &j : nullptr);
  Normal nm;
  double sq = 0.;
  for (size_t i = 0; i < r.size(); ++i) {
    sq += r[i] * r[i];
    if (!with_jacobian) continue;
    const double* ji = &j[kN * i];
    for (int a = 0; a < kN; ++a) {
      nm.g[a] += ji[a] * r[i];
      for (int b = a; b < kN; ++b) nm.h[Tri(a, b)] += ji[a] * ji[b];
    }
  }
  nm.cost = 0.5 * sq;
  return nm;
}

// Cholesky solve of the symmetric positive definite system A y = b (A as upper triangle)
bool SolveSpd(const double* a, const double* b, double* y) {
  double l[kN][kN] = {};
  for (int i = 0; i < kN; ++i) {
    for (int j = 0; j <= i; ++j) {
      double s = a[Tri(j, i)];
      for (int k = 0; k < j; ++k) s -= l[i][k] * l[j][k];
      if (i == j) {
        if (!(s > 0.)) return false;
        l[i][i] = std::sqrt(s);
      } else {
        l[i][j] = s / l[j][j];
      }
    }
  }
  double z[kN];
  for (int i = 0; i < kN; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= l[i][k] * z[k];
    z[i] = s / l[i][i];
  }
  for (int i = kN - 1; i >= 0; --i) {
    double s = z[i];
    for (int k = i + 1; k < kN; ++k) s -= l[k][i] * y[k];
    y[i] = s / l[i][i];
  }
  for (int i = 0; i < kN; ++i)
    if (!std::isfinite(y[i])) return false;
  return true;
}

double Norm(const double* v, int n) {
  double s = 0.;
  for (int i = 0; i < n; ++i) s += v[i] * v[i];
  return std::sqrt(s);
}

}  // namespace

void CeresMatch3D(const std::vector<PointCloudAndHybridGrid>& clouds,
                  const CeresScanMatcherOptions3D& options, const double target_translation[3],
                  const double initial_pose[7], double pose_estimate[7],
                  CeresSummary2D* summary, std::vector<CeresIterationTrace>* trace) {
  const double kInitialRadius = 1e4, kMaxRadius = 1e16, kMinRadius = 1e-32;
  const double kMinRelativeDecrease = 1e-3;
  const double kMinLmDiagonal = 1e-6, kMaxLmDiagonal = 1e32;
  const int kMaxConsecutiveInvalidSteps = 5;
  const double kFunctionTolerance = 1e-6, kGradientTolerance = 1e-10, kParameterTolerance = 1e-8;
  const int max_nonmonotonic = options.use_nonmonotonic_steps ? 5 : 0;

  double x[7], best[7];
  for (int k = 0; k < 7; ++k) x[k] = best[k] = initial_pose[k];
  const double* target_rotation = initial_pose + 3;   // ceres_scan_matcher_3d.cc:148-151
  CeresSummary2D sum;

  Normal at_x = Evaluate(clouds, options, target_translation, target_rotation, x, true);
  double x_cost = at_x.cost, x_norm = Norm(x, 7);
  sum.initial_cost = x_cost;
  double minimum_cost = x_cost;
  double scale[kN];
  for (int a = 0; a < kN; ++a) scale[a] = 1.0 / (1.0 + std::sqrt(at_x.h[Tri(a, a)]));
  double radius = kInitialRadius, decrease_factor = 2.0;
  bool reuse_diagonal = false;
  double diagonal[kN] = {};
  double current_cost = x_cost, reference_cost = x_cost, candidate_cost_ev = x_cost;
  double ev_minimum_cost = x_cost;
  double acc_reference = 0., acc_candidate = 0.;
  int num_nonmonotonic = 0, num_invalid = 0, iteration = 0;
  bool last_step_successful = false;

  while (true) {
    if (last_step_successful) {
      ++sum.num_successful_steps;
      if (x_cost < minimum_cost) {
        minimum_cost = x_cost;
        for (int k = 0; k < 7; ++k) best[k] = x[k];
      }
    }
    // |x - (x (+) -g)|_inf
    double gmax = 0.;
    {
      double neg[kN], moved[7];
      for (int a = 0; a < kN; ++a) neg[a] = -at_x.g[a];
      Plus(x, neg, moved);
      for (int k = 0; k < 7; ++k) gmax = std::max(gmax, std::abs(x[k] - moved[k]));
    }
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

    double hs[kH], gs[kN];
    for (int a = 0; a < kN; ++a) {
      gs[a] = at_x.g[a] * scale[a];
      for (int b = a; b < kN; ++b) hs[Tri(a, b)] = at_x.h[Tri(a, b)] * scale[a] * scale[b];
    }
    if (!reuse_diagonal)
      for (int a = 0; a < kN; ++a)
        diagonal[a] = std::min(std::max(hs[Tri(a, a)], kMinLmDiagonal), kMaxLmDiagonal);
    double am[kH];
    for (int i = 0; i < kH; ++i) am[i] = hs[i];
    for (int a = 0; a < kN; ++a) am[Tri(a, a)] = hs[Tri(a, a)] + diagonal[a] / radius;
    double y[kN];
    bool valid = SolveSpd(am, gs, y);
    reuse_diagonal = true;
    double step[kN] = {}, model_cost_change = 0.;
    if (valid) {
      for (int a = 0; a < kN; ++a) step[a] = -y[a];
      double sg = 0., shs = 0.;
      for (int a = 0; a < kN; ++a) {
        sg += step[a] * gs[a];
        double row = 0.;
        for (int b = 0; b < kN; ++b) row += hs[a <= b ? Tri(a, b) : Tri(b, a)] * step[b];
        shs += step[a] * row;
      }
      model_cost_change = -(sg + 0.5 * shs);
      valid = !(model_cost_change < 0.0);
    }
    if (!valid) {
      if (++num_invalid >= kMaxConsecutiveInvalidSteps) {
        sum.termination = kCeresInvalidSteps;
        record(kStepInvalid);
        break;
      }
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = false;
      record(kStepInvalid);
      continue;
    }
    num_invalid = 0;

    double delta[kN], cand[7];
    for (int a = 0; a < kN; ++a) delta[a] = step[a] * scale[a];
    Plus(x, delta, cand);
    const double candidate_cost =
        Evaluate(clouds, options, target_translation, target_rotation, cand, false).cost;
    double diff[7];
    for (int k = 0; k < 7; ++k) diff[k] = x[k] - cand[k];
    rec.candidate_cost = candidate_cost;
    rec.model_cost_change = model_cost_change;
    rec.step_norm = Norm(diff, 7);
    rec.step_norm_threshold = kParameterTolerance * (x_norm + kParameterTolerance);
    if (Norm(diff, 7) <= kParameterTolerance * (x_norm + kParameterTolerance)) {
      sum.termination = kCeresParameterTolerance;
      record(kStepParameterTolerance);
      break;
    }
    rec.cost_change = std::abs(x_cost - candidate_cost);
    rec.cost_change_threshold = kFunctionTolerance * x_cost;
    if (std::abs(x_cost - candidate_cost) <= kFunctionTolerance * x_cost) {
      sum.termination = kCeresFunctionTolerance;
      record(kStepFunctionTolerance);
      break;
    }
    const double relative_decrease = (current_cost - candidate_cost) / model_cost_change;
    const double historical_decrease =
        (reference_cost - candidate_cost) / (acc_reference + model_cost_change);
    const double step_quality = std::max(relative_decrease, historical_decrease);
    rec.step_quality = step_quality;
    if (step_quality > kMinRelativeDecrease) {
      for (int k = 0; k < 7; ++k) x[k] = cand[k];
      x_norm = Norm(x, 7);
      at_x = Evaluate(clouds, options, target_translation, target_rotation, x, true);
      x_cost = at_x.cost;
      last_step_successful = true;
      const double t = 2.0 * step_quality - 1.0;
      radius = radius / std::max(1.0 / 3.0, 1.0 - t * t * t);
      radius = std::min(kMaxRadius, radius);
      decrease_factor = 2.0;
      reuse_diagonal = false;
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
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = true;
      record(kStepRejected);
    }
  }
  sum.iterations = iteration;
  sum.final_cost = minimum_cost;
  for (int k = 0; k < 7; ++k) pose_estimate[k] = best[k];
  if (summary != nullptr) *summary = sum;
}

}  // namespace oracle
