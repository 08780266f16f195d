// Post-match refinement: CeresScanMatcher2D::Match
// (mapping/internal/2d/scan_matching/ceres_scan_matcher_2d.cc:62-107), the call
// ConstraintBuilder2D makes on every found match (constraint_builder_2d.cc:245-249).
//
// Ceres itself is not linked (it is a third-party dependency of the reference, absent here,
// pinned there at commit 58c5edae, bazel/repositories.bzl:136-142).  What runs instead is a
// batched solver for exactly the problem that call builds — 3 parameters {x, y, theta},
// n + 3 residuals — one CTA per match, the whole trust-region loop on the device:
//   * residuals of the reference's cost functors (occupied_space_cost_function_2d.cc:42-69,
//     translation_delta_cost_functor_2d.h:41-45, rotation_delta_cost_functor_2d.h:40-43),
//     the occupied-space term through Ceres' BiCubicInterpolator (Catmull-Rom splines over the
//     4 x 4 cells around the point) with the kPadding = INT_MAX / 4 coordinate shift the
//     reference applies (:61-66, :72) — the shift quantises the interpolation coordinate to
//     2^-23 of a cell, so it has to be reproduced;
//   * threads stride the scan points, accumulate cost = 1/2 |r|^2, g = J^T r and H = J^T J
//     (10 doubles) and the block reduces them; thread 0 then runs the trust-region minimiser
//     of trust_region.cuh with the 3 parameters, x (+) delta = x + delta and the gradient
//     tolerance measured as max |g_i|.
// Doubles throughout, compiled without FMA contraction (Makefile: -fmad=false for this
// file) so that every per-point value is the one the oracle's restatement computes; sums are
// block-tree ordered, cos / sin come from the device's double-precision routines (<= 2 ulp).
#include <algorithm>
#include <climits>
#include <cmath>

// CSM_REFINE_DEVICE_ONLY: tests/emulation/refine2d_emulation.cc includes the kernels below
// into a CPU harness (SIMT shims, one std::thread per CUDA thread) to check their control
// flow against the oracle where no GPU is present; the library itself never defines it.
#ifndef CSM_REFINE_DEVICE_ONLY
#include "rtgrid.cuh"
#endif
#include "trust_region.cuh"

namespace csm {

constexpr int kPadding = INT_MAX / 4;   // occupied_space_cost_function_2d.cc:72

struct RefJobDev {
  const uint16_t* cells;   // the submap grid on the device (row pitch `pitch`)
  int nx, ny, pitch, n;
  long long xyz_off;       // first float of the job's cloud in the upload buffer
  double resolution, max_x, max_y;
  double target[2];        // target_translation
  double init[3];          // initial_pose_estimate {x, y, angle}
  // TSDF2D jobs only (wcells == nullptr selects the ProbabilityGrid cost, as
  // Grid2D::GetGridType() does in ceres_scan_matcher_2d.cc:74-91): the weight cells and the
  // TSDValueConverter constants of the job's grid (MakeTsdfConversion)
  const uint16_t* wcells;
  float tsd_scale, tsd_bias, w_scale, w_bias, truncation;
};

struct RefOpts {
  double occupied_space_weight, translation_weight, rotation_weight;
  int use_nonmonotonic_steps, max_num_iterations;
  float k_scale, cost_bias, max_cost;   // value -> correspondence cost (value_conversion_tables.cc:29-37)
};

using RefResultDev = ResultDev<3>;   // trust_region.cuh

// GridArrayAdapter::GetValue (occupied_space_cost_function_2d.cc:78-87)
__device__ __forceinline__ double PaddedValue(const RefJobDev& J, const RefOpts& P, int row,
                                              int column) {
  const int iy = row - kPadding, ix = column - kPadding;
  if (ix < 0 || iy < 0 || ix >= J.nx || iy >= J.ny) return static_cast<double>(P.max_cost);
  const int value = __ldg(J.cells + static_cast<size_t>(iy) * J.pitch + ix) & 0x7fff;
  const float cost = value == 0 ? P.max_cost
                                : __fadd_rn(__fmul_rn(__int2float_rn(value), P.k_scale), P.cost_bias);
  return static_cast<double>(cost);
}

// ceres/cubic_interpolation.h, CubicHermiteSpline (Catmull-Rom)
template <bool kValue, bool kDeriv>
__device__ __forceinline__ void CubicHermiteSpline(double p0, double p1, double p2, double p3,
                                                   double x, double* f, double* dfdx) {
  const double a = 0.5 * (-p0 + 3.0 * p1 - 3.0 * p2 + p3);
  const double b = 0.5 * (2.0 * p0 - 5.0 * p1 + 4.0 * p2 - p3);
  const double c = 0.5 * (-p0 + p2);
  const double d = p1;
  if (kValue) *f = d + x * (c + x * (b + x * a));
  if (kDeriv) *dfdx = c + x * (2.0 * b + 3.0 * a * x);
}

// BiCubicInterpolator::Evaluate
template <bool kJac>
__device__ __forceinline__ void BiCubic(const RefJobDev& J, const RefOpts& P, double r, double c,
                                        double* f, double* dfdr, double* dfdc) {
  const int row = static_cast<int>(floor(r));
  const int col = static_cast<int>(floor(c));
  double fr[4], dfr[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int rr = row - 1 + k;
    CubicHermiteSpline<true, kJac>(PaddedValue(J, P, rr, col - 1), PaddedValue(J, P, rr, col),
                                   PaddedValue(J, P, rr, col + 1), PaddedValue(J, P, rr, col + 2),
                                   c - col, &fr[k], &dfr[k]);
  }
  CubicHermiteSpline<true, kJac>(fr[0], fr[1], fr[2], fr[3], r - row, f, dfdr);
  if (kJac) CubicHermiteSpline<true, false>(dfr[0], dfr[1], dfr[2], dfr[3], r - row, dfdc, nullptr);
}

// One occupied-space residual (and its Jacobian row) at pose x with cs = cos, sn = sin of x[2].
template <bool kJac>
__device__ __forceinline__ void PointResidual(const RefJobDev& J, const RefOpts& P,
                                              double scaling, const double* x, double cs,
                                              double sn, double px, double py, double* res,
                                              double* jrow) {
  const double wx = (cs * px + (-sn) * py) + x[0] * 1.0;
  const double wy = (sn * px + cs * py) + x[1] * 1.0;
  double f, dfdr = 0., dfdc = 0.;
  if (!kJac) {
    const double r = (J.max_x - wx) / J.resolution - 0.5 + static_cast<double>(kPadding);
    const double c = (J.max_y - wy) / J.resolution - 0.5 + static_cast<double>(kPadding);
    BiCubic<false>(J, P, r, c, &f, nullptr, nullptr);
    *res = scaling * f;
    return;
  }
  // on dual numbers the division by the resolution multiplies by its reciprocal
  const double inverse_resolution = 1.0 / J.resolution;
  const double r = (J.max_x - wx) * inverse_resolution - 0.5 + static_cast<double>(kPadding);
  const double c = (J.max_y - wy) * inverse_resolution - 0.5 + static_cast<double>(kPadding);
  BiCubic<true>(J, P, r, c, &f, &dfdr, &dfdc);
  *res = scaling * f;
  const double dwx[3] = {1.0, 0.0, (-sn) * px + (-cs) * py};
  const double dwy[3] = {0.0, 1.0, cs * px + (-sn) * py};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double dr = -dwx[k] * inverse_resolution, dc = -dwy[k] * inverse_resolution;
    jrow[k] = scaling * (dfdr * dr + dfdc * dc);
  }
}

// ---- TSDFMatchCostFunction2D (tsdf_match_cost_function_2d.cc:42-65) through
// InterpolatedTSDF2D (interpolated_tsdf_2d.h) -----------------------------------------------
// r_i = n * scaling * cost_i * w_i / W with W = sum_j w_j: not point-separable, so one
// evaluation is two block passes — W and dW/d(x, y, theta) first, then the residuals.  On dual
// numbers every operation follows ceres/jet.h (a Jet divided by a Jet multiplies by the
// reciprocal of the denominator's value); the interpolation's lower pixel is found on the
// scalar part, in float, as the reference does.

// TSDF2D::GetWeight (tsdf_2d.cc:85-91): 0 outside the limits and for value 0
__device__ __forceinline__ float TsdfWeight(const RefJobDev& J, int ix, int iy) {
  if (ix < 0 || iy < 0 || ix >= J.nx || iy >= J.ny) return 0.f;
  const int value = __ldg(J.wcells + static_cast<size_t>(iy) * J.pitch + ix) & 0x7fff;
  return value == 0 ? 0.f : __fadd_rn(__fmul_rn(__int2float_rn(value), J.w_scale), J.w_bias);
}

// Grid2D::GetCorrespondenceCost with the TSDF bounds +-truncation: value 0 (and outside the
// limits) gives +truncation; the update marker is masked
__device__ __forceinline__ float TsdfCost(const RefJobDev& J, int ix, int iy) {
  if (ix < 0 || iy < 0 || ix >= J.nx || iy >= J.ny) return J.truncation;
  const int value = __ldg(J.cells + static_cast<size_t>(iy) * J.pitch + ix) & 0x7fff;
  return value == 0 ? J.truncation
                    : __fadd_rn(__fmul_rn(__int2float_rn(value), J.tsd_scale), J.tsd_bias);
}

// MapLimits::GetCellIndex of a float point: ix from y, iy from x (double arithmetic, lround)
__device__ __forceinline__ void TsdfCellIndex(const RefJobDev& J, float px, float py, int* ix,
                                              int* iy) {
  *ix = static_cast<int>(lround((J.max_y - static_cast<double>(py)) / J.resolution - 0.5));
  *iy = static_cast<int>(lround((J.max_x - static_cast<double>(px)) / J.resolution - 0.5));
}

struct TsdfCorners {
  float x1, y1, dx, dy;          // centre of the lower pixel, x2 - x1 and y2 - y1 (float)
  float w11, w12, w21, w22;
  int ix, iy;                    // index1
};

// ComputeInterpolationDataPoints + the four weights around (x, y)
__device__ __forceinline__ void TsdfCornersAt(const RefJobDev& J, double x, double y,
                                              TsdfCorners* c) {
  int cx, cy;   // CenterOfLowerPixel: GetCellCenter(GetCellIndex(Vector2f(x, y)))
  TsdfCellIndex(J, static_cast<float>(x), static_cast<float>(y), &cx, &cy);
  float lx = static_cast<float>(J.max_x - J.resolution * (cy + 0.5));
  float ly = static_cast<float>(J.max_y - J.resolution * (cx + 0.5));
  if (lx > x) lx = static_cast<float>(lx - J.resolution);
  if (ly > y) ly = static_cast<float>(ly - J.resolution);
  const float res = static_cast<float>(J.resolution);
  c->x1 = lx;
  c->y1 = ly;
  c->dx = __fadd_rn(lx, res) - lx;
  c->dy = __fadd_rn(ly, res) - ly;
  TsdfCellIndex(J, lx, ly, &c->ix, &c->iy);
  c->w11 = TsdfWeight(J, c->ix, c->iy);
  c->w12 = TsdfWeight(J, c->ix - 1, c->iy);
  c->w21 = TsdfWeight(J, c->ix, c->iy - 1);
  c->w22 = TsdfWeight(J, c->ix - 1, c->iy - 1);
}

// InterpolateBilinear at (x, y); kJac: also the derivatives f_v from (x_v, y_v)
template <bool kJac>
__device__ __forceinline__ void TsdfBilinear(const TsdfCorners& c, float q11, float q12,
                                             float q21, float q22, double x, const double* xv,
                                             double y, const double* yv, double* f,
                                             double* fv) {
  const double c12 = static_cast<double>(q12 - q11), c22 = static_cast<double>(q22 - q21);
  if (!kJac) {
    const double nx = (x - static_cast<double>(c.x1)) / static_cast<double>(c.dx);
    const double ny = (y - static_cast<double>(c.y1)) / static_cast<double>(c.dy);
    const double q1 = c12 * ny + static_cast<double>(q11);
    const double q2 = c22 * ny + static_cast<double>(q21);
    *f = (q2 - q1) * nx + q1;
    return;
  }
  const double inx = 1.0 / static_cast<double>(c.dx), iny = 1.0 / static_cast<double>(c.dy);
  const double nx = (x - static_cast<double>(c.x1)) * inx;
  const double ny = (y - static_cast<double>(c.y1)) * iny;
  const double q1 = c12 * ny + static_cast<double>(q11);
  const double q2 = c22 * ny + static_cast<double>(q21);
  const double d = q2 - q1;
  *f = d * nx + q1;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double nxv = xv[k] * inx, nyv = yv[k] * iny;
    const double q1v = c12 * nyv, q2v = c22 * nyv;
    fv[k] = (d * nxv + (q2v - q1v) * nx) + q1v;
  }
}

// Interpolated weight (and, kCost, correspondence cost) of one point at pose x
template <bool kJac, bool kCost>
__device__ __forceinline__ void TsdfPoint(const RefJobDev& J, const double* x, double cs,
                                          double sn, double px, double py, double* w,
                                          double* wv, double* cost, double* costv) {
  const double wx = (cs * px + (-sn) * py) + x[0] * 1.0;
  const double wy = (sn * px + cs * py) + x[1] * 1.0;
  const double dwx[3] = {1.0, 0.0, (-sn) * px + (-cs) * py};
  const double dwy[3] = {0.0, 1.0, cs * px + (-sn) * py};
  TsdfCorners c;
  TsdfCornersAt(J, wx, wy, &c);
  TsdfBilinear<kJac>(c, c.w11, c.w12, c.w21, c.w22, wx, dwx, wy, dwy, w, wv);
  if (!kCost) return;
  if (c.w11 == 0.f || c.w12 == 0.f || c.w21 == 0.f || c.w22 == 0.f) {
    *cost = static_cast<double>(J.truncation);   // GetMaxCorrespondenceCost(), no derivative
    if (kJac) costv[0] = costv[1] = costv[2] = 0.;
    return;
  }
  TsdfBilinear<kJac>(c, TsdfCost(J, c.ix, c.iy), TsdfCost(J, c.ix - 1, c.iy),
                     TsdfCost(J, c.ix, c.iy - 1), TsdfCost(J, c.ix - 1, c.iy - 1), wx, dwx, wy,
                     dwy, cost, costv);
}

// One TSDF residual (and Jacobian row) given W (and dW).  The functor's
// T(n) * scaling * cost * w, then /= W.
template <bool kJac>
__device__ __forceinline__ void TsdfResidual(double ns, double W, const double* Wv, double w,
                                             const double* wv, double cost,
                                             const double* costv, double* res, double* jrow) {
  const double a = ns * cost;
  if (!kJac) {
    *res = (a * w) / W;
    return;
  }
  const double inv = 1.0 / W;
  const double r = a * w;
  *res = r * inv;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double rv = a * wv[k] + (ns * costv[k]) * w;
    jrow[k] = (rv - *res * Wv[k]) * inv;
  }
}

enum { kGridProbability = 0, kGridTsdf = 1 };

// cost, gradient and normal matrix of all three residual blocks at x (block-wide; the
// result lands in s_tot: {cost, g[3], h[6]}).  false (block-uniform) where the cost function
// returns false: a TSDF scan that sees no weight (summed_weight == 0).
template <int kGrid, bool kJac>
__device__ __forceinline__ bool EvaluateAt(const RefJobDev& J, const RefOpts& P,
                                           const float* __restrict__ xyz, const double* x,
                                           double (*s_part)[10], double* s_tot) {
  const double scaling = P.occupied_space_weight / sqrt(static_cast<double>(J.n));
  double sn, cs;
  sincos(x[2], &sn, &cs);
  double acc[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) acc[k] = 0.;
  double W = 0., Wv[3] = {0., 0., 0.};
  if (kGrid == kGridTsdf) {
    // pass 1: summed_weight and its derivatives
    for (int i = threadIdx.x; i < J.n; i += kRefThreads) {
      const double px = static_cast<double>(xyz[3 * static_cast<size_t>(i)]);
      const double py = static_cast<double>(xyz[3 * static_cast<size_t>(i) + 1]);
      double w, wv[3];
      TsdfPoint<kJac, false>(J, x, cs, sn, px, py, &w, wv, nullptr, nullptr);
      acc[0] += w;
      if (kJac) {
        acc[1] += wv[0];
        acc[2] += wv[1];
        acc[3] += wv[2];
      }
    }
    BlockSum<kJac ? 4 : 1>(acc, s_part, s_tot);
    W = s_tot[0];
    if (kJac) {
      Wv[0] = s_tot[1];
      Wv[1] = s_tot[2];
      Wv[2] = s_tot[3];
    }
    if (W == 0.) {   // the weights are >= 0: W == 0 whatever the order of the sum
      __syncthreads();   // every thread has read s_tot before the caller reuses it
      return false;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[k] = 0.;
  }
  const double ns = static_cast<double>(J.n) * scaling;
  for (int i = threadIdx.x; i < J.n; i += kRefThreads) {
    const double px = static_cast<double>(xyz[3 * static_cast<size_t>(i)]);
    const double py = static_cast<double>(xyz[3 * static_cast<size_t>(i) + 1]);
    double res, jr[3];
    if (kGrid == kGridTsdf) {
      double w, wv[3], cost, costv[3];
      TsdfPoint<kJac, true>(J, x, cs, sn, px, py, &w, wv, &cost, costv);
      TsdfResidual<kJac>(ns, W, Wv, w, wv, cost, costv, &res, jr);
    } else {
      PointResidual<kJac>(J, P, scaling, x, cs, sn, px, py, &res, jr);
    }
    acc[0] += res * res;
    if (kJac) {
      acc[1] += jr[0] * res;
      acc[2] += jr[1] * res;
      acc[3] += jr[2] * res;
      acc[4] += jr[0] * jr[0];
      acc[5] += jr[0] * jr[1];
      acc[6] += jr[0] * jr[2];
      acc[7] += jr[1] * jr[1];
      acc[8] += jr[1] * jr[2];
      acc[9] += jr[2] * jr[2];
    }
  }
  BlockSum<kJac ? 10 : 1>(acc, s_part, s_tot);
  if (threadIdx.x == 0) {
    // translation / rotation priors (the rotation prior is on the INITIAL angle,
    // ceres_scan_matcher_2d.cc:94-97)
    const double wt = P.translation_weight, wr = P.rotation_weight;
    const double r0 = wt * (x[0] - J.target[0]), r1 = wt * (x[1] - J.target[1]);
    const double r2 = wr * (x[2] - J.init[2]);
    double sq = s_tot[0];
    sq += r0 * r0;
    sq += r1 * r1;
    sq += r2 * r2;
    s_tot[0] = 0.5 * sq;
    if (kJac) {
      s_tot[1] += wt * r0;
      s_tot[2] += wt * r1;
      s_tot[3] += wr * r2;
      s_tot[4] += wt * wt;
      s_tot[7] += wt * wt;
      s_tot[9] += wr * wr;
    }
  }
  __syncthreads();
  return true;
}

// The 2D match for the minimiser: {x, y, theta} with x (+) delta = x + delta.
template <int kGrid>
struct Match2D {
  static constexpr int kAmbient = 3, kN = 3;
  const RefJobDev& J;
  const RefOpts& P;
  const float* __restrict__ xyz;
  double (*s_part)[10];

  template <bool kJac>
  __device__ __forceinline__ bool Evaluate(const double* x, double* s_tot) const {
    return EvaluateAt<kGrid, kJac>(J, P, xyz, x, s_part, s_tot);
  }
  __device__ __forceinline__ static void Plus(const double* x, const double* delta,
                                              double* out) {
#pragma unroll
    for (int k = 0; k < 3; ++k) out[k] = x[k] + delta[k];
  }
  __device__ __forceinline__ static double GradientMaxNorm(const double*, const double* g) {
    return fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
  }
};

// One CTA per match; the grid type of the job's handle selects the cost function
// (block-uniform branch), so a batch may mix ProbabilityGrid and TSDF2D jobs.
__global__ void __launch_bounds__(kRefThreads)
k_ceres_match2d(const RefJobDev* __restrict__ jobs, RefOpts P, const float* __restrict__ cloud,
                RefResultDev* __restrict__ results) {
  __shared__ double s_part[kRefWarps][10];
  __shared__ double s_tot[10];
  __shared__ double s_pose[3];
  __shared__ int s_cmd;
  const RefJobDev J = jobs[blockIdx.x];
  const float* __restrict__ xyz = cloud + J.xyz_off;
  TrustRegionState<3, 3> S;   // thread 0's registers
  if (J.wcells == nullptr)
    TrustRegionMinimize(Match2D<kGridProbability>{J, P, xyz, s_part}, J.init,
                        P.max_num_iterations, P.use_nonmonotonic_steps, S, s_tot, s_pose, s_cmd,
                        results + blockIdx.x);
  else
    TrustRegionMinimize(Match2D<kGridTsdf>{J, P, xyz, s_part}, J.init, P.max_num_iterations,
                        P.use_nonmonotonic_steps, S, s_tot, s_pose, s_cmd, results + blockIdx.x);
}

// Test hook: residuals (and Jacobian rows) of one job at one pose, one thread per residual.
__global__ void k_ceres_evaluate2d(RefJobDev J, RefOpts P, const float* __restrict__ xyz,
                                   double px, double py, double pt, double cs, double sn,
                                   int with_jacobian, double* __restrict__ residuals,
                                   double* __restrict__ jacobian) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double x[3] = {px, py, pt};
  const double scaling = P.occupied_space_weight / sqrt(static_cast<double>(J.n));
  if (i < J.n) {
    const double qx = static_cast<double>(xyz[3 * static_cast<size_t>(i)]);
    const double qy = static_cast<double>(xyz[3 * static_cast<size_t>(i) + 1]);
    double res, jr[3] = {0., 0., 0.};
    if (with_jacobian) {
      PointResidual<true>(J, P, scaling, x, cs, sn, qx, qy, &res, jr);
      jacobian[3 * static_cast<size_t>(i)] = jr[0];
      jacobian[3 * static_cast<size_t>(i) + 1] = jr[1];
      jacobian[3 * static_cast<size_t>(i) + 2] = jr[2];
    } else {
      PointResidual<false>(J, P, scaling, x, cs, sn, qx, qy, &res, jr);
    }
    residuals[i] = res;
  } else if (i == J.n) {
    const size_t n = J.n;
    residuals[n] = P.translation_weight * (x[0] - J.target[0]);
    residuals[n + 1] = P.translation_weight * (x[1] - J.target[1]);
    residuals[n + 2] = P.rotation_weight * (x[2] - J.init[2]);
    if (with_jacobian) {
      for (int k = 0; k < 9; ++k) jacobian[3 * n + k] = 0.;
      jacobian[3 * n + 0] = P.translation_weight;
      jacobian[3 * (n + 1) + 1] = P.translation_weight;
      jacobian[3 * (n + 2) + 2] = P.rotation_weight;
    }
  }
}

// Test hook, TSDF2D: the residuals need W first, so one CTA reduces it (block-tree order, as
// the solver does) and then writes every residual; *valid = 0 where summed_weight == 0.
template <bool kJac>
__device__ __forceinline__ void EvaluateTsdf(const RefJobDev& J, const RefOpts& P,
                                             const float* __restrict__ xyz, const double* x,
                                             double cs, double sn, double* __restrict__ residuals,
                                             double* __restrict__ jacobian, int* valid) {
  __shared__ double s_part[kRefWarps][10];
  __shared__ double s_tot[10];
  double acc[4] = {0., 0., 0., 0.};
  for (int i = threadIdx.x; i < J.n; i += kRefThreads) {
    double w, wv[3];
    TsdfPoint<kJac, false>(J, x, cs, sn, static_cast<double>(xyz[3 * static_cast<size_t>(i)]),
                           static_cast<double>(xyz[3 * static_cast<size_t>(i) + 1]), &w, wv,
                           nullptr, nullptr);
    acc[0] += w;
    if (kJac) {
      acc[1] += wv[0];
      acc[2] += wv[1];
      acc[3] += wv[2];
    }
  }
  BlockSum<kJac ? 4 : 1>(acc, s_part, s_tot);
  const double W = s_tot[0];
  const double Wv[3] = {kJac ? s_tot[1] : 0., kJac ? s_tot[2] : 0., kJac ? s_tot[3] : 0.};
  if (threadIdx.x == 0) *valid = W == 0. ? 0 : 1;
  if (W == 0.) return;
  const double ns = static_cast<double>(J.n) * (P.occupied_space_weight / sqrt(static_cast<double>(J.n)));
  for (int i = threadIdx.x; i < J.n; i += kRefThreads) {
    double w, wv[3], cost, costv[3], res, jr[3];
    TsdfPoint<kJac, true>(J, x, cs, sn, static_cast<double>(xyz[3 * static_cast<size_t>(i)]),
                          static_cast<double>(xyz[3 * static_cast<size_t>(i) + 1]), &w, wv, &cost,
                          costv);
    TsdfResidual<kJac>(ns, W, Wv, w, wv, cost, costv, &res, jr);
    residuals[i] = res;
    if (kJac) {
      jacobian[3 * static_cast<size_t>(i)] = jr[0];
      jacobian[3 * static_cast<size_t>(i) + 1] = jr[1];
      jacobian[3 * static_cast<size_t>(i) + 2] = jr[2];
    }
  }
}

__global__ void __launch_bounds__(kRefThreads)
k_ceres_evaluate2d_tsdf(RefJobDev J, RefOpts P, const float* __restrict__ xyz, double px,
                        double py, double pt, double cs, double sn, int with_jacobian,
                        double* __restrict__ residuals, double* __restrict__ jacobian,
                        int* __restrict__ valid) {
  const double x[3] = {px, py, pt};
  if (with_jacobian)
    EvaluateTsdf<true>(J, P, xyz, x, cs, sn, residuals, jacobian, valid);
  else
    EvaluateTsdf<false>(J, P, xyz, x, cs, sn, residuals, jacobian, valid);
  if (threadIdx.x == 0) {   // the two prior blocks, as k_ceres_evaluate2d writes them
    const size_t n = J.n;
    residuals[n] = P.translation_weight * (x[0] - J.target[0]);
    residuals[n + 1] = P.translation_weight * (x[1] - J.target[1]);
    residuals[n + 2] = P.rotation_weight * (x[2] - J.init[2]);
    if (with_jacobian) {
      for (int k = 0; k < 9; ++k) jacobian[3 * n + k] = 0.;
      jacobian[3 * n + 0] = P.translation_weight;
      jacobian[3 * (n + 1) + 1] = P.translation_weight;
      jacobian[3 * (n + 2) + 2] = P.rotation_weight;
    }
  }
}

}  // namespace csm

#ifndef CSM_REFINE_DEVICE_ONLY
using namespace csm;

namespace {

csm_status FillOpts(const csm_ceres_options2d* o, RefOpts* P) {
  CSM_REQUIRE(o != nullptr, "null options");
  // CHECK_GT(..., 0.) in ceres_scan_matcher_2d.cc:72,87,92
  CSM_REQUIRE(o->occupied_space_weight > 0. && o->translation_weight > 0. &&
              o->rotation_weight > 0., "weights must be positive");
  CSM_REQUIRE(o->max_num_iterations > 0, "max_num_iterations");   // ceres_solver_options.cc:31
  P->occupied_space_weight = o->occupied_space_weight;
  P->translation_weight = o->translation_weight;
  P->rotation_weight = o->rotation_weight;
  P->use_nonmonotonic_steps = o->use_nonmonotonic_steps != 0;
  P->max_num_iterations = o->max_num_iterations;
  // probability_values.h:64-67 and value_conversion_tables.cc:29-37 evaluated in float
  const float kMinProbability = 0.1f;
  const float kMaxProbability = 1.f - kMinProbability;
  const float kMinCost = 1.f - kMaxProbability;
  const float kMaxCost = 1.f - kMinProbability;
  P->k_scale = (kMaxCost - kMinCost) / 32766.f;
  P->cost_bias = kMinCost - P->k_scale;
  P->max_cost = kMaxCost;
  return CSM_OK;
}

void FillJob(const csm_rt_grid2d* grid, int n, long long xyz_off, const double target[2],
             const double init[3], RefJobDev* j) {
  std::memset(j, 0, sizeof(*j));
  j->cells = grid->g.cells;
  j->nx = grid->g.nx;
  j->ny = grid->g.ny;
  j->pitch = grid->g.pitch;
  j->n = n;
  j->xyz_off = xyz_off;
  j->resolution = grid->g.resolution;
  j->max_x = grid->g.max_x;
  j->max_y = grid->g.max_y;
  j->target[0] = target[0];
  j->target[1] = target[1];
  j->init[0] = init[0];
  j->init[1] = init[1];
  j->init[2] = init[2];
  if (grid->d_wcells != nullptr) {   // TSDF2D: TSDFMatchCostFunction2D
    const TsdfConversion c = MakeTsdfConversion(grid->truncation, grid->max_weight);
    j->wcells = grid->g.wcells;
    j->tsd_scale = c.tsd_scale;
    j->tsd_bias = c.tsd_bias;
    j->w_scale = c.w_scale;
    j->w_bias = c.w_bias;
    j->truncation = grid->truncation;
  }
}

}  // namespace

extern "C" {

csm_status csm_ceres_match2d_batch(const csm_ceres_job2d* jobs, int32_t num_jobs,
                                   const csm_ceres_options2d* options,
                                   csm_ceres_result2d* results, csm_stats* stats) {
  CSM_REQUIRE(jobs && results, "null pointer");
  CSM_REQUIRE(num_jobs >= 1, "empty batch");
  RefOpts P;
  CSM_TRY(FillOpts(options, &P));
  const int device = jobs[0].grid ? jobs[0].grid->ctx->device : -1;
  long long floats = 0;
  for (int j = 0; j < num_jobs; ++j) {
    CSM_REQUIRE(jobs[j].grid != nullptr && jobs[j].xyz != nullptr, "null pointer");
    CSM_REQUIRE(jobs[j].num_points >= 1, "empty point cloud");
    CSM_REQUIRE(jobs[j].grid->ctx->device == device, "grids of one batch share a device");
    floats += 3LL * jobs[j].num_points;
  }
  CSM_REQUIRE(floats < (1LL << 31), "batch too large");
  LaneGuard guard;
  CSM_TRY(AcquireLane(device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t off_jobs = (static_cast<size_t>(floats) * 4 + 255) / 256 * 256;
  const size_t up_bytes = off_jobs + sizeof(RefJobDev) * num_jobs;
  PinnedBuf& up = ctx->P("ref_upload");
  DevBuf& d_up = ctx->D("ref_upload");
  DevBuf& d_out = ctx->D("ref_results");
  PinnedBuf& rb = ctx->P("ref_readback");
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(d_up.Reserve(up_bytes));
  CSM_TRY(d_out.Reserve(sizeof(RefResultDev) * num_jobs));
  CSM_TRY(rb.Reserve(sizeof(RefResultDev) * num_jobs));
  char* h = up.as<char>();
  RefJobDev* hj = reinterpret_cast<RefJobDev*>(h + off_jobs);
  long long off = 0;
  for (int j = 0; j < num_jobs; ++j) {
    std::memcpy(reinterpret_cast<float*>(h) + off, jobs[j].xyz,
                sizeof(float) * 3 * static_cast<size_t>(jobs[j].num_points));
    FillJob(jobs[j].grid, jobs[j].num_points, off, jobs[j].target_translation,
            jobs[j].initial_pose, &hj[j]);
    off += 3LL * jobs[j].num_points;
  }
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_CUDA(cudaMemcpyAsync(d_up.p, h, up_bytes, cudaMemcpyHostToDevice, s));
  ProfBegin(ctx);
  k_ceres_match2d<<<num_jobs, kRefThreads, 0, s>>>(
      reinterpret_cast<const RefJobDev*>(d_up.as<char>() + off_jobs), P, d_up.as<float>(),
      d_out.as<RefResultDev>());
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, "k_ceres_match2d", static_cast<double>(num_jobs));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(rb.p, d_out.p, sizeof(RefResultDev) * num_jobs,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  const RefResultDev* r = rb.as<RefResultDev>();
  for (int j = 0; j < num_jobs; ++j) {
    csm_ceres_result2d& o = results[j];
    std::memset(&o, 0, sizeof(o));
    std::memcpy(o.pose_estimate, r[j].pose, sizeof(double) * 3);
    o.initial_cost = r[j].initial_cost;
    o.final_cost = r[j].final_cost;
    o.iterations = r[j].iterations;
    o.num_successful_steps = r[j].num_successful_steps;
    o.termination = r[j].termination;
  }
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    stats->device_ms = ms;
    stats->host_syncs = 1;
  }
  return CSM_OK;
}

csm_status csm_ceres_evaluate2d(const csm_rt_grid2d* grid, const float* xyz, int32_t num_points,
                                const csm_ceres_options2d* options,
                                const double target_translation[2], double target_angle,
                                const double pose[3], double* residuals, double* jacobian) {
  CSM_REQUIRE(grid && xyz && target_translation && pose && residuals, "null pointer");
  CSM_REQUIRE(num_points >= 1, "empty point cloud");
  CSM_REQUIRE(grid->d_wcells == nullptr, "the grid must be a ProbabilityGrid");
  RefOpts P;
  CSM_TRY(FillOpts(options, &P));
  LaneGuard guard;
  CSM_TRY(AcquireLane(grid->ctx->device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t n = static_cast<size_t>(num_points);
  DevBuf& d_xyz = ctx->D("ref_eval_xyz");
  DevBuf& d_res = ctx->D("ref_eval_res");
  DevBuf& d_jac = ctx->D("ref_eval_jac");
  CSM_TRY(d_xyz.Reserve(sizeof(float) * 3 * n));
  CSM_TRY(d_res.Reserve(sizeof(double) * (n + 3)));
  CSM_TRY(d_jac.Reserve(sizeof(double) * 3 * (n + 3)));
  CSM_CUDA(cudaMemcpyAsync(d_xyz.p, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, s));
  RefJobDev J;
  const double init[3] = {pose[0], pose[1], target_angle};   // init[2] carries the prior's angle
  FillJob(grid, num_points, 0, target_translation, init, &J);
  // the hook takes cos / sin from the host's libm so that its values can be compared bit for
  // bit with the oracle's; the solver kernel evaluates them on the device
  k_ceres_evaluate2d<<<static_cast<int>((n + 1 + 255) / 256), 256, 0, s>>>(
      J, P, d_xyz.as<float>(), pose[0], pose[1], pose[2], std::cos(pose[2]), std::sin(pose[2]),
      jacobian != nullptr, d_res.as<double>(), d_jac.as<double>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(residuals, d_res.p, sizeof(double) * (n + 3), cudaMemcpyDeviceToHost, s));
  if (jacobian)
    CSM_CUDA(cudaMemcpyAsync(jacobian, d_jac.p, sizeof(double) * 3 * (n + 3),
                             cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

csm_status csm_ceres_evaluate2d_checked(const csm_rt_grid2d* grid, const float* xyz,
                                        int32_t num_points, const csm_ceres_options2d* options,
                                        const double target_translation[2], double target_angle,
                                        const double pose[3], double* residuals,
                                        double* jacobian, int32_t* valid) {
  CSM_REQUIRE(grid && xyz && target_translation && pose && residuals && valid, "null pointer");
  CSM_REQUIRE(num_points >= 1, "empty point cloud");
  if (grid->d_wcells == nullptr) {   // a ProbabilityGrid's cost function never fails
    CSM_TRY(csm_ceres_evaluate2d(grid, xyz, num_points, options, target_translation,
                                 target_angle, pose, residuals, jacobian));
    *valid = 1;
    return CSM_OK;
  }
  RefOpts P;
  CSM_TRY(FillOpts(options, &P));
  LaneGuard guard;
  CSM_TRY(AcquireLane(grid->ctx->device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t n = static_cast<size_t>(num_points);
  DevBuf& d_xyz = ctx->D("ref_eval_xyz");
  DevBuf& d_res = ctx->D("ref_eval_res");
  DevBuf& d_jac = ctx->D("ref_eval_jac");
  DevBuf& d_valid = ctx->D("ref_eval_valid");
  CSM_TRY(d_xyz.Reserve(sizeof(float) * 3 * n));
  CSM_TRY(d_res.Reserve(sizeof(double) * (n + 3)));
  CSM_TRY(d_jac.Reserve(sizeof(double) * 3 * (n + 3)));
  CSM_TRY(d_valid.Reserve(sizeof(int)));
  CSM_CUDA(cudaMemcpyAsync(d_xyz.p, xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, s));
  CSM_CUDA(cudaMemsetAsync(d_res.p, 0, sizeof(double) * (n + 3), s));
  CSM_CUDA(cudaMemsetAsync(d_jac.p, 0, sizeof(double) * 3 * (n + 3), s));
  RefJobDev J;
  const double init[3] = {pose[0], pose[1], target_angle};   // init[2] carries the prior's angle
  FillJob(grid, num_points, 0, target_translation, init, &J);
  // host cos / sin, as in csm_ceres_evaluate2d
  k_ceres_evaluate2d_tsdf<<<1, kRefThreads, 0, s>>>(
      J, P, d_xyz.as<float>(), pose[0], pose[1], pose[2], std::cos(pose[2]), std::sin(pose[2]),
      jacobian != nullptr, d_res.as<double>(), d_jac.as<double>(), d_valid.as<int>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(residuals, d_res.p, sizeof(double) * (n + 3), cudaMemcpyDeviceToHost, s));
  if (jacobian)
    CSM_CUDA(cudaMemcpyAsync(jacobian, d_jac.p, sizeof(double) * 3 * (n + 3),
                             cudaMemcpyDeviceToHost, s));
  int v = 0;
  CSM_CUDA(cudaMemcpyAsync(&v, d_valid.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  *valid = v;
  return CSM_OK;
}

}  // extern "C"
#endif  // CSM_REFINE_DEVICE_ONLY
