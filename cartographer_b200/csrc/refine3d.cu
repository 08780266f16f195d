// Post-match refinement in 3D: CeresScanMatcher3D::Match
// (mapping/internal/3d/scan_matching/ceres_scan_matcher_3d.cc:95-157) as ConstraintBuilder3D
// calls it on every found match (constraint_builder_3d.cc:265-275): occupied-space blocks for
// the (high-resolution cloud, high-resolution grid) and (low-resolution cloud, low-resolution
// grid) pairs, a translation prior and a rotation prior, over {translation[3], rotation[4]}
// with Ceres' QuaternionParameterization (only_optimize_yaw = false).  A cloud may also carry
// an IntensityHybridGrid, as LocalTrajectoryBuilder3D passes one with use_intensities
// (ceres_scan_matcher_3d.cc:123-139): then an IntensityCostFunction3D block
// (intensity_cost_function_3d.h:67-85) under ceres::HuberLoss(huber_scale) follows that
// cloud's occupied-space block.  The constraint builder passes no intensity grid.
//
// As in refine2d.cu, Ceres is not linked: one CTA per match runs the whole trust-region loop
// on the device.  Per point: Eigen's quaternion * vector + translation and its derivative by
// the 7 ambient parameters, the 8 voxel probabilities around the point, the smoothstep
// interpolation of interpolated_grid.h:49-96 on dual numbers over (x, y, z)
// (occupied_space_cost_function_3d.h:68-78), then the residual row in the 6-dimensional
// tangent space (ambient row times the parameterisation's 4 x 3 plus-Jacobian).  The block
// reduces cost, J^T r and the upper triangle of J^T J (28 doubles); thread 0 runs the
// trust-region minimiser of trust_region.cuh (the one refine2d.cu runs), its state in shared
// memory, with 6 parameters, x (+) delta = {t + dt, exp(dq) * q} and the gradient tolerance
// measured as |x - (x (+) -g)|_inf.  Doubles, no FMA contraction (-fmad=false).
//
// The Huber loss acts on a whole intensity block, so its squared norm s_b must be known
// before the block's rows can enter g and H: each intensity block is reduced on its own
// (one more BlockSum into s_blk) and thread 0 adds rho(s_b) to the cost, rho'(s_b) J^T r to g
// and rho'(s_b) J^T J to H.  That is Ceres' Corrector (ceres/corrector.cc) in its alpha = 0
// branch, the only one HuberLoss reaches (rho'' <= 0), restated from Ceres' published
// algorithm (ceres/loss_function.cc, HuberLoss::Evaluate).  A job with no intensity grid runs
// exactly the occupied-space path.
#include <algorithm>
#include <cmath>

// see refine2d.cu: tests/emulation includes the device code below into a CPU harness
#ifndef CSM_REFINE_DEVICE_ONLY
#include "grid3d.cuh"
#endif
#include "trust_region.cuh"

namespace csm {

constexpr int kRef3N = 6;                              // tangent-space parameters
constexpr int kRef3H = kRef3N * (kRef3N + 1) / 2;      // upper triangle of J^T J
constexpr int kRef3Acc = 1 + kRef3N + kRef3H;          // 28
constexpr int kRef3MaxClouds = 2;

struct Ref3Cloud {
  const uint16_t* vol;     // dense box of HybridGrid values (csm_grid3d)
  int lo[3], n[3];
  float resolution, k_scale, bias, min_probability;
  int npts;
  long long xyz_off;       // first float of the cloud in the upload buffer
};

// A cloud's IntensityCostFunction3D block (ivol == nullptr where the cloud has none).  Kept
// apart from Ref3JobDev so that a batch without intensity blocks stages and copies exactly
// the occupied-space record.
struct Ref3IntensityCloud {
  const float* ivol;       // dense box of GetIntensity values (csm_intensity_grid3d)
  int ilo[3], in[3];
  float iresolution, intensity_threshold;
  double intensity_weight, huber_scale;   // intensity_cost_function_options_b
  long long intensity_off; // first float of the cloud's intensities in the upload buffer
};

struct Ref3IntensityJobDev {
  Ref3IntensityCloud c[kRef3MaxClouds];
};

struct Ref3JobDev {
  Ref3Cloud c[kRef3MaxClouds];
  int num_clouds, pad;
  double target_t[3];
  double init[7];          // {t xyz, q wxyz}; init + 3 is also the rotation prior's target
};

struct Ref3Opts {
  double occupied_space_weight[kRef3MaxClouds];
  double translation_weight, rotation_weight;
  int use_nonmonotonic_steps, max_num_iterations;
};

using Ref3ResultDev = ResultDev<7>;   // trust_region.cuh

// ---- dual numbers over (x, y, z) with ceres/jet.h's arithmetic ------------------------
struct D3 {
  double a, v0, v1, v2;
};
__device__ __forceinline__ D3 Add(const D3& f, const D3& g) {
  return D3{f.a + g.a, f.v0 + g.v0, f.v1 + g.v1, f.v2 + g.v2};
}
__device__ __forceinline__ D3 Sub(const D3& f, const D3& g) {
  return D3{f.a - g.a, f.v0 - g.v0, f.v1 - g.v1, f.v2 - g.v2};
}
__device__ __forceinline__ D3 AddS(const D3& f, double s) { return D3{f.a + s, f.v0, f.v1, f.v2}; }
__device__ __forceinline__ D3 Mul(const D3& f, const D3& g) {
  return D3{f.a * g.a, f.a * g.v0 + f.v0 * g.a, f.a * g.v1 + f.v1 * g.a, f.a * g.v2 + f.v2 * g.a};
}
__device__ __forceinline__ D3 MulS(const D3& f, double s) {
  return D3{f.a * s, f.v0 * s, f.v1 * s, f.v2 * s};
}

// HybridGrid::GetCellIndex (mapping/3d/hybrid_grid.h:428-433) of a float coordinate
__device__ __forceinline__ int CellOf(float p, float resolution) {
  return static_cast<int>(lroundf(__fdiv_rn(p, resolution)));
}

// HybridGrid::GetProbability (hybrid_grid.h:521-523) as a double
__device__ __forceinline__ double Probability(const Ref3Cloud& G, int x, int y, int z) {
  const int ix = x - G.lo[0], iy = y - G.lo[1], iz = z - G.lo[2];
  int value = 0;
  if (static_cast<unsigned>(ix) < static_cast<unsigned>(G.n[0]) &&
      static_cast<unsigned>(iy) < static_cast<unsigned>(G.n[1]) &&
      static_cast<unsigned>(iz) < static_cast<unsigned>(G.n[2]))
    value = __ldg(G.vol + (static_cast<size_t>(iz) * G.n[1] + iy) * G.n[0] + ix) & 0x7fff;
  const float prob = value == 0 ? G.min_probability
                                : __fadd_rn(__fmul_rn(__int2float_rn(value), G.k_scale), G.bias);
  return static_cast<double>(prob);
}

// The value sources of InterpolatedGrid<T>::GetValue (interpolated_grid.h:146-157)
struct ProbabilityValues {   // HybridGrid
  const Ref3Cloud& G;
  __device__ __forceinline__ float resolution() const { return G.resolution; }
  __device__ __forceinline__ double operator()(int x, int y, int z) const {
    return Probability(G, x, y, z);
  }
};
struct IntensityValues {     // IntensityHybridGrid: the box holds GetIntensity, 0 outside it
  const Ref3IntensityCloud& G;
  __device__ __forceinline__ float resolution() const { return G.iresolution; }
  __device__ __forceinline__ double operator()(int x, int y, int z) const {
    const int ix = x - G.ilo[0], iy = y - G.ilo[1], iz = z - G.ilo[2];
    float value = 0.f;
    if (static_cast<unsigned>(ix) < static_cast<unsigned>(G.in[0]) &&
        static_cast<unsigned>(iy) < static_cast<unsigned>(G.in[1]) &&
        static_cast<unsigned>(iz) < static_cast<unsigned>(G.in[2]))
      value = __ldg(G.ivol + (static_cast<size_t>(iz) * G.in[1] + iy) * G.in[0] + ix);
    return static_cast<double>(value);
  }
};

// InterpolatedGrid<T>::GetInterpolatedValue (interpolated_grid.h:49-96)
template <bool kDual, class Values>
__device__ __forceinline__ D3 Interpolate(const Values& value, double x, double y, double z) {
  // CenterOfLowerVoxel (:115-135)
  const float res = value.resolution();
  float cx = __fmul_rn(__int2float_rn(CellOf(static_cast<float>(x), res)), res);
  float cy = __fmul_rn(__int2float_rn(CellOf(static_cast<float>(y), res)), res);
  float cz = __fmul_rn(__int2float_rn(CellOf(static_cast<float>(z), res)), res);
  if (static_cast<double>(cx) > x) cx = __fsub_rn(cx, res);
  if (static_cast<double>(cy) > y) cy = __fsub_rn(cy, res);
  if (static_cast<double>(cz) > z) cz = __fsub_rn(cz, res);
  const double x1 = cx, y1 = cy, z1 = cz;
  const double x2 = __fadd_rn(cx, res), y2 = __fadd_rn(cy, res), z2 = __fadd_rn(cz, res);
  const int i = CellOf(cx, res), j = CellOf(cy, res), k = CellOf(cz, res);
  const double q111 = value(i, j, k), q112 = value(i, j, k + 1);
  const double q121 = value(i, j + 1, k), q122 = value(i, j + 1, k + 1);
  const double q211 = value(i + 1, j, k), q212 = value(i + 1, j, k + 1);
  const double q221 = value(i + 1, j + 1, k), q222 = value(i + 1, j + 1, k + 1);
  D3 nx, ny, nz;
  if (kDual) {
    const double ix = 1.0 / (x2 - x1), iy = 1.0 / (y2 - y1), iz = 1.0 / (z2 - z1);
    nx = D3{(x - x1) * ix, 1.0 * ix, 0.0 * ix, 0.0 * ix};
    ny = D3{(y - y1) * iy, 0.0 * iy, 1.0 * iy, 0.0 * iy};
    nz = D3{(z - z1) * iz, 0.0 * iz, 0.0 * iz, 1.0 * iz};
  } else {
    nx = D3{(x - x1) / (x2 - x1), 0., 0., 0.};
    ny = D3{(y - y1) / (y2 - y1), 0., 0., 0.};
    nz = D3{(z - z1) / (z2 - z1), 0., 0., 0.};
  }
  const D3 nxx = Mul(nx, nx), nxxx = Mul(nx, nxx);
  const D3 nyy = Mul(ny, ny), nyyy = Mul(ny, nyy);
  const D3 nzz = Mul(nz, nz), nzzz = Mul(nz, nzz);
  // (qa - qb) * n^3 * 2. + (qb - qa) * n^2 * 3. + qa, scalars first
  const D3 q11 = AddS(Add(MulS(MulS(nzzz, q111 - q112), 2.), MulS(MulS(nzz, q112 - q111), 3.)), q111);
  const D3 q12 = AddS(Add(MulS(MulS(nzzz, q121 - q122), 2.), MulS(MulS(nzz, q122 - q121), 3.)), q121);
  const D3 q21 = AddS(Add(MulS(MulS(nzzz, q211 - q212), 2.), MulS(MulS(nzz, q212 - q211), 3.)), q211);
  const D3 q22 = AddS(Add(MulS(MulS(nzzz, q221 - q222), 2.), MulS(MulS(nzz, q222 - q221), 3.)), q221);
  const D3 q1 = Add(Add(MulS(Mul(Sub(q11, q12), nyyy), 2.), MulS(Mul(Sub(q12, q11), nyy), 3.)), q11);
  const D3 q2 = Add(Add(MulS(Mul(Sub(q21, q22), nyyy), 2.), MulS(Mul(Sub(q22, q21), nyy), 3.)), q21);
  return Add(Add(MulS(Mul(Sub(q1, q2), nxxx), 2.), MulS(Mul(Sub(q2, q1), nxx), 3.)), q1);
}

__device__ __forceinline__ void Cross3(const double* a, const double* b, double* out) {
  out[0] = a[1] * b[2] - a[2] * b[1];
  out[1] = a[2] * b[0] - a[0] * b[2];
  out[2] = a[0] * b[1] - a[1] * b[0];
}

// ceres::QuaternionParameterization::ComputeJacobian (4 x 3, row-major)
__device__ __forceinline__ void PlusJacobian(const double* q, double* jac) {
  jac[0] = -q[1]; jac[1] = -q[2]; jac[2] = -q[3];
  jac[3] = q[0];  jac[4] = q[3];  jac[5] = -q[2];
  jac[6] = -q[3]; jac[7] = q[0];  jac[8] = q[1];
  jac[9] = q[2];  jac[10] = -q[1]; jac[11] = q[0];
}

__device__ __forceinline__ void ToLocal(const double* ambient, const double* pj, double* row) {
  row[0] = ambient[0];
  row[1] = ambient[1];
  row[2] = ambient[2];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    row[3 + k] = ambient[3] * pj[k] + ambient[4] * pj[3 + k] + ambient[5] * pj[6 + k] +
                 ambient[6] * pj[9 + k];
}

// x (+) delta (QuaternionParameterization::Plus on the rotation block)
__device__ __forceinline__ void Plus7(const double* x, const double* delta, double* out) {
  for (int k = 0; k < 3; ++k) out[k] = x[k] + delta[k];
  const double* d = delta + 3;
  const double norm_delta = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  if (norm_delta > 0.0) {
    const double sin_delta_by_delta = sin(norm_delta) / norm_delta;
    const double z[4] = {cos(norm_delta), sin_delta_by_delta * d[0], sin_delta_by_delta * d[1],
                         sin_delta_by_delta * d[2]};
    const double* w = x + 3;
    out[3] = z[0] * w[0] - z[1] * w[1] - z[2] * w[2] - z[3] * w[3];
    out[4] = z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2];
    out[5] = z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1];
    out[6] = z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0];
  } else {
    for (int k = 3; k < 7; ++k) out[k] = x[k];
  }
}

// The grid value interpolated at pose * p and (kJac) its derivative by the 7 ambient
// parameters, dp[k] = grad . d world / d param k.
template <bool kJac, class Values>
__device__ __forceinline__ D3 InterpolateAtPoint(const Values& values, const double* pose,
                                                 double px, double py, double pz, double* dp) {
  // Eigen QuaternionBase::_transformVector (q not normalised) + translation
  const double p[3] = {px, py, pz};
  const double w = pose[3];
  const double qv[3] = {pose[4], pose[5], pose[6]};
  double uv[3], c[3], world[3];
  Cross3(qv, p, uv);
  uv[0] += uv[0];
  uv[1] += uv[1];
  uv[2] += uv[2];
  Cross3(qv, uv, c);
#pragma unroll
  for (int k = 0; k < 3; ++k) world[k] = ((p[k] + w * uv[k]) + c[k]) + pose[k];
  const D3 f = Interpolate<kJac>(values, world[0], world[1], world[2]);
  if (!kJac) return f;
  // d world / d t = I
  dp[0] = (f.v0 * 1.0 + f.v1 * 0.0) + f.v2 * 0.0;
  dp[1] = (f.v0 * 0.0 + f.v1 * 1.0) + f.v2 * 0.0;
  dp[2] = (f.v0 * 0.0 + f.v1 * 0.0) + f.v2 * 1.0;
  // d world / d w = uv
  dp[3] = (f.v0 * uv[0] + f.v1 * uv[1]) + f.v2 * uv[2];
#pragma unroll
  for (int k = 0; k < 3; ++k) {   // d world / d qv[k] = w * duv + e_k x uv + qv x duv
    double e[3] = {0., 0., 0.};
    e[k] = 1.0;
    double duv[3], t1[3], t2[3];
    Cross3(e, p, duv);
    duv[0] += duv[0];
    duv[1] += duv[1];
    duv[2] += duv[2];
    Cross3(e, uv, t1);
    Cross3(qv, duv, t2);
    const double d0 = (w * duv[0] + t1[0]) + t2[0];
    const double d1 = (w * duv[1] + t1[1]) + t2[1];
    const double d2 = (w * duv[2] + t1[2]) + t2[2];
    dp[4 + k] = (f.v0 * d0 + f.v1 * d1) + f.v2 * d2;
  }
  return f;
}

// One occupied-space residual and (kJac) its tangent-space Jacobian row.
template <bool kJac>
__device__ __forceinline__ void PointResidual3(const Ref3Cloud& G, double scaling,
                                               const double* pose, const double* pj, double px,
                                               double py, double pz, double* res, double* row) {
  double ambient[7];   // dp, then the ambient row in place
  const D3 f = InterpolateAtPoint<kJac>(ProbabilityValues{G}, pose, px, py, pz, ambient);
  *res = scaling * (1. - f.a);   // occupied_space_cost_function_3d.h:75
  if (!kJac) return;
#pragma unroll
  for (int k = 0; k < 7; ++k) ambient[k] = scaling * (-ambient[k]);
  ToLocal(ambient, pj, row);
}

// One IntensityCostFunction3D residual (intensity_cost_function_3d.h:67-80) and (kJac) its
// tangent-space row; a return brighter than the threshold gives 0 and a zero row.
template <bool kJac>
__device__ __forceinline__ void IntensityResidual3(const Ref3IntensityCloud& G, double scaling,
                                                   float threshold, const double* pose,
                                                   const double* pj, double px, double py,
                                                   double pz, float intensity, double* res,
                                                   double* row) {
  if (intensity > threshold) {
    *res = 0.;
    if (kJac) {
#pragma unroll
      for (int a = 0; a < kRef3N; ++a) row[a] = 0.;
    }
    return;
  }
  double ambient[7];   // dp, then the ambient row in place
  const D3 f = InterpolateAtPoint<kJac>(IntensityValues{G}, pose, px, py, pz, ambient);
  *res = scaling * (f.a - static_cast<double>(intensity));
  if (!kJac) return;
#pragma unroll
  for (int k = 0; k < 7; ++k) ambient[k] = scaling * ambient[k];
  ToLocal(ambient, pj, row);
}

// ceres::HuberLoss(a)::Evaluate at s = the block's squared norm: rho and rho'
__device__ __forceinline__ void HuberRho(double a, double s, double* rho, double* rho1) {
  const double b = a * a;
  if (s > b) {   // outlier region
    const double r = sqrt(s);
    *rho = 2.0 * a * r - b;
    *rho1 = fmax(DBL_MIN, a / r);
  } else {
    *rho = s;
    *rho1 = 1.0;
  }
}

// The 3 + 3 prior residuals and their tangent-space rows (thread 0).
__device__ __forceinline__ void PriorRows(const Ref3JobDev& J, const Ref3Opts& P,
                                          const double* pose, const double* pj, double* res,
                                          double (*rows)[kRef3N]) {
  for (int k = 0; k < 3; ++k) {
    res[k] = P.translation_weight * (pose[k] - J.target_t[k]);
    for (int a = 0; a < kRef3N; ++a) rows[k][a] = 0.;
    rows[k][k] = P.translation_weight;
  }
  const double z[4] = {J.init[3], -J.init[4], -J.init[5], -J.init[6]};
  const double* w = pose + 3;
  const double delta[3] = {z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2],
                           z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1],
                           z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0]};
  const double ddelta[3][4] = {{z[1], z[0], -z[3], z[2]},
                               {z[2], z[3], z[0], -z[1]},
                               {z[3], -z[2], z[1], z[0]}};
  for (int k = 0; k < 3; ++k) {
    res[3 + k] = P.rotation_weight * delta[k];
    double ambient[7] = {0., 0., 0., 0., 0., 0., 0.};
    for (int c = 0; c < 4; ++c) ambient[3 + c] = P.rotation_weight * ddelta[k][c];
    ToLocal(ambient, pj, rows[3 + k]);
  }
}

// Block-wide evaluation at `pose`: s_tot = {cost, g[6], h[21]} (g, h only with kJac).  With
// kIntensity the intensity blocks of I are reduced one by one into s_blk and corrected by
// thread 0.
template <bool kJac, bool kIntensity>
__device__ __forceinline__ void EvaluateAt3(const Ref3JobDev& J, const Ref3IntensityJobDev* I,
                                            const Ref3Opts& P,
                                            const float* __restrict__ cloud, const double* pose,
                                            double (*s_part)[kRef3Acc], double* s_tot,
                                            double* s_blk) {
  double pj[12];
  PlusJacobian(pose + 3, pj);
  double acc[kRef3Acc];
#pragma unroll
  for (int k = 0; k < kRef3Acc; ++k) acc[k] = 0.;
  for (int b = 0; b < J.num_clouds; ++b) {
    const Ref3Cloud& G = J.c[b];
    const float* __restrict__ xyz = cloud + G.xyz_off;
    const double scaling = P.occupied_space_weight[b] / sqrt(static_cast<double>(G.npts));
    for (int i = threadIdx.x; i < G.npts; i += kRefThreads) {
      const double px = static_cast<double>(xyz[3 * static_cast<size_t>(i)]);
      const double py = static_cast<double>(xyz[3 * static_cast<size_t>(i) + 1]);
      const double pz = static_cast<double>(xyz[3 * static_cast<size_t>(i) + 2]);
      double res, row[kRef3N];
      PointResidual3<kJac>(G, scaling, pose, pj, px, py, pz, &res, row);
      acc[0] += res * res;
      if (kJac) {
#pragma unroll
        for (int a = 0; a < kRef3N; ++a) {
          acc[1 + a] += row[a] * res;
#pragma unroll
          for (int c = a; c < kRef3N; ++c) acc[1 + kRef3N + Tri<kRef3N>(a, c)] += row[a] * row[c];
        }
      }
    }
  }
  BlockSum<kJac ? kRef3Acc : 1>(acc, s_part, s_tot);
  for (int b = 0; kIntensity && b < J.num_clouds; ++b) {
    const Ref3IntensityCloud& G = I->c[b];
    if (G.ivol == nullptr) continue;
    const int npts = J.c[b].npts;
    const float* __restrict__ xyz = cloud + J.c[b].xyz_off;
    const float* __restrict__ intensities = cloud + G.intensity_off;
    // ceres_scan_matcher_3d.cc:133-136: weight / sqrt(n) over the whole cloud
    const double scaling = G.intensity_weight / sqrt(static_cast<double>(npts));
    const float threshold = G.intensity_threshold;
#pragma unroll
    for (int k = 0; k < kRef3Acc; ++k) acc[k] = 0.;
    for (int i = threadIdx.x; i < npts; i += kRefThreads) {
      const double px = static_cast<double>(xyz[3 * static_cast<size_t>(i)]);
      const double py = static_cast<double>(xyz[3 * static_cast<size_t>(i) + 1]);
      const double pz = static_cast<double>(xyz[3 * static_cast<size_t>(i) + 2]);
      double res, row[kRef3N];
      IntensityResidual3<kJac>(G, scaling, threshold, pose, pj, px, py, pz, intensities[i], &res,
                               row);
      acc[0] += res * res;
      if (kJac) {
#pragma unroll
        for (int a = 0; a < kRef3N; ++a) {
          acc[1 + a] += row[a] * res;
#pragma unroll
          for (int c = a; c < kRef3N; ++c) acc[1 + kRef3N + Tri<kRef3N>(a, c)] += row[a] * row[c];
        }
      }
    }
    BlockSum<kJac ? kRef3Acc : 1>(acc, s_part, s_blk);
    if (threadIdx.x == 0) {
      double rho, rho1;
      HuberRho(G.huber_scale, s_blk[0], &rho, &rho1);
      s_tot[0] += rho;
      if (kJac) {
        for (int k = 1; k < kRef3Acc; ++k) s_tot[k] += rho1 * s_blk[k];
      }
    }
  }
  if (threadIdx.x == 0) {
    double res[6], rows[6][kRef3N];
    PriorRows(J, P, pose, pj, res, rows);
    double sq = s_tot[0];
    for (int k = 0; k < 6; ++k) sq += res[k] * res[k];
    s_tot[0] = 0.5 * sq;
    if (kJac) {
      for (int k = 0; k < 6; ++k)
        for (int a = 0; a < kRef3N; ++a) {
          s_tot[1 + a] += rows[k][a] * res[k];
          for (int c = a; c < kRef3N; ++c) s_tot[1 + kRef3N + Tri<kRef3N>(a, c)] += rows[k][a] * rows[k][c];
        }
    }
  }
  __syncthreads();
}

// The 3D match for the minimiser: {t, q} moved in the tangent space of
// QuaternionParameterization; the gradient tolerance is measured as |x - (x (+) -g)|_inf.
template <bool kIntensity>
struct Match3D {
  static constexpr int kAmbient = 7, kN = kRef3N;
  const Ref3JobDev& J;
  const Ref3IntensityJobDev* I;   // read only with kIntensity
  const Ref3Opts& P;
  const float* __restrict__ cloud;
  double (*s_part)[kRef3Acc];
  double* s_blk;

  template <bool kJac>
  __device__ __forceinline__ bool Evaluate(const double* x, double* s_tot) const {
    EvaluateAt3<kJac, kIntensity>(J, I, P, cloud, x, s_part, s_tot, s_blk);
    return true;
  }
  __device__ __forceinline__ static void Plus(const double* x, const double* delta,
                                              double* out) {
    Plus7(x, delta, out);
  }
  __device__ __forceinline__ static double GradientMaxNorm(const double* x, const double* g) {
    double neg[kRef3N], moved[7], gmax = 0.;
#pragma unroll
    for (int a = 0; a < kRef3N; ++a) neg[a] = -g[a];
    Plus7(x, neg, moved);
#pragma unroll
    for (int k = 0; k < 7; ++k) gmax = fmax(gmax, fabs(x[k] - moved[k]));
    return gmax;
  }
};

// One CTA per job.  kIntensity = false compiles out the intensity blocks: a batch in which no
// job has one runs exactly the occupied-space solver; a job without intensity blocks gives
// the same bits in either instantiation.
template <bool kIntensity>
__device__ __forceinline__ void CeresMatch3DBlock(const Ref3JobDev* __restrict__ jobs,
                                                  const Ref3IntensityJobDev* I,
                                                  const Ref3Opts& P,
                                                  const float* __restrict__ cloud,
                                                  Ref3ResultDev* __restrict__ results) {
  __shared__ double s_part[kRefWarps][kRef3Acc];
  __shared__ double s_tot[kRef3Acc];
  __shared__ double s_blk[kIntensity ? kRef3Acc : 1];
  __shared__ double s_pose[7];
  __shared__ int s_cmd;
  __shared__ TrustRegionState<7, kRef3N> S;
  __shared__ Ref3JobDev J;
  if (threadIdx.x == 0) J = jobs[blockIdx.x];
  __syncthreads();
  TrustRegionMinimize(Match3D<kIntensity>{J, I, P, cloud, s_part, s_blk}, J.init,
                      P.max_num_iterations, P.use_nonmonotonic_steps, S, s_tot, s_pose, s_cmd,
                      results + blockIdx.x);
}

__global__ void __launch_bounds__(kRefThreads)
k_ceres_match3d(const Ref3JobDev* __restrict__ jobs, Ref3Opts P, const float* __restrict__ cloud,
                Ref3ResultDev* __restrict__ results) {
  CeresMatch3DBlock<false>(jobs, nullptr, P, cloud, results);
}

__global__ void __launch_bounds__(kRefThreads)
k_ceres_match3d_intensity(const Ref3JobDev* __restrict__ jobs,
                          const Ref3IntensityJobDev* __restrict__ intensity_jobs, Ref3Opts P,
                          const float* __restrict__ cloud, Ref3ResultDev* __restrict__ results) {
  __shared__ Ref3IntensityJobDev I;
  if (threadIdx.x == 0) I = intensity_jobs[blockIdx.x];
  CeresMatch3DBlock<true>(jobs, &I, P, cloud, results);   // (its first barrier publishes I)
}

// Test hook: residuals (and tangent-space Jacobian rows) of one job at one pose, in the
// residual-block order of the problem: per cloud its occupied-space block, then its intensity
// block if it has one; then the priors.  Residuals are uncorrected (no loss function), as
// CostFunction::Evaluate gives them.
// I == nullptr: no intensity blocks.
__device__ __forceinline__ void EvaluateRows3(const Ref3JobDev& J, const Ref3IntensityJobDev* I,
                                              const Ref3Opts& P, const float* __restrict__ cloud,
                                              const double* __restrict__ pose7, int with_jacobian,
                                              double* __restrict__ residuals,
                                              double* __restrict__ jacobian) {
  auto has = [&](int b) { return I != nullptr && I->c[b].ivol != nullptr; };
  double pose[7], pj[12];
  for (int k = 0; k < 7; ++k) pose[k] = pose7[k];
  PlusJacobian(pose + 3, pj);
  int total = 0;
  for (int b = 0; b < J.num_clouds; ++b) total += J.c[b].npts * (has(b) ? 2 : 1);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) {
    int b = 0, local = i;
    bool intensity = false;
    while (local >= J.c[b].npts) {
      local -= J.c[b].npts;
      if (has(b)) {
        if (local < J.c[b].npts) {
          intensity = true;
          break;
        }
        local -= J.c[b].npts;
      }
      ++b;
    }
    const Ref3Cloud& G = J.c[b];
    const float* xyz = cloud + G.xyz_off;
    const double scaling = (intensity ? I->c[b].intensity_weight : P.occupied_space_weight[b]) /
                           sqrt(static_cast<double>(G.npts));
    const double px = static_cast<double>(xyz[3 * static_cast<size_t>(local)]);
    const double py = static_cast<double>(xyz[3 * static_cast<size_t>(local) + 1]);
    const double pz = static_cast<double>(xyz[3 * static_cast<size_t>(local) + 2]);
    double res, row[kRef3N];
    if (intensity) {
      const Ref3IntensityCloud& K = I->c[b];
      const float value = cloud[K.intensity_off + local];
      if (with_jacobian)
        IntensityResidual3<true>(K, scaling, K.intensity_threshold, pose, pj, px, py, pz, value,
                                 &res, row);
      else
        IntensityResidual3<false>(K, scaling, K.intensity_threshold, pose, pj, px, py, pz, value,
                                  &res, row);
    } else if (with_jacobian) {
      PointResidual3<true>(G, scaling, pose, pj, px, py, pz, &res, row);
    } else {
      PointResidual3<false>(G, scaling, pose, pj, px, py, pz, &res, row);
    }
    if (with_jacobian)
      for (int a = 0; a < kRef3N; ++a) jacobian[kRef3N * static_cast<size_t>(i) + a] = row[a];
    residuals[i] = res;
  } else if (i == total) {
    double res[6], rows[6][kRef3N];
    PriorRows(J, P, pose, pj, res, rows);
    for (int k = 0; k < 6; ++k) {
      residuals[total + k] = res[k];
      if (with_jacobian)
        for (int a = 0; a < kRef3N; ++a)
          jacobian[kRef3N * static_cast<size_t>(total + k) + a] = rows[k][a];
    }
  }
}

__global__ void k_ceres_evaluate3d(const Ref3JobDev* __restrict__ job, Ref3Opts P,
                                   const float* __restrict__ cloud, const double* __restrict__ pose7,
                                   int with_jacobian, double* __restrict__ residuals,
                                   double* __restrict__ jacobian) {
  EvaluateRows3(*job, nullptr, P, cloud, pose7, with_jacobian, residuals, jacobian);
}

__global__ void k_ceres_evaluate3d_intensity(const Ref3JobDev* __restrict__ job,
                                             const Ref3IntensityJobDev* __restrict__ intensity_job,
                                             Ref3Opts P, const float* __restrict__ cloud,
                                             const double* __restrict__ pose7, int with_jacobian,
                                             double* __restrict__ residuals,
                                             double* __restrict__ jacobian) {
  EvaluateRows3(*job, intensity_job, P, cloud, pose7, with_jacobian, residuals, jacobian);
}

}  // namespace csm

#ifndef CSM_REFINE_DEVICE_ONLY
using namespace csm;

namespace {

csm_status FillOpts3(const csm_ceres_options3d* o, int max_clouds, Ref3Opts* P) {
  CSM_REQUIRE(o != nullptr, "null options");
  // CHECK_GT(..., 0.) in ceres_scan_matcher_3d.cc:114,143,148
  for (int b = 0; b < max_clouds; ++b)
    CSM_REQUIRE(o->occupied_space_weight[b] > 0., "occupied_space_weight must be positive");
  CSM_REQUIRE(o->translation_weight > 0. && o->rotation_weight > 0., "weights must be positive");
  CSM_REQUIRE(o->max_num_iterations > 0, "max_num_iterations");
  CSM_REQUIRE(o->only_optimize_yaw == 0,
              "only_optimize_yaw (YawOnlyQuaternionPlus) is not supported");
  for (int b = 0; b < kRef3MaxClouds; ++b) P->occupied_space_weight[b] = o->occupied_space_weight[b];
  P->translation_weight = o->translation_weight;
  P->rotation_weight = o->rotation_weight;
  P->use_nonmonotonic_steps = o->use_nonmonotonic_steps != 0;
  P->max_num_iterations = o->max_num_iterations;
  return CSM_OK;
}

csm_status CheckJob(const csm_ceres_job3d& j, int device) {
  CSM_REQUIRE(j.num_clouds >= 1 && j.num_clouds <= kRef3MaxClouds, "1 or 2 point clouds");
  for (int b = 0; b < j.num_clouds; ++b) {
    CSM_REQUIRE(j.grid[b] != nullptr && j.xyz[b] != nullptr, "null pointer");
    CSM_REQUIRE(j.num_points[b] >= 1, "empty point cloud");
    CSM_REQUIRE(j.grid[b]->ctx->device == device, "grids of one batch share a device");
    // a NaN would reach lroundf in CellOf: refused, as the inserters do
    CSM_REQUIRE(Finite(j.xyz[b], 3 * static_cast<size_t>(j.num_points[b])), "non-finite point");
  }
  CSM_REQUIRE(Finite(j.target_translation, 3) && Finite(j.initial_pose, 7),
              "non-finite target or pose");
  return CSM_OK;
}

void FillJob3(const csm_ceres_job3d& j, long long* float_off, Ref3JobDev* d) {
  std::memset(d, 0, sizeof(*d));
  d->num_clouds = j.num_clouds;
  for (int b = 0; b < j.num_clouds; ++b) {
    const Grid3Dev& g = j.grid[b]->g;
    Ref3Cloud& c = d->c[b];
    c.vol = g.p;
    for (int a = 0; a < 3; ++a) {
      c.lo[a] = g.lo[a];
      c.n[a] = g.n[a];
    }
    c.resolution = g.resolution;
    c.k_scale = g.k_scale;
    c.bias = g.bias;
    c.min_probability = g.min_probability;
    c.npts = j.num_points[b];
    c.xyz_off = *float_off;
    *float_off += 3LL * j.num_points[b];
  }
  for (int k = 0; k < 3; ++k) d->target_t[k] = j.target_translation[k];
  for (int k = 0; k < 7; ++k) d->init[k] = j.initial_pose[k];
}

// Whether cloud b of job j has an intensity block (ij may be null: none has).
bool HasIntensity(const csm_ceres_job3d* jobs, const csm_ceres_intensity_job3d* ij, int j,
                  int b) {
  return ij != nullptr && b < jobs[j].num_clouds && ij[j].intensity_grid[b] != nullptr;
}

csm_status CheckIntensityJob(const csm_ceres_job3d& j, const csm_ceres_intensity_job3d& ij,
                             int device) {
  for (int b = 0; b < j.num_clouds; ++b) {
    if (ij.intensity_grid[b] == nullptr) continue;
    CSM_REQUIRE(ij.intensities[b] != nullptr, "an intensity grid needs the cloud's intensities");
    CSM_REQUIRE(ij.intensity_grid[b]->ctx->device == device, "grids of one batch share a device");
    CSM_REQUIRE(Finite(ij.intensities[b], static_cast<size_t>(j.num_points[b])),
                "non-finite intensity");
  }
  return CSM_OK;
}

// CHECK_GT(..., 0) in ceres_scan_matcher_3d.cc:124-127, for the clouds that use them
csm_status CheckIntensityOpts3(const csm_ceres_intensity_options3d* o, const bool used[2]) {
  for (int b = 0; b < kRef3MaxClouds; ++b) {
    if (!used[b]) continue;
    CSM_REQUIRE(o != nullptr, "null intensity options");
    CSM_REQUIRE(o->huber_scale[b] > 0., "huber_scale must be positive");
    CSM_REQUIRE(o->weight[b] > 0., "intensity weight must be positive");
    CSM_REQUIRE(o->intensity_threshold[b] > 0.f, "intensity_threshold must be positive");
  }
  return CSM_OK;
}

// Points the job's intensity blocks at their grids, their options and at intensities placed
// from *float_off.
void FillIntensity3(const csm_ceres_job3d& j, const csm_ceres_intensity_job3d* ij,
                    const csm_ceres_intensity_options3d* o, long long* float_off,
                    Ref3IntensityJobDev* d) {
  std::memset(d, 0, sizeof(*d));
  for (int b = 0; ij != nullptr && b < j.num_clouds; ++b) {
    const csm_intensity_grid3d* g = ij->intensity_grid[b];
    if (g == nullptr) continue;
    Ref3IntensityCloud& c = d->c[b];
    c.ivol = g->d_vol;
    for (int a = 0; a < 3; ++a) {
      c.ilo[a] = g->box.lo[a];
      c.in[a] = g->box.n[a];
    }
    c.iresolution = g->resolution;
    c.intensity_threshold = o->intensity_threshold[b];
    c.intensity_weight = o->weight[b];
    c.huber_scale = o->huber_scale[b];
    c.intensity_off = *float_off;
    *float_off += j.num_points[b];
  }
}

// Validation shared by the batch and the evaluate hook: *floats = the upload's float count,
// *any_intensity = whether some job has an intensity block, P = the solver options.
csm_status Prepare3(const csm_ceres_job3d* jobs, const csm_ceres_intensity_job3d* ij,
                    int num_jobs, const csm_ceres_options3d* options,
                    const csm_ceres_intensity_options3d* intensity_options, int* device,
                    long long* floats, bool* any_intensity, Ref3Opts* P) {
  CSM_REQUIRE(jobs[0].num_clouds >= 1 && jobs[0].grid[0] != nullptr, "null pointer");
  *device = jobs[0].grid[0]->ctx->device;
  int max_clouds = 0;
  bool used[kRef3MaxClouds] = {false, false};
  *floats = 0;
  for (int j = 0; j < num_jobs; ++j) {
    CSM_TRY(CheckJob(jobs[j], *device));
    if (ij != nullptr) CSM_TRY(CheckIntensityJob(jobs[j], ij[j], *device));
    max_clouds = std::max(max_clouds, jobs[j].num_clouds);
    for (int b = 0; b < jobs[j].num_clouds; ++b) {
      *floats += 3LL * jobs[j].num_points[b];
      if (HasIntensity(jobs, ij, j, b)) {
        used[b] = true;
        *floats += jobs[j].num_points[b];
      }
    }
  }
  CSM_REQUIRE(*floats < (1LL << 31), "batch too large");
  CSM_TRY(FillOpts3(options, max_clouds, P));
  *any_intensity = used[0] || used[1];
  return CheckIntensityOpts3(intensity_options, used);
}

// Job j's records and point data into the upload buffer h (floats from *off); hi may be null
// when no job of the batch has an intensity block.
void Stage3(const csm_ceres_job3d* jobs, const csm_ceres_intensity_job3d* ij,
            const csm_ceres_intensity_options3d* io, int j, long long* off, char* h,
            Ref3JobDev* hj, Ref3IntensityJobDev* hi) {
  const csm_ceres_job3d& job = jobs[j];
  FillJob3(job, off, hj);
  if (hi != nullptr) FillIntensity3(job, ij != nullptr ? &ij[j] : nullptr, io, off, hi);
  float* f = reinterpret_cast<float*>(h);
  for (int b = 0; b < job.num_clouds; ++b) {
    std::memcpy(f + hj->c[b].xyz_off, job.xyz[b],
                sizeof(float) * 3 * static_cast<size_t>(job.num_points[b]));
    if (HasIntensity(jobs, ij, j, b))
      std::memcpy(f + hi->c[b].intensity_off, ij[j].intensities[b],
                  sizeof(float) * static_cast<size_t>(job.num_points[b]));
  }
}

csm_status MatchBatch3(const csm_ceres_job3d* jobs, const csm_ceres_intensity_job3d* ij,
                       int32_t num_jobs, const csm_ceres_options3d* options,
                       const csm_ceres_intensity_options3d* intensity_options,
                       csm_ceres_result3d* results, csm_stats* stats) {
  CSM_REQUIRE(jobs && results, "null pointer");
  CSM_REQUIRE(num_jobs >= 1, "empty batch");
  int device;
  long long floats;
  Ref3Opts P;
  bool any_intensity;
  CSM_TRY(Prepare3(jobs, ij, num_jobs, options, intensity_options, &device, &floats,
                   &any_intensity, &P));
  LaneGuard guard;
  CSM_TRY(AcquireLane(device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t off_jobs = (static_cast<size_t>(floats) * 4 + 255) / 256 * 256;
  const size_t off_ijobs = off_jobs + sizeof(Ref3JobDev) * num_jobs;
  const size_t up_bytes = off_ijobs + (any_intensity ? sizeof(Ref3IntensityJobDev) * num_jobs : 0);
  PinnedBuf& up = ctx->P("ref3_upload");
  DevBuf& d_up = ctx->D("ref3_upload");
  DevBuf& d_out = ctx->D("ref3_results");
  PinnedBuf& rb = ctx->P("ref3_readback");
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(d_up.Reserve(up_bytes));
  CSM_TRY(d_out.Reserve(sizeof(Ref3ResultDev) * num_jobs));
  CSM_TRY(rb.Reserve(sizeof(Ref3ResultDev) * num_jobs));
  char* h = up.as<char>();
  Ref3JobDev* hj = reinterpret_cast<Ref3JobDev*>(h + off_jobs);
  Ref3IntensityJobDev* hi =
      any_intensity ? reinterpret_cast<Ref3IntensityJobDev*>(h + off_ijobs) : nullptr;
  long long off = 0;
  for (int j = 0; j < num_jobs; ++j)
    Stage3(jobs, ij, intensity_options, j, &off, h, &hj[j], hi ? &hi[j] : nullptr);
  CSM_CUDA(cudaEventRecord(ctx->ev0, s));
  CSM_CUDA(cudaMemcpyAsync(d_up.p, h, up_bytes, cudaMemcpyHostToDevice, s));
  ProfBegin(ctx);
  const Ref3JobDev* d_jobs = reinterpret_cast<const Ref3JobDev*>(d_up.as<char>() + off_jobs);
  if (any_intensity)
    k_ceres_match3d_intensity<<<num_jobs, kRefThreads, 0, s>>>(
        d_jobs, reinterpret_cast<const Ref3IntensityJobDev*>(d_up.as<char>() + off_ijobs), P,
        d_up.as<float>(), d_out.as<Ref3ResultDev>());
  else
    k_ceres_match3d<<<num_jobs, kRefThreads, 0, s>>>(d_jobs, P, d_up.as<float>(),
                                                    d_out.as<Ref3ResultDev>());
  CSM_LAUNCH_CHECK();
  ProfEnd(ctx, any_intensity ? "k_ceres_match3d_intensity" : "k_ceres_match3d",
          static_cast<double>(num_jobs));
  CSM_CUDA(cudaEventRecord(ctx->ev1, s));
  CSM_CUDA(cudaMemcpyAsync(rb.p, d_out.p, sizeof(Ref3ResultDev) * num_jobs,
                           cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  const Ref3ResultDev* r = rb.as<Ref3ResultDev>();
  for (int j = 0; j < num_jobs; ++j) {
    csm_ceres_result3d& o = results[j];
    std::memset(&o, 0, sizeof(o));
    std::memcpy(o.pose_estimate, r[j].pose, sizeof(double) * 7);
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

csm_status Evaluate3(const csm_ceres_job3d* job, const csm_ceres_intensity_job3d* ij,
                     const csm_ceres_options3d* options,
                     const csm_ceres_intensity_options3d* intensity_options, const double pose[7],
                     double* residuals, double* jacobian) {
  CSM_REQUIRE(job && pose && residuals, "null pointer");
  CSM_REQUIRE(Finite(pose, 7), "non-finite pose");
  int device;
  long long floats;
  Ref3Opts P;
  bool any_intensity;
  CSM_TRY(Prepare3(job, ij, 1, options, intensity_options, &device, &floats, &any_intensity,
                   &P));
  size_t rows = 6;
  for (int b = 0; b < job->num_clouds; ++b)
    rows += static_cast<size_t>(job->num_points[b]) * (HasIntensity(job, ij, 0, b) ? 2 : 1);
  LaneGuard guard;
  CSM_TRY(AcquireLane(device, &guard));
  Ctx* ctx = guard.lane;
  CSM_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  const size_t off_job = (static_cast<size_t>(floats) * 4 + 255) / 256 * 256;
  const size_t off_ijob = off_job + (sizeof(Ref3JobDev) + 255) / 256 * 256;
  const size_t off_pose = off_ijob + (sizeof(Ref3IntensityJobDev) + 255) / 256 * 256;
  const size_t up_bytes = off_pose + 64;
  PinnedBuf& up = ctx->P("ref3_eval_upload");
  DevBuf& d_up = ctx->D("ref3_eval_upload");
  DevBuf& d_res = ctx->D("ref3_eval_res");
  DevBuf& d_jac = ctx->D("ref3_eval_jac");
  CSM_TRY(up.Reserve(up_bytes));
  CSM_TRY(d_up.Reserve(up_bytes));
  CSM_TRY(d_res.Reserve(sizeof(double) * rows));
  CSM_TRY(d_jac.Reserve(sizeof(double) * kRef3N * rows));
  char* h = up.as<char>();
  long long off = 0;
  Stage3(job, ij, intensity_options, 0, &off, h, reinterpret_cast<Ref3JobDev*>(h + off_job),
         reinterpret_cast<Ref3IntensityJobDev*>(h + off_ijob));
  std::memcpy(h + off_pose, pose, sizeof(double) * 7);
  CSM_CUDA(cudaMemcpyAsync(d_up.p, h, up_bytes, cudaMemcpyHostToDevice, s));
  const dim3 grid(static_cast<unsigned>((rows + 255) / 256));
  const Ref3JobDev* d_job = reinterpret_cast<const Ref3JobDev*>(d_up.as<char>() + off_job);
  const double* d_pose = reinterpret_cast<const double*>(d_up.as<char>() + off_pose);
  if (any_intensity)
    k_ceres_evaluate3d_intensity<<<grid, 256, 0, s>>>(
        d_job, reinterpret_cast<const Ref3IntensityJobDev*>(d_up.as<char>() + off_ijob), P,
        d_up.as<float>(), d_pose, jacobian != nullptr, d_res.as<double>(), d_jac.as<double>());
  else
    k_ceres_evaluate3d<<<grid, 256, 0, s>>>(d_job, P, d_up.as<float>(), d_pose,
                                            jacobian != nullptr, d_res.as<double>(),
                                            d_jac.as<double>());
  CSM_LAUNCH_CHECK();
  CSM_CUDA(cudaMemcpyAsync(residuals, d_res.p, sizeof(double) * rows, cudaMemcpyDeviceToHost, s));
  if (jacobian)
    CSM_CUDA(cudaMemcpyAsync(jacobian, d_jac.p, sizeof(double) * kRef3N * rows,
                             cudaMemcpyDeviceToHost, s));
  CSM_CUDA(cudaStreamSynchronize(s));
  return CSM_OK;
}

}  // namespace

extern "C" {

csm_status csm_ceres_match3d_batch(const csm_ceres_job3d* jobs, int32_t num_jobs,
                                   const csm_ceres_options3d* options,
                                   csm_ceres_result3d* results, csm_stats* stats) {
  return MatchBatch3(jobs, nullptr, num_jobs, options, nullptr, results, stats);
}

csm_status csm_ceres_match3d_intensity_batch(
    const csm_ceres_job3d* jobs, const csm_ceres_intensity_job3d* intensity_jobs,
    int32_t num_jobs, const csm_ceres_options3d* options,
    const csm_ceres_intensity_options3d* intensity_options, csm_ceres_result3d* results,
    csm_stats* stats) {
  CSM_REQUIRE(intensity_jobs != nullptr, "null pointer");
  return MatchBatch3(jobs, intensity_jobs, num_jobs, options, intensity_options, results, stats);
}

csm_status csm_ceres_evaluate3d(const csm_ceres_job3d* job, const csm_ceres_options3d* options,
                                const double pose[7], double* residuals, double* jacobian) {
  return Evaluate3(job, nullptr, options, nullptr, pose, residuals, jacobian);
}

csm_status csm_ceres_evaluate3d_intensity(const csm_ceres_job3d* job,
                                          const csm_ceres_intensity_job3d* intensity_job,
                                          const csm_ceres_options3d* options,
                                          const csm_ceres_intensity_options3d* intensity_options,
                                          const double pose[7], double* residuals,
                                          double* jacobian) {
  CSM_REQUIRE(intensity_job != nullptr, "null pointer");
  return Evaluate3(job, intensity_job, options, intensity_options, pose, residuals, jacobian);
}

}  // extern "C"
#endif  // CSM_REFINE_DEVICE_ONLY
