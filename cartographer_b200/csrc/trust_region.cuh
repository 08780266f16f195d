// The trust-region minimiser of the post-match refinement (refine2d.cu, refine3d.cu): what
// Ceres' TrustRegionMinimizer does with Solver::Options defaults + {DENSE_QR,
// use_nonmonotonic_steps, max_num_iterations} (ceres_scan_matcher_2d.cc:52-57,
// ceres_scan_matcher_3d.cc, ceres_solver_options.cc:37-44), one problem per CTA:
//   Jacobi column scaling fixed at the first Jacobian, Levenberg-Marquardt damping
//   D^2 = clamp(diag(Js^T Js)) / radius, the damped normal equations by Cholesky (Ceres:
//   Householder QR of [Js; D] — the same minimiser), step quality against the model decrease,
//   non-monotonic acceptance (Conn, Gould & Toint, Alg. 10.1.2), radius update, and the
//   function / gradient / parameter tolerances; the lowest-cost iterate is what is returned,
//   as Ceres does under non-monotonic steps.
//
// A Problem supplies
//   kAmbient, kN                      parameter and tangent-space dimensions;
//   Evaluate<kJac>(x, s_tot) -> bool  block-wide: s_tot = {1/2 sum r^2, g[kN], upper triangle
//                                     of H (Tri)}, g and H only with kJac; false (block-uniform)
//                                     where the cost function fails;
//   Plus(x, delta, out)               x (+) delta;
//   GradientMaxNorm(x, g)             the gradient-tolerance measure.
// The solver's state is touched by thread 0 only; the caller decides where it lives (every
// loop over kN / kAmbient is unrolled so that a kernel-local state can stay in registers).
// Sums run in index order from their first term (0. + x is not x when x is -0.), and the
// callers are compiled without FMA contraction (Makefile: -fmad=false).
#pragma once

#include <cfloat>
#include <cmath>

namespace csm {

constexpr int kRefThreads = 256;
constexpr int kRefWarps = kRefThreads / 32;

// index of (i, j), i <= j, in the row-major upper triangle of a kN x kN matrix
template <int kN>
__device__ __forceinline__ constexpr int Tri(int i, int j) {
  return i * kN - i * (i - 1) / 2 + (j - i);
}

// Block sum of acc[0 .. kCount); every thread returns with the totals in s_tot.
template <int kCount, int kWidth>
__device__ __forceinline__ void BlockSum(const double* acc, double (*s_part)[kWidth],
                                         double* s_tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kCount; ++k) {
    double v = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) s_part[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < kCount) {
    double v = 0.;
#pragma unroll
    for (int w = 0; w < kRefWarps; ++w) v += s_part[w][threadIdx.x];
    s_tot[threadIdx.x] = v;
  }
  __syncthreads();
}

template <int kN>
__device__ __forceinline__ double Norm(const double* v) {
  double s = v[0] * v[0];
#pragma unroll
  for (int i = 1; i < kN; ++i) s += v[i] * v[i];
  return sqrt(s);
}

// Cholesky solve of A y = b, A symmetric positive definite (upper triangle, Tri order);
// false where A is not numerically positive definite or y is not finite.
template <int kN>
__device__ __forceinline__ bool SolveSpd(const double* a, const double* b, double* y) {
  double l[kN][kN];
#pragma unroll
  for (int i = 0; i < kN; ++i) {
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      double s = a[Tri<kN>(j, i)];
#pragma unroll
      for (int k = 0; k < j; ++k) s -= l[i][k] * l[j][k];
      if (i == j) {
        if (!(s > 0.)) return false;
        l[i][i] = sqrt(s);
      } else {
        l[i][j] = s / l[j][j];
      }
    }
  }
  double z[kN];
#pragma unroll
  for (int i = 0; i < kN; ++i) {
    double s = b[i];
#pragma unroll
    for (int k = 0; k < i; ++k) s -= l[i][k] * z[k];
    z[i] = s / l[i][i];
  }
#pragma unroll
  for (int i = kN - 1; i >= 0; --i) {
    double s = z[i];
#pragma unroll
    for (int k = i + 1; k < kN; ++k) s -= l[k][i] * y[k];
    y[i] = s / l[i][i];
  }
  bool finite = true;
#pragma unroll
  for (int i = 0; i < kN; ++i) finite = finite && isfinite(y[i]);
  return finite;
}

enum { kCmdEvalCandidate = 0, kCmdAccept = 1, kCmdRejected = 2, kCmdDone = 3 };
// csm_abi.h's termination codes
enum {
  kTermNoConvergence = 0, kTermFunctionTolerance = 1, kTermGradientTolerance = 2,
  kTermParameterTolerance = 3, kTermMinRadius = 4, kTermInvalidSteps = 5,
  kTermEvaluationFailed = 6
};

template <int kAmbient>
struct ResultDev {
  double pose[kAmbient];
  double initial_cost, final_cost;
  int iterations, num_successful_steps, termination, pad;
};

template <int kAmbient, int kN>
struct TrustRegionState {
  static constexpr int kH = kN * (kN + 1) / 2;
  double x[kAmbient], best[kAmbient], cand[kAmbient];
  double g[kN], h[kH], scale[kN], diagonal[kN];
  double x_cost, x_norm, minimum_cost, initial_cost;
  double radius, decrease_factor;
  double current_cost, reference_cost, candidate_cost_ev, ev_minimum_cost;
  double acc_reference, acc_candidate, model_cost_change;
  bool reuse_diagonal, last_step_successful;
  int num_nonmonotonic, num_invalid, iteration, successful, termination;
};

// Minimise `problem` from `init` (block-wide; s_tot, s_pose and s_cmd in shared memory).
// Where the cost function fails Ceres' minimiser does: at a trial point the candidate's cost
// is the largest double, so the step is rejected; at the initial point (or at an accepted
// point, for its Jacobian) the solve ends as FAILURE and the parameters keep `init`.
template <class Problem>
__device__ __forceinline__ void TrustRegionMinimize(
    const Problem& problem, const double* init, int max_num_iterations,
    bool use_nonmonotonic_steps, TrustRegionState<Problem::kAmbient, Problem::kN>& S,
    double* s_tot, double* s_pose, int& s_cmd, ResultDev<Problem::kAmbient>* result) {
  constexpr int kAmbient = Problem::kAmbient, kN = Problem::kN;
  constexpr int kH = TrustRegionState<kAmbient, kN>::kH;
  // Solver::Options defaults the reference leaves untouched
  const double kInitialRadius = 1e4, kMaxRadius = 1e16, kMinRadius = 1e-32;
  const double kMinRelativeDecrease = 1e-3, kMinLmDiagonal = 1e-6, kMaxLmDiagonal = 1e32;
  const int kMaxConsecutiveInvalidSteps = 5;
  const double kFunctionTolerance = 1e-6, kGradientTolerance = 1e-10, kParameterTolerance = 1e-8;
  const int max_nonmonotonic = use_nonmonotonic_steps ? 5 : 0;

  bool failed = !problem.template Evaluate<true>(init, s_tot);
  if (failed) {
    if (threadIdx.x == 0) {
      // Solver::Summary keeps its defaults (costs -1) when iteration zero fails
      ResultDev<kAmbient> out;
#pragma unroll
      for (int k = 0; k < kAmbient; ++k) out.pose[k] = init[k];
      out.initial_cost = out.final_cost = -1.;
      out.iterations = out.num_successful_steps = 0;
      out.termination = kTermEvaluationFailed;
      out.pad = 0;
      *result = out;
    }
    return;
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < kAmbient; ++k) S.x[k] = S.best[k] = S.cand[k] = init[k];
    S.x_cost = s_tot[0];
#pragma unroll
    for (int a = 0; a < kN; ++a) S.g[a] = s_tot[1 + a];
#pragma unroll
    for (int a = 0; a < kH; ++a) S.h[a] = s_tot[1 + kN + a];
    S.x_norm = Norm<kAmbient>(S.x);
    S.initial_cost = S.minimum_cost = S.x_cost;
    S.current_cost = S.reference_cost = S.candidate_cost_ev = S.ev_minimum_cost = S.x_cost;
#pragma unroll
    for (int a = 0; a < kN; ++a) {
      S.scale[a] = 1.0 / (1.0 + sqrt(S.h[Tri<kN>(a, a)]));
      S.diagonal[a] = 0.;
    }
    S.radius = kInitialRadius;
    S.decrease_factor = 2.0;
    S.reuse_diagonal = false;
    S.last_step_successful = false;
    S.acc_reference = S.acc_candidate = S.model_cost_change = 0.;
    S.num_nonmonotonic = S.num_invalid = S.iteration = S.successful = 0;
    S.termination = kTermNoConvergence;
  }
  __syncthreads();   // s_tot is overwritten by the next evaluation

  while (true) {
    // ---- thread 0: close the previous iteration, stopping tests, next trial step ----
    if (threadIdx.x == 0) {
      int cmd = kCmdEvalCandidate;
      while (true) {   // (repeats only after an invalid step)
        if (S.last_step_successful) {
          ++S.successful;
          if (S.x_cost < S.minimum_cost) {
            S.minimum_cost = S.x_cost;
#pragma unroll
            for (int k = 0; k < kAmbient; ++k) S.best[k] = S.x[k];
          }
          S.last_step_successful = false;
        }
        if (S.iteration >= max_num_iterations) { S.termination = kTermNoConvergence; cmd = kCmdDone; break; }
        if (Problem::GradientMaxNorm(S.x, S.g) <= kGradientTolerance) { S.termination = kTermGradientTolerance; cmd = kCmdDone; break; }
        if (S.radius <= kMinRadius) { S.termination = kTermMinRadius; cmd = kCmdDone; break; }
        ++S.iteration;
        double hs[kH], gs[kN];
#pragma unroll
        for (int a = 0; a < kN; ++a) {
          gs[a] = S.g[a] * S.scale[a];
#pragma unroll
          for (int c = a; c < kN; ++c)
            hs[Tri<kN>(a, c)] = S.h[Tri<kN>(a, c)] * S.scale[a] * S.scale[c];
        }
        if (!S.reuse_diagonal) {
#pragma unroll
          for (int a = 0; a < kN; ++a)
            S.diagonal[a] = fmin(fmax(hs[Tri<kN>(a, a)], kMinLmDiagonal), kMaxLmDiagonal);
        }
        double am[kH];
#pragma unroll
        for (int i = 0; i < kH; ++i) am[i] = hs[i];
#pragma unroll
        for (int a = 0; a < kN; ++a) am[Tri<kN>(a, a)] = hs[Tri<kN>(a, a)] + S.diagonal[a] / S.radius;
        double y[kN];
        bool valid = SolveSpd<kN>(am, gs, y);
        S.reuse_diagonal = true;
        double step[kN];
#pragma unroll
        for (int a = 0; a < kN; ++a) step[a] = 0.;
        if (valid) {
#pragma unroll
          for (int a = 0; a < kN; ++a) step[a] = -y[a];
          double hs_step[kN];
#pragma unroll
          for (int a = 0; a < kN; ++a) {
            hs_step[a] = hs[Tri<kN>(0, a)] * step[0];
#pragma unroll
            for (int c = 1; c < kN; ++c)
              hs_step[a] += hs[a <= c ? Tri<kN>(a, c) : Tri<kN>(c, a)] * step[c];
          }
          double sg = step[0] * gs[0], shs = step[0] * hs_step[0];
#pragma unroll
          for (int a = 1; a < kN; ++a) {
            sg += step[a] * gs[a];
            shs += step[a] * hs_step[a];
          }
          S.model_cost_change = -(sg + 0.5 * shs);
          valid = !(S.model_cost_change < 0.0);
        }
        if (!valid) {
          if (++S.num_invalid >= kMaxConsecutiveInvalidSteps) { S.termination = kTermInvalidSteps; cmd = kCmdDone; break; }
          S.radius = S.radius / S.decrease_factor;
          S.decrease_factor *= 2.0;
          S.reuse_diagonal = false;
          continue;
        }
        S.num_invalid = 0;
        double delta[kN];
#pragma unroll
        for (int a = 0; a < kN; ++a) delta[a] = step[a] * S.scale[a];
        Problem::Plus(S.x, delta, S.cand);
        break;
      }
#pragma unroll
      for (int k = 0; k < kAmbient; ++k) s_pose[k] = S.cand[k];
      s_cmd = cmd;
    }
    __syncthreads();
    if (s_cmd == kCmdDone) break;
    {
      double p[kAmbient];
#pragma unroll
      for (int k = 0; k < kAmbient; ++k) p[k] = s_pose[k];
      __syncthreads();
      // the candidate's cost, plain doubles
      const bool ok = problem.template Evaluate<false>(p, s_tot);
      if (threadIdx.x == 0) s_tot[0] = ok ? s_tot[0] : DBL_MAX;
    }
    // ---- thread 0: tolerances on the trial step, step quality --------------------
    if (threadIdx.x == 0) {
      const double candidate_cost = s_tot[0];
      int cmd = kCmdRejected;
      double diff[kAmbient];
#pragma unroll
      for (int k = 0; k < kAmbient; ++k) diff[k] = S.x[k] - S.cand[k];
      if (Norm<kAmbient>(diff) <= kParameterTolerance * (S.x_norm + kParameterTolerance)) {
        S.termination = kTermParameterTolerance;   // the step is not taken
        cmd = kCmdDone;
      } else if (fabs(S.x_cost - candidate_cost) <= kFunctionTolerance * S.x_cost) {
        S.termination = kTermFunctionTolerance;    // the step is not taken
        cmd = kCmdDone;
      } else {
        const double relative_decrease = (S.current_cost - candidate_cost) / S.model_cost_change;
        const double historical_decrease =
            (S.reference_cost - candidate_cost) / (S.acc_reference + S.model_cost_change);
        const double step_quality = fmax(relative_decrease, historical_decrease);
        if (step_quality > kMinRelativeDecrease) {
          cmd = kCmdAccept;
#pragma unroll
          for (int k = 0; k < kAmbient; ++k) S.x[k] = S.cand[k];
          S.x_norm = Norm<kAmbient>(S.x);
          const double t = 2.0 * step_quality - 1.0;
          S.radius = S.radius / fmax(1.0 / 3.0, 1.0 - t * t * t);
          S.radius = fmin(kMaxRadius, S.radius);
          S.decrease_factor = 2.0;
          S.reuse_diagonal = false;
          S.current_cost = candidate_cost;
          S.acc_candidate += S.model_cost_change;
          S.acc_reference += S.model_cost_change;
          if (S.current_cost < S.ev_minimum_cost) {
            S.ev_minimum_cost = S.current_cost;
            S.num_nonmonotonic = 0;
            S.candidate_cost_ev = S.current_cost;
            S.acc_candidate = 0.;
          } else {
            ++S.num_nonmonotonic;
            if (S.current_cost > S.candidate_cost_ev) {
              S.candidate_cost_ev = S.current_cost;
              S.acc_candidate = 0.;
            }
          }
          if (S.num_nonmonotonic == max_nonmonotonic) {
            S.reference_cost = S.candidate_cost_ev;
            S.acc_reference = S.acc_candidate;
          }
        } else {
          S.radius = S.radius / S.decrease_factor;
          S.decrease_factor *= 2.0;
          S.reuse_diagonal = true;
        }
      }
      s_cmd = cmd;
    }
    __syncthreads();
    if (s_cmd == kCmdDone) break;
    if (s_cmd == kCmdAccept) {
      double p[kAmbient];
#pragma unroll
      for (int k = 0; k < kAmbient; ++k) p[k] = s_pose[k];
      __syncthreads();
      // residuals + Jacobian at the new x
      if (!problem.template Evaluate<true>(p, s_tot)) {
        failed = true;
        break;
      }
      if (threadIdx.x == 0) {
        S.x_cost = s_tot[0];
#pragma unroll
        for (int a = 0; a < kN; ++a) S.g[a] = s_tot[1 + a];
#pragma unroll
        for (int a = 0; a < kH; ++a) S.h[a] = s_tot[1 + kN + a];
        S.last_step_successful = true;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (failed) {   // FAILURE: the parameters keep the initial estimate
#pragma unroll
      for (int k = 0; k < kAmbient; ++k) S.best[k] = init[k];
      S.minimum_cost = S.initial_cost;
      S.termination = kTermEvaluationFailed;
    }
    ResultDev<kAmbient> out;
#pragma unroll
    for (int k = 0; k < kAmbient; ++k) out.pose[k] = S.best[k];
    out.initial_cost = S.initial_cost;
    out.final_cost = S.minimum_cost;
    out.iterations = S.iteration;
    out.num_successful_steps = S.successful;
    out.termination = S.termination;
    out.pad = 0;
    *result = out;
  }
}

}  // namespace csm
