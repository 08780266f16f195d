"""CPU restatement of CeresScanMatcher2D on a TSDF2D — TEST INFRASTRUCTURE ONLY.

What is restated (the product's device code is checked against this, never the reverse):
  * TSDF2D's cells (mapping/internal/2d/tsdf_2d.cc): SetCell with the update marker,
    GetWeight (0 outside the limits) and Grid2D::GetCorrespondenceCost with the TSDF bounds
    +-truncation (value 0 and outside the limits give +truncation), the TSDValueConverter
    (tsd_value_converter.{h,cc}) and the value -> float tables in float32;
  * InterpolatedTSDF2D (scan_matching/interpolated_tsdf_2d.h): the lower pixel found on the
    scalar part in float through MapLimits::GetCellIndex / GetCellCenter, bilinear
    interpolation, the constant maximum cost (no derivative) where a corner weight is 0;
  * TSDFMatchCostFunction2D (tsdf_match_cost_function_2d.cc:42-65) on plain doubles and on
    dual numbers in ceres/jet.h's operation order (a Jet divided by a Jet multiplies by the
    reciprocal of the denominator's value), returning "invalid" where summed_weight == 0;
  * the trust-region loop of the ProbabilityGrid oracle (oracle/oracle_ceres2d.cc, the same
    restatement of Ceres' published minimiser and the same caveat) plus what Ceres' minimiser
    does when a cost function fails: at the initial point (or for the Jacobian at an accepted
    point) the solve ends as FAILURE and the parameters keep the initial estimate; at a trial
    point the candidate cost is the largest double, so the step is rejected.

Sums over points are numpy's, not the device's block-tree order: parity with the device is
to the tolerances of the tests, not bit for bit.
"""
import math
import sys

import numpy as np

from oracle.pyoracle import ceres_trace_record

F = np.float32
UPDATE_MARKER = 1 << 15
DBL_MAX = sys.float_info.max
# csm_ceres_result2d::termination; 6 = the cost function failed where Ceres stops (FAILURE)
CERES_TERMINATION = ("NO_CONVERGENCE", "FUNCTION_TOLERANCE", "GRADIENT_TOLERANCE",
                     "PARAMETER_TOLERANCE", "MIN_TRUST_REGION_RADIUS", "INVALID_STEPS",
                     "EVALUATION_FAILED")


def lround(v):
    """std::lround of doubles (halves away from zero), elementwise."""
    v = np.asarray(v, np.float64)
    t = np.trunc(v)
    return (t + np.where(np.abs(v - t) >= 0.5, np.sign(v), 0.0)).astype(np.int64)


class TSDValueConverter:
    def __init__(self, truncation, max_weight):
        self.max_tsd = F(truncation)
        self.min_tsd = -self.max_tsd
        self.max_weight = F(max_weight)
        self.tsd_resolution = F(32766) / (self.max_tsd - self.min_tsd)
        self.weight_resolution = F(32766) / (self.max_weight - F(0))
        # value_conversion_tables.cc: value * scale + (lower - scale) for value > 0
        self.tsd_scale = (self.max_tsd - self.min_tsd) / F(32766)
        self.tsd_bias = self.min_tsd - self.tsd_scale
        self.w_scale = (self.max_weight - F(0)) / F(32766)
        self.w_bias = F(0) - self.w_scale

    def tsd_to_value(self, tsd):
        c = np.clip(F(tsd), self.min_tsd, self.max_tsd)
        return int(lround(np.float64((c - self.min_tsd) * self.tsd_resolution))) + 1

    def weight_to_value(self, weight):
        c = np.clip(F(weight), F(0), self.max_weight)
        return int(lround(np.float64((c - F(0)) * self.weight_resolution))) + 1

    def value_to_cost(self, values):
        """Grid2D's value -> correspondence cost table with bounds +-truncation."""
        v = np.asarray(values, np.int64) & 0x7fff
        return np.where(v == 0, self.max_tsd, v.astype(F) * self.tsd_scale + self.tsd_bias).astype(F)

    def value_to_weight(self, values):
        v = np.asarray(values, np.int64) & 0x7fff
        return np.where(v == 0, F(0), v.astype(F) * self.w_scale + self.w_bias).astype(F)


class TSDF2D:
    """tsd / weight cells [y, x] (flat index num_x * y + x) with MapLimits."""

    def __init__(self, num_x, num_y, resolution, max_x, max_y, truncation, max_weight,
                 tsd_cells=None, weight_cells=None):
        self.num_x, self.num_y = int(num_x), int(num_y)
        self.resolution, self.max_x, self.max_y = float(resolution), float(max_x), float(max_y)
        self.truncation_distance, self.max_weight = float(F(truncation)), float(F(max_weight))
        self.conv = TSDValueConverter(truncation, max_weight)
        shape = (self.num_y, self.num_x)
        self.tsd_cells = (np.zeros(shape, np.uint16) if tsd_cells is None
                          else np.array(tsd_cells, np.uint16).reshape(shape))
        self.weight_cells = (np.zeros(shape, np.uint16) if weight_cells is None
                             else np.array(weight_cells, np.uint16).reshape(shape))

    @classmethod
    def from_spec(cls, spec):
        ny, nx = spec.tsd_cells.shape
        return cls(nx, ny, spec.resolution, spec.max_x, spec.max_y, spec.truncation_distance,
                   spec.max_weight, spec.tsd_cells, spec.weight_cells)

    def cell_index(self, px, py):
        """MapLimits::GetCellIndex(Vector2f): (ix from y, iy from x)."""
        px = np.asarray(px, F).astype(np.float64)
        py = np.asarray(py, F).astype(np.float64)
        return (lround((self.max_y - py) / self.resolution - 0.5),
                lround((self.max_x - px) / self.resolution - 0.5))

    def cell_center(self, ix, iy):
        """MapLimits::GetCellCenter, stored to float."""
        return ((self.max_x - self.resolution * (np.asarray(iy) + 0.5)).astype(F),
                (self.max_y - self.resolution * (np.asarray(ix) + 0.5)).astype(F))

    def _inside(self, ix, iy):
        return (ix >= 0) & (iy >= 0) & (ix < self.num_x) & (iy < self.num_y)

    def set_cell(self, ix, iy, tsd, weight):
        """TSDF2D::SetCell (tsdf_2d.cc:55-68): a cell already updated is left alone."""
        if self.tsd_cells[iy, ix] >= UPDATE_MARKER:
            return
        self.tsd_cells[iy, ix] = self.conv.tsd_to_value(tsd) + UPDATE_MARKER
        self.weight_cells[iy, ix] = self.conv.weight_to_value(weight)

    def finish_update(self):
        self.tsd_cells &= 0x7fff

    def get_weight(self, ix, iy):
        ix, iy = np.asarray(ix), np.asarray(iy)
        inside = self._inside(ix, iy)
        v = self.weight_cells[np.where(inside, iy, 0), np.where(inside, ix, 0)]
        return np.where(inside, self.conv.value_to_weight(v), F(0)).astype(F)

    def get_correspondence_cost(self, ix, iy):
        ix, iy = np.asarray(ix), np.asarray(iy)
        inside = self._inside(ix, iy)
        v = self.tsd_cells[np.where(inside, iy, 0), np.where(inside, ix, 0)]
        return np.where(inside, self.conv.value_to_cost(v), self.conv.max_tsd).astype(F)


def _corners(g, x, y):
    """ComputeInterpolationDataPoints and index1 of InterpolatedTSDF2D at doubles (x, y)."""
    cx, cy = g.cell_index(x.astype(F), y.astype(F))
    lx, ly = g.cell_center(cx, cy)
    lx = np.where(lx.astype(np.float64) > x, (lx.astype(np.float64) - g.resolution).astype(F), lx)
    ly = np.where(ly.astype(np.float64) > y, (ly.astype(np.float64) - g.resolution).astype(F), ly)
    res = F(g.resolution)
    dx = (lx + res) - lx
    dy = (ly + res) - ly
    ix, iy = g.cell_index(lx, ly)
    return lx, ly, dx, dy, ix, iy


def _bilinear(c, q11, q12, q21, q22, x, xv, y, yv, jac):
    """InterpolateBilinear; jac: value and derivatives on dual numbers (xv, yv: [n, 3])."""
    x1, y1, dx, dy = c[:4]
    c12 = (q12 - q11).astype(np.float64)
    c22 = (q22 - q21).astype(np.float64)
    if not jac:
        nx = (x - x1.astype(np.float64)) / dx.astype(np.float64)
        ny = (y - y1.astype(np.float64)) / dy.astype(np.float64)
        q1 = c12 * ny + q11.astype(np.float64)
        q2 = c22 * ny + q21.astype(np.float64)
        return (q2 - q1) * nx + q1, None
    inx = 1.0 / dx.astype(np.float64)
    iny = 1.0 / dy.astype(np.float64)
    nx = (x - x1.astype(np.float64)) * inx
    ny = (y - y1.astype(np.float64)) * iny
    q1 = c12 * ny + q11.astype(np.float64)
    q2 = c22 * ny + q21.astype(np.float64)
    d = q2 - q1
    nxv = xv * inx[:, None]
    nyv = yv * iny[:, None]
    q1v = c12[:, None] * nyv
    q2v = c22[:, None] * nyv
    return d * nx + q1, (d[:, None] * nxv + (q2v - q1v) * nx[:, None]) + q1v


def interpolate(g, x, y, xv=None, yv=None):
    """InterpolatedTSDF2D::GetWeight and ::GetCorrespondenceCost at doubles (x, y); with xv,
    yv ([n, 3] derivatives of x, y) also their derivatives.  Returns (w, wv, cost, costv)."""
    x = np.atleast_1d(np.asarray(x, np.float64))
    y = np.atleast_1d(np.asarray(y, np.float64))
    jac = xv is not None
    c = _corners(g, x, y)
    ix, iy = c[4], c[5]
    w11, w12 = g.get_weight(ix, iy), g.get_weight(ix - 1, iy)
    w21, w22 = g.get_weight(ix, iy - 1), g.get_weight(ix - 1, iy - 1)
    w, wv = _bilinear(c, w11, w12, w21, w22, x, xv, y, yv, jac)
    q, qv = _bilinear(c, g.get_correspondence_cost(ix, iy), g.get_correspondence_cost(ix - 1, iy),
                      g.get_correspondence_cost(ix, iy - 1),
                      g.get_correspondence_cost(ix - 1, iy - 1), x, xv, y, yv, jac)
    known = (w11 != 0) & (w12 != 0) & (w21 != 0) & (w22 != 0)
    cost = np.where(known, q, np.float64(g.conv.max_tsd))
    costv = np.where(known[:, None], qv, 0.0) if jac else None
    return w, wv, cost, costv


def evaluate(g, xyz, pose, target_xy, target_angle, occupied_space_weight=20.0,
             translation_weight=10.0, rotation_weight=1.0, jacobian=True):
    """Residuals (n + 3), row-major Jacobian ((n + 3) x 3, or None) and validity of the three
    residual blocks of CeresScanMatcher2D::Match on a TSDF2D at `pose`."""
    xyz = np.asarray(xyz, F)
    n = len(xyz)
    px = xyz[:, 0].astype(np.float64)
    py = xyz[:, 1].astype(np.float64)
    cs, sn = math.cos(pose[2]), math.sin(pose[2])
    wx = (cs * px + (-sn) * py) + pose[0] * 1.0
    wy = (sn * px + cs * py) + pose[1] * 1.0
    xv = yv = None
    if jacobian:
        xv = np.zeros((n, 3))
        yv = np.zeros((n, 3))
        xv[:, 0] = 1.0
        xv[:, 2] = (-sn) * px + (-cs) * py
        yv[:, 1] = 1.0
        yv[:, 2] = cs * px + (-sn) * py
    w, wv, cost, costv = interpolate(g, wx, wy, xv, yv)
    scaling = occupied_space_weight / math.sqrt(float(n))
    ns = float(n) * scaling
    res = np.zeros(n + 3)
    jac = np.zeros((n + 3, 3)) if jacobian else None
    W = float(np.sum(w))
    valid = W != 0.0
    if valid:
        a = ns * cost
        if not jacobian:
            res[:n] = (a * w) / W
        else:
            inv = 1.0 / W
            Wv = wv.sum(axis=0)
            res[:n] = (a * w) * inv
            rv = a[:, None] * wv + (ns * costv) * w[:, None]
            jac[:n] = (rv - res[:n, None] * Wv[None, :]) * inv
    res[n] = translation_weight * (pose[0] - target_xy[0])
    res[n + 1] = translation_weight * (pose[1] - target_xy[1])
    res[n + 2] = rotation_weight * (pose[2] - target_angle)
    if jacobian:
        jac[n, 0] = translation_weight
        jac[n + 1, 1] = translation_weight
        jac[n + 2, 2] = rotation_weight
    return res, jac, valid


def _normal(g, xyz, x, target, target_angle, opts, with_jacobian, evaluator=None):
    r, j, valid = (evaluator or evaluate)(g, xyz, x, target, target_angle, opts[0], opts[1],
                                          opts[2], with_jacobian)
    if not valid:
        return None
    cost = 0.5 * float(np.dot(r, r))
    if not with_jacobian:
        return cost, None, None
    gr = j.T @ r
    h = j.T @ j
    return cost, gr, np.array([h[0, 0], h[0, 1], h[0, 2], h[1, 1], h[1, 2], h[2, 2]])


def _solve_spd3(a, b):
    if not a[0] > 0.0:
        return None
    l00 = math.sqrt(a[0])
    l10, l20 = a[1] / l00, a[2] / l00
    l11sq = a[3] - l10 * l10
    if not l11sq > 0.0:
        return None
    l11 = math.sqrt(l11sq)
    l21 = (a[4] - l20 * l10) / l11
    l22sq = a[5] - l20 * l20 - l21 * l21
    if not l22sq > 0.0:
        return None
    l22 = math.sqrt(l22sq)
    z0 = b[0] / l00
    z1 = (b[1] - l10 * z0) / l11
    z2 = (b[2] - l20 * z0 - l21 * z1) / l22
    y2 = z2 / l22
    y1 = (z1 - l21 * y2) / l11
    y0 = (z0 - l10 * y1 - l20 * y2) / l00
    y = [y0, y1, y2]
    return y if all(math.isfinite(v) for v in y) else None


def _norm3(v):
    return math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])


def match(g, xyz, target_xy, initial_pose, occupied_space_weight=20.0, translation_weight=10.0,
          rotation_weight=1.0, use_nonmonotonic_steps=True, max_num_iterations=10,
          evaluator=None, trace=None):
    """CeresScanMatcher2D::Match on a TSDF2D; the summary dict of pyoracle.ceres2d_match.
    `trace`: a list that receives one pyoracle.ceres_trace_record per pass of the loop.
    `evaluator` replaces the cost (same signature and return as evaluate()): the tests run
    this loop on the ProbabilityGrid cost of oracle/ to keep it equal to the C++ loop there."""
    opts = (occupied_space_weight, translation_weight, rotation_weight)
    k_min_radius, k_max_radius = 1e-32, 1e16
    max_nonmonotonic = 5 if use_nonmonotonic_steps else 0
    init = [float(v) for v in initial_pose]
    target = [float(target_xy[0]), float(target_xy[1])]
    target_angle = init[2]
    x = list(init)
    best = list(x)

    trial_failures = [0]   # trial points where the cost function failed (for the tests)

    def done(pose, initial_cost, final_cost, iterations, successful, termination):
        return dict(pose=np.array(pose, np.float64), initial_cost=initial_cost,
                    final_cost=final_cost, iterations=iterations,
                    num_successful_steps=successful, termination=CERES_TERMINATION[termination],
                    trial_failures=trial_failures[0])

    at_x = _normal(g, xyz, x, target, target_angle, opts, True, evaluator)
    if at_x is None:
        return done(init, -1.0, -1.0, 0, 0, 6)
    x_cost, gr, h = at_x
    x_norm = _norm3(x)
    initial_cost = minimum_cost = x_cost
    scale = [1.0 / (1.0 + math.sqrt(h[0])), 1.0 / (1.0 + math.sqrt(h[3])),
             1.0 / (1.0 + math.sqrt(h[5]))]
    radius, decrease_factor = 1e4, 2.0
    reuse_diagonal = False
    diagonal = [0.0, 0.0, 0.0]
    current_cost = reference_cost = candidate_cost_ev = ev_minimum_cost = x_cost
    acc_reference = acc_candidate = 0.0
    num_nonmonotonic = num_invalid = iteration = successful = 0
    last_step_successful = False
    termination = 0
    while True:
        if last_step_successful:
            successful += 1
            if x_cost < minimum_cost:
                minimum_cost = x_cost
                best = list(x)
            last_step_successful = False
        gmax = max(abs(gr[0]), max(abs(gr[1]), abs(gr[2])))
        rec = dict(x_cost=x_cost, gradient_max_norm=gmax, radius_before=radius,
                   reused_diagonal=reuse_diagonal)

        def record(outcome, **more):
            if trace is not None:
                trace.append(ceres_trace_record(outcome, radius_after=radius, **rec, **more))
        if iteration >= max_num_iterations:
            termination = 0
            record("LOOP_EXIT")
            break
        if gmax <= 1e-10:
            termination = 2
            record("LOOP_EXIT")
            break
        if radius <= k_min_radius:
            termination = 4
            record("LOOP_EXIT")
            break
        iteration += 1
        hs = [h[0] * scale[0] * scale[0], h[1] * scale[0] * scale[1], h[2] * scale[0] * scale[2],
              h[3] * scale[1] * scale[1], h[4] * scale[1] * scale[2], h[5] * scale[2] * scale[2]]
        gs = [gr[0] * scale[0], gr[1] * scale[1], gr[2] * scale[2]]
        if not reuse_diagonal:
            diagonal = [min(max(hs[0], 1e-6), 1e32), min(max(hs[3], 1e-6), 1e32),
                        min(max(hs[5], 1e-6), 1e32)]
        a = [hs[0] + diagonal[0] / radius, hs[1], hs[2], hs[3] + diagonal[1] / radius, hs[4],
             hs[5] + diagonal[2] / radius]
        y = _solve_spd3(a, gs)
        reuse_diagonal = True
        valid = y is not None
        if valid:
            step = [-y[0], -y[1], -y[2]]
            hs_step = [hs[0] * step[0] + hs[1] * step[1] + hs[2] * step[2],
                       hs[1] * step[0] + hs[3] * step[1] + hs[4] * step[2],
                       hs[2] * step[0] + hs[4] * step[1] + hs[5] * step[2]]
            model_cost_change = -((step[0] * gs[0] + step[1] * gs[1] + step[2] * gs[2]) +
                                  0.5 * (step[0] * hs_step[0] + step[1] * hs_step[1] +
                                         step[2] * hs_step[2]))
            valid = not (model_cost_change < 0.0)
        if not valid:
            num_invalid += 1
            if num_invalid >= 5:
                termination = 5
                record("INVALID")
                break
            radius = radius / decrease_factor
            decrease_factor *= 2.0
            reuse_diagonal = False
            record("INVALID")
            continue
        num_invalid = 0
        cand = [x[0] + step[0] * scale[0], x[1] + step[1] * scale[1], x[2] + step[2] * scale[2]]
        at_cand = _normal(g, xyz, cand, target, target_angle, opts, False, evaluator)
        candidate_cost = DBL_MAX if at_cand is None else at_cand[0]
        trial_failures[0] += at_cand is None
        diff = [x[0] - cand[0], x[1] - cand[1], x[2] - cand[2]]
        rec.update(candidate_cost=candidate_cost, model_cost_change=model_cost_change,
                   step_norm=_norm3(diff), step_norm_threshold=1e-8 * (x_norm + 1e-8))
        if _norm3(diff) <= 1e-8 * (x_norm + 1e-8):
            termination = 3
            record("PARAMETER_TOLERANCE")
            break
        rec.update(cost_change=abs(x_cost - candidate_cost), cost_change_threshold=1e-6 * x_cost)
        if abs(x_cost - candidate_cost) <= 1e-6 * x_cost:
            termination = 1
            record("FUNCTION_TOLERANCE")
            break
        relative_decrease = (current_cost - candidate_cost) / model_cost_change
        historical_decrease = (reference_cost - candidate_cost) / (acc_reference + model_cost_change)
        step_quality = max(relative_decrease, historical_decrease)
        rec.update(step_quality=step_quality)
        if step_quality > 1e-3:
            x = cand
            x_norm = _norm3(x)
            t = 2.0 * step_quality - 1.0
            radius = min(k_max_radius, radius / max(1.0 / 3.0, 1.0 - t * t * t))
            decrease_factor = 2.0
            reuse_diagonal = False
            current_cost = candidate_cost
            rec.update(evaluator_minimum_cost=ev_minimum_cost,
                       evaluator_candidate_cost=candidate_cost_ev)
            acc_candidate += model_cost_change
            acc_reference += model_cost_change
            if current_cost < ev_minimum_cost:
                ev_minimum_cost = current_cost
                num_nonmonotonic = 0
                candidate_cost_ev = current_cost
                acc_candidate = 0.0
            else:
                num_nonmonotonic += 1
                if current_cost > candidate_cost_ev:
                    candidate_cost_ev = current_cost
                    acc_candidate = 0.0
            if num_nonmonotonic == max_nonmonotonic:
                reference_cost = candidate_cost_ev
                acc_reference = acc_candidate
                rec.update(reference_switched=True)
            record("ACCEPTED")
            at_x = _normal(g, xyz, x, target, target_angle, opts, True, evaluator)
            if at_x is None:   # FAILURE: the parameters keep the initial estimate
                return done(init, initial_cost, initial_cost, iteration, successful, 6)
            x_cost, gr, h = at_x
            last_step_successful = True
        else:
            radius = radius / decrease_factor
            decrease_factor *= 2.0
            reuse_diagonal = True
            record("REJECTED")
    return done(best, initial_cost, minimum_cost, iteration, successful, termination)
