"""CPU restatement of CeresScanMatcher3D with intensity blocks — TEST INFRASTRUCTURE ONLY.

What is restated (the product's device code is checked against this, never the reverse):
  * IntensityHybridGrid (mapping/3d/hybrid_grid.h:547-570): AddIntensity, and GetIntensity as
    the float mean sum / count, 0 where nothing was added;
  * InterpolatedGrid<IntensityHybridGrid> (interpolated_grid.h:49-157): the float
    CenterOfLowerVoxel and the smoothstep on plain doubles or on dual numbers over (x, y, z),
    in the operation order of oracle/oracle_ceres3d.cc's InterpolatedProbability;
  * IntensityCostFunction3D (intensity_cost_function_3d.h:67-80) with the scaling
    weight / sqrt(n) of ceres_scan_matcher_3d.cc:128-139: residual and tangent-space row per
    point, 0 and a zero row for returns brighter than the threshold;
  * ceres::HuberLoss (ceres/loss_function.cc, HuberLoss::Evaluate) applied per residual block
    the way Ceres' Corrector (ceres/corrector.cc) applies it in its alpha = 0 branch, the only
    one HuberLoss reaches: the block adds rho(s_b) / 2 to the cost, rho'(s_b) J^T r to the
    gradient and rho'(s_b) J^T J to the Gauss-Newton Hessian;
  * the trust-region loop of oracle/oracle_ceres3d.cc (CeresMatch3D, the same restatement of
    Ceres' published minimiser and the same caveat) on those normal equations.
The occupied-space and prior residuals come from the C++ oracle (pyoracle.ceres3d_evaluate),
unchanged.  Sums over points are numpy's, not the device's block-tree order: parity with the
device is to the tolerances of the tests, not bit for bit.
"""
import math
import sys

import numpy as np

from oracle import pyoracle

F = np.float32
DBL_MIN = sys.float_info.min
CERES_TERMINATION = pyoracle.CERES_TERMINATION


def lround(v):
    """std::lround (halves away from zero), elementwise."""
    v = np.asarray(v, np.float64)
    t = np.trunc(v)
    return (t + np.where(np.abs(v - t) >= 0.5, np.sign(v), 0.0)).astype(np.int64)


def cell_index(resolution, p):
    """HybridGridBase::GetCellIndex (hybrid_grid.h:428-433) of float points."""
    return lround(np.asarray(p, F) / F(resolution))


class IntensityHybridGrid:
    """IntensityHybridGrid from the flat form of HybridGridBase<AverageIntensityData>:
    indices (n x 3), sums (n float32), counts (n int32)."""

    def __init__(self, resolution, indices=(), sums=(), counts=()):
        self.resolution = float(F(resolution))
        self.cells = {}
        for i, s, c in zip(np.asarray(indices, np.int64).reshape(-1, 3),
                           np.asarray(sums, F).reshape(-1), np.asarray(counts, np.int64)):
            self.cells[tuple(int(v) for v in i)] = (F(s), int(c))
        self._box = None

    def add_intensity(self, index, intensity):
        key = tuple(int(v) for v in index)
        s, c = self.cells.get(key, (F(0), 0))
        self.cells[key] = (F(s + F(intensity)), c + 1)
        self._box = None

    def get_intensity(self, x, y, z):
        s, c = self.cells.get((int(x), int(y), int(z)), (F(0), 0))
        return float(F(0) if c == 0 else F(s / F(c)))

    def _values(self, ix, iy, iz):
        """GetIntensity at integer index arrays, as doubles."""
        if self._box is None:
            if self.cells:
                idx = np.array(list(self.cells), np.int64)
                lo, hi = idx.min(0), idx.max(0)
                box = np.zeros(tuple(hi - lo + 1), F)
                for (k, (s, c)) in self.cells.items():
                    box[k[0] - lo[0], k[1] - lo[1], k[2] - lo[2]] = F(0) if c == 0 else F(s / F(c))
                self._box = (lo, box)
            else:
                self._box = (np.zeros(3, np.int64), np.zeros((0, 0, 0), F))
        lo, box = self._box
        jx, jy, jz = ix - lo[0], iy - lo[1], iz - lo[2]
        inside = ((jx >= 0) & (jx < box.shape[0]) & (jy >= 0) & (jy < box.shape[1]) &
                  (jz >= 0) & (jz < box.shape[2]))
        out = np.zeros(len(ix), np.float64)
        out[inside] = box[jx[inside], jy[inside], jz[inside]]
        return out


# ---- dual numbers over (x, y, z) with ceres/jet.h's arithmetic, on arrays of points -------
def _mul(f, g):
    return (f[0] * g[0], f[0] * g[1] + f[1] * g[0], f[0] * g[2] + f[2] * g[0],
            f[0] * g[3] + f[3] * g[0])


def _scale(f, s):
    return (f[0] * s, f[1] * s, f[2] * s, f[3] * s)


def _add(f, g):
    return tuple(a + b for a, b in zip(f, g))


def _sub(f, g):
    return tuple(a - b for a, b in zip(f, g))


def _adds(f, s):
    return (f[0] + s, f[1], f[2], f[3])


def interpolate(grid, x, y, z, dual):
    """InterpolatedGrid<IntensityHybridGrid>::GetInterpolatedValue at arrays (x, y, z): the
    value and (dual) its derivative by (x, y, z) as a 4-tuple of arrays."""
    res = F(grid.resolution)
    corner, nodes = [], []
    for w in (x, y, z):
        w = np.asarray(w, np.float64)
        c = (lround(w.astype(F) / res).astype(F) * res).astype(F)   # CenterOfLowerVoxel
        c = np.where(c.astype(np.float64) > w, (c - res).astype(F), c)
        w1, w2 = c.astype(np.float64), (c + res).astype(F).astype(np.float64)
        corner.append(lround(c / res))
        zero = np.zeros_like(w)
        if dual:
            inv = 1.0 / (w2 - w1)
            nodes.append([(w - w1) * inv, inv])
        else:
            nodes.append([(w - w1) / (w2 - w1), zero])
    z0 = np.zeros_like(np.asarray(x, np.float64))
    nx = (nodes[0][0], 1.0 * nodes[0][1], 0.0 * nodes[0][1], 0.0 * nodes[0][1]) if dual else \
        (nodes[0][0], z0, z0, z0)
    ny = (nodes[1][0], 0.0 * nodes[1][1], 1.0 * nodes[1][1], 0.0 * nodes[1][1]) if dual else \
        (nodes[1][0], z0, z0, z0)
    nz = (nodes[2][0], 0.0 * nodes[2][1], 0.0 * nodes[2][1], 1.0 * nodes[2][1]) if dual else \
        (nodes[2][0], z0, z0, z0)
    i, j, k = corner

    def q(dx, dy, dz):
        return grid._values(i + dx, j + dy, k + dz)
    q111, q112, q121, q122 = q(0, 0, 0), q(0, 0, 1), q(0, 1, 0), q(0, 1, 1)
    q211, q212, q221, q222 = q(1, 0, 0), q(1, 0, 1), q(1, 1, 0), q(1, 1, 1)
    nxx, nyy, nzz = _mul(nx, nx), _mul(ny, ny), _mul(nz, nz)
    nxxx, nyyy, nzzz = _mul(nx, nxx), _mul(ny, nyy), _mul(nz, nzz)

    def blend_z(qa, qb):   # (qa - qb) * n^3 * 2. + (qb - qa) * n^2 * 3. + qa
        return _adds(_add(_scale(_scale(nzzz, qa - qb), 2.), _scale(_scale(nzz, qb - qa), 3.)), qa)
    q11, q12 = blend_z(q111, q112), blend_z(q121, q122)
    q21, q22 = blend_z(q211, q212), blend_z(q221, q222)

    def blend(qa, qb, n3, n2):
        return _add(_add(_scale(_mul(_sub(qa, qb), n3), 2.), _scale(_mul(_sub(qb, qa), n2), 3.)), qa)
    q1, q2 = blend(q11, q12, nyyy, nyy), blend(q21, q22, nyyy, nyy)
    return blend(q1, q2, nxxx, nxx)


def interpolated_intensity(grid, x, y, z, gradient=False):
    f = interpolate(grid, np.array([x]), np.array([y]), np.array([z]), gradient)
    if gradient:
        return float(f[0][0]), np.array([f[1][0], f[2][0], f[3][0]])
    return float(f[0][0])


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _plus_jacobian(q):
    """ceres::QuaternionParameterization::ComputeJacobian (4 x 3, row-major)."""
    return [-q[1], -q[2], -q[3], q[0], q[3], -q[2], -q[3], q[0], q[1], q[2], -q[1], q[0]]


def intensity_rows(grid, xyz, intensities, pose, scaling, threshold, jacobian):
    """IntensityCostFunction3D's residuals and (jacobian) tangent-space rows at pose."""
    pose = [float(v) for v in pose]
    p = np.asarray(xyz, F).astype(np.float64)
    p = (p[:, 0], p[:, 1], p[:, 2])
    w, qv = pose[3], (pose[4], pose[5], pose[6])
    uv = _cross(qv, p)
    uv = tuple(u + u for u in uv)
    c = _cross(qv, uv)
    world = [((p[k] + w * uv[k]) + c[k]) + pose[k] for k in range(3)]
    f = interpolate(grid, world[0], world[1], world[2], jacobian)
    inten = np.asarray(intensities, F)
    skip = inten > F(threshold)
    res = scaling * (f[0] - inten.astype(np.float64))
    res[skip] = 0.0
    if not jacobian:
        return res, None
    g = f[1:]
    dworld = []
    for k in range(3):
        d = [0.0, 0.0, 0.0]
        d[k] = 1.0
        dworld.append(d)
    dworld.append(list(uv))
    for k in range(3):   # d world / d qv[k] = w * duv + e_k x uv + qv x duv
        e = [0.0, 0.0, 0.0]
        e[k] = 1.0
        duv = _cross(e, p)
        duv = tuple(u + u for u in duv)
        t1, t2 = _cross(e, uv), _cross(qv, duv)
        dworld.append([(w * duv[m] + t1[m]) + t2[m] for m in range(3)])
    ambient = [scaling * ((g[0] * d[0] + g[1] * d[1]) + g[2] * d[2]) for d in dworld]
    pj = _plus_jacobian(pose[3:])
    rows = np.zeros((len(res), 6))
    for k in range(3):
        rows[:, k] = ambient[k]
        rows[:, 3 + k] = (ambient[3] * pj[k] + ambient[4] * pj[3 + k] + ambient[5] * pj[6 + k] +
                          ambient[6] * pj[9 + k])
    rows[skip] = 0.0
    return res, rows


def _split(entries):
    pairs = [(e[0], e[1]) for e in entries]
    blocks = [(e[2], e[3]) if len(e) > 2 and e[2] is not None else None for e in entries]
    return pairs, blocks


def evaluate(entries, pose, target_translation, target_rotation, intensity_options,
             occupied_space_weights=(5.0, 30.0), translation_weight=10.0, rotation_weight=1.0,
             jacobian=True):
    """entries = [(xyz, pyoracle.HybridGrid) or (xyz, HybridGrid, IntensityHybridGrid | None,
    intensities)]; intensity_options[b] = (weight, huber_scale, intensity_threshold).  All
    residuals in the problem's block order — per entry its occupied-space residuals, then its
    intensity residuals where it has a grid; then 3 translation and 3 rotation residuals —
    uncorrected by the loss, and (jacobian) the rows x 6 tangent-space Jacobian."""
    pairs, blocks = _split(entries)
    r0, j0 = pyoracle.ceres3d_evaluate(pairs, pose, target_translation, target_rotation,
                                       occupied_space_weights, translation_weight,
                                       rotation_weight, jacobian=jacobian)
    rs, js, row = [], [], 0
    for b, (xyz, _) in enumerate(pairs):
        n = len(xyz)
        rs.append(r0[row:row + n])
        js.append(j0[row:row + n] if jacobian else None)
        row += n
        if blocks[b] is None:
            continue
        grid, inten = blocks[b]
        weight, _, threshold = intensity_options[b]
        r, j = intensity_rows(grid, xyz, inten, pose, weight / math.sqrt(float(n)), threshold,
                              jacobian)
        rs.append(r)
        js.append(j)
    rs.append(r0[row:])
    js.append(j0[row:] if jacobian else None)
    return np.concatenate(rs), (np.concatenate(js) if jacobian else None)


def huber(a, s):
    """ceres::HuberLoss(a)::Evaluate: (rho(s), rho'(s))."""
    b = a * a
    if s > b:
        r = math.sqrt(s)
        return 2.0 * a * r - b, max(DBL_MIN, a / r)
    return s, 1.0


TRI = [(a, c) for a in range(6) for c in range(a, 6)]


def _block_normal(r, j):
    if j is None:
        return float(np.sum(r * r)), None, None
    return (float(np.sum(r * r)), np.array([np.sum(j[:, a] * r) for a in range(6)]),
            np.array([np.sum(j[:, a] * j[:, c]) for a, c in TRI]))


def normal(entries, pose, target_translation, target_rotation, intensity_options,
           occupied_space_weights=(5.0, 30.0), translation_weight=10.0, rotation_weight=1.0,
           jacobian=True):
    """(cost, g[6], upper triangle of H[21]) the minimiser consumes at pose, each intensity
    block corrected by its HuberLoss."""
    pairs, blocks = _split(entries)
    r, j = evaluate(entries, pose, target_translation, target_rotation, intensity_options,
                    occupied_space_weights, translation_weight, rotation_weight, jacobian)
    plain = np.ones(len(r), bool)
    row, corrected = 0, []
    for b, (xyz, _) in enumerate(pairs):
        row += len(xyz)
        if blocks[b] is not None:
            plain[row:row + len(xyz)] = False
            corrected.append((b, row, row + len(xyz)))
            row += len(xyz)
    sq, g, h = _block_normal(r[plain], j[plain] if jacobian else None)
    for b, lo, hi in corrected:
        sb, gb, hb = _block_normal(r[lo:hi], j[lo:hi] if jacobian else None)
        rho, rho1 = huber(intensity_options[b][1], sb)
        sq += rho
        if jacobian:
            g = g + rho1 * gb
            h = h + rho1 * hb
    return 0.5 * sq, g, h


def plus(x, delta):
    """x (+) delta: QuaternionParameterization::Plus on the rotation block."""
    out = [x[k] + delta[k] for k in range(3)] + list(x[3:])
    d = delta[3:]
    nd = math.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    if nd > 0.0:
        s = math.sin(nd) / nd
        z = (math.cos(nd), s * d[0], s * d[1], s * d[2])
        w = x[3:]
        out[3:] = [z[0] * w[0] - z[1] * w[1] - z[2] * w[2] - z[3] * w[3],
                   z[0] * w[1] + z[1] * w[0] + z[2] * w[3] - z[3] * w[2],
                   z[0] * w[2] - z[1] * w[3] + z[2] * w[0] + z[3] * w[1],
                   z[0] * w[3] + z[1] * w[2] - z[2] * w[1] + z[3] * w[0]]
    return out


def _tri(a, c):
    return a * 6 - a * (a - 1) // 2 + (c - a) if a <= c else _tri(c, a)


def _solve_spd(am, b):
    l = [[0.0] * 6 for _ in range(6)]
    for i in range(6):
        for j in range(i + 1):
            s = am[_tri(j, i)]
            for k in range(j):
                s -= l[i][k] * l[j][k]
            if i == j:
                if not s > 0.0:
                    return None
                l[i][i] = math.sqrt(s)
            else:
                l[i][j] = s / l[j][j]
    z = [0.0] * 6
    for i in range(6):
        s = b[i]
        for k in range(i):
            s -= l[i][k] * z[k]
        z[i] = s / l[i][i]
    y = [0.0] * 6
    for i in range(5, -1, -1):
        s = z[i]
        for k in range(i + 1, 6):
            s -= l[k][i] * y[k]
        y[i] = s / l[i][i]
    return y if all(math.isfinite(v) for v in y) else None


def _norm(v):
    return math.sqrt(sum(x * x for x in v))


def match(entries, target_translation, initial_pose, intensity_options,
          occupied_space_weights=(5.0, 30.0), translation_weight=10.0, rotation_weight=1.0,
          use_nonmonotonic_steps=False, max_num_iterations=10):
    """CeresScanMatcher3D::Match with intensity blocks: oracle_ceres3d.cc's CeresMatch3D on the
    Huber-corrected normal equations -> dict(pose, initial_cost, final_cost, iterations, ...)."""
    k_initial_radius, k_max_radius, k_min_radius = 1e4, 1e16, 1e-32
    k_min_relative_decrease, k_min_diag, k_max_diag = 1e-3, 1e-6, 1e32
    k_max_invalid, k_ftol, k_gtol, k_ptol = 5, 1e-6, 1e-10, 1e-8
    max_nonmonotonic = 5 if use_nonmonotonic_steps else 0
    target_rotation = [float(v) for v in initial_pose[3:]]
    kw = dict(occupied_space_weights=occupied_space_weights,
              translation_weight=translation_weight, rotation_weight=rotation_weight)

    def ev(x, jac):
        return normal(entries, x, target_translation, target_rotation, intensity_options,
                      jacobian=jac, **kw)
    x = [float(v) for v in initial_pose]
    best = list(x)
    x_cost, gx, hx = ev(x, True)
    x_norm = _norm(x)
    initial_cost = minimum_cost = x_cost
    scale = [1.0 / (1.0 + math.sqrt(hx[_tri(a, a)])) for a in range(6)]
    radius, decrease_factor, reuse_diagonal = k_initial_radius, 2.0, False
    diagonal = [0.0] * 6
    current_cost = reference_cost = candidate_cost_ev = ev_minimum_cost = x_cost
    acc_reference = acc_candidate = 0.0
    num_nonmonotonic = num_invalid = iteration = successful = 0
    last_step_successful = False
    while True:
        if last_step_successful:
            successful += 1
            if x_cost < minimum_cost:
                minimum_cost, best = x_cost, list(x)
        if iteration >= max_num_iterations:
            termination = 0
            break
        moved = plus(x, [-v for v in gx])
        if max(abs(x[k] - moved[k]) for k in range(7)) <= k_gtol:
            termination = 2
            break
        if radius <= k_min_radius:
            termination = 4
            break
        iteration += 1
        last_step_successful = False
        gs = [gx[a] * scale[a] for a in range(6)]
        hs = [0.0] * 21
        for a in range(6):
            for c in range(a, 6):
                hs[_tri(a, c)] = hx[_tri(a, c)] * scale[a] * scale[c]
        if not reuse_diagonal:
            diagonal = [min(max(hs[_tri(a, a)], k_min_diag), k_max_diag) for a in range(6)]
        am = list(hs)
        for a in range(6):
            am[_tri(a, a)] = hs[_tri(a, a)] + diagonal[a] / radius
        y = _solve_spd(am, gs)
        reuse_diagonal = True
        valid = y is not None
        if valid:
            step = [-v for v in y]
            sg = shs = 0.0
            for a in range(6):
                sg += step[a] * gs[a]
                row = 0.0
                for c in range(6):
                    row += hs[_tri(a, c)] * step[c]
                shs += step[a] * row
            model_cost_change = -(sg + 0.5 * shs)
            valid = not model_cost_change < 0.0
        if not valid:
            num_invalid += 1
            if num_invalid >= k_max_invalid:
                termination = 5
                break
            radius /= decrease_factor
            decrease_factor *= 2.0
            reuse_diagonal = False
            continue
        num_invalid = 0
        cand = plus(x, [step[a] * scale[a] for a in range(6)])
        candidate_cost = ev(cand, False)[0]
        if _norm([x[k] - cand[k] for k in range(7)]) <= k_ptol * (x_norm + k_ptol):
            termination = 3
            break
        if abs(x_cost - candidate_cost) <= k_ftol * x_cost:
            termination = 1
            break
        relative_decrease = (current_cost - candidate_cost) / model_cost_change
        historical_decrease = (reference_cost - candidate_cost) / (acc_reference +
                                                                   model_cost_change)
        step_quality = max(relative_decrease, historical_decrease)
        if step_quality > k_min_relative_decrease:
            x = cand
            x_norm = _norm(x)
            x_cost, gx, hx = ev(x, True)
            last_step_successful = True
            t = 2.0 * step_quality - 1.0
            radius = min(k_max_radius, radius / max(1.0 / 3.0, 1.0 - t * t * t))
            decrease_factor, reuse_diagonal = 2.0, False
            current_cost = candidate_cost
            acc_candidate += model_cost_change
            acc_reference += model_cost_change
            if current_cost < ev_minimum_cost:
                ev_minimum_cost, num_nonmonotonic = current_cost, 0
                candidate_cost_ev, acc_candidate = current_cost, 0.0
            else:
                num_nonmonotonic += 1
                if current_cost > candidate_cost_ev:
                    candidate_cost_ev, acc_candidate = current_cost, 0.0
            if num_nonmonotonic == max_nonmonotonic:
                reference_cost, acc_reference = candidate_cost_ev, acc_candidate
        else:
            radius /= decrease_factor
            decrease_factor *= 2.0
            reuse_diagonal = True
    return dict(pose=np.array(best), initial_cost=initial_cost, final_cost=minimum_cost,
                iterations=iteration, num_successful_steps=successful,
                termination=CERES_TERMINATION[termination])
