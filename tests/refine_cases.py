"""Case tables of the refinement edge tests — TEST INFRASTRUCTURE ONLY.

One copy of the problems that tests/test_gpu_refine_kernels.py runs on the device and
tests/test_refine_branches_cpu.py runs through the traced oracles and the CPU emulation of
trust_region.cuh: noise grids, a large initial offset and small prior weights, which make
the quadratic model poor and so reach the minimiser's rejections, rising accepted costs and
reference-cost switches.  Every problem is generated from a seed; every solver case names the
branches its trace must show (BRANCHES) and is checked for its distance from every threshold
the minimiser decides on (assert_margins)."""
import math

import numpy as np

MARGIN = 1e-6          # relative distance every deciding quantity keeps from its threshold
MIN_RELATIVE_DECREASE = 1e-3
GRADIENT_TOLERANCE = 1e-10
K_PADDING = (2 ** 31 - 1) // 4


# ---- what a trace shows -------------------------------------------------------------------
def outcomes(trace):
    """One letter per pass: A(ccepted) R(ejected) I(nvalid) P F (tolerance stops) L(oop exit)."""
    return "".join(t["outcome"][0] for t in trace)


def _accepted(trace):
    return [t for t in trace if t["outcome"] == "ACCEPTED"]


BRANCHES = {
    # a rejected step: the next pass keeps the damping diagonal and the radius is halved
    "rejected": lambda r: any(
        a["outcome"] == "REJECTED" and b["reused_diagonal"]
        and a["radius_after"] == a["radius_before"] / 2.0
        for a, b in zip(r["trace"], r["trace"][1:])),
    # rejections in a row: decrease_factor doubles, so the second divides the radius by 4
    "two_rejections": lambda r: any(
        a["outcome"] == b["outcome"] == "REJECTED"
        and b["radius_after"] == b["radius_before"] / 4.0
        for a, b in zip(r["trace"], r["trace"][1:])),
    "three_rejections": lambda r: "RRR" in outcomes(r["trace"]),
    # an accepted step whose cost is above the cost it left (non-monotonic steps)
    "accepted_rising": lambda r: any(t["candidate_cost"] > t["x_cost"] for t in _accepted(r["trace"])),
    # the reference cost replaced after max_consecutive_nonmonotonic_steps = 5 accepted steps
    # that did not improve the minimum
    "reference_switch": lambda r: any(
        t["reference_switched"] and t["candidate_cost"] > t["x_cost"] for t in _accepted(r["trace"])),
    # the returned iterate is not the last one accepted
    "best_not_last": lambda r: bool(_accepted(r["trace"])) and
    r["final_cost"] < _accepted(r["trace"])[-1]["candidate_cost"] * (1.0 - 1e-9),
    "max_iterations": lambda r: r["termination"] == "NO_CONVERGENCE"
    and r["trace"][-1]["outcome"] == "LOOP_EXIT" and r["iterations"] >= 1,
    "gradient_at_start": lambda r: r["termination"] == "GRADIENT_TOLERANCE"
    and r["iterations"] == 0 and outcomes(r["trace"]) == "L",
    "function_tolerance": lambda r: r["termination"] == "FUNCTION_TOLERANCE"
    and r["trace"][-1]["outcome"] == "FUNCTION_TOLERANCE",
    "parameter_tolerance": lambda r: r["termination"] == "PARAMETER_TOLERANCE"
    and r["trace"][-1]["outcome"] == "PARAMETER_TOLERANCE",
    # TSDF: a trial point that sees no weight costs DBL_MAX and is rejected
    "trial_failure": lambda r: r.get("trial_failures", 0) >= 1 and any(
        t["outcome"] == "REJECTED" and t["candidate_cost"] > 1e300 for t in r["trace"]),
}


def _apart(value, threshold):
    return abs(value - threshold) >= MARGIN * max(abs(value), abs(threshold))


def assert_margins(result):
    """Every quantity the minimiser compared with a threshold is at least MARGIN (relative)
    away from it, so that the device's tree-ordered sums and its cos / sin cannot flip the
    decision."""
    for k, t in enumerate(result["trace"]):
        where = (k, t["outcome"])
        assert _apart(t["gradient_max_norm"], GRADIENT_TOLERANCE), where
        if not math.isnan(t["step_norm"]):
            assert _apart(t["step_norm"], t["step_norm_threshold"]), where
        if not math.isnan(t["cost_change"]):
            assert _apart(t["cost_change"], t["cost_change_threshold"]), where
        if not math.isnan(t["step_quality"]):
            assert _apart(t["step_quality"], MIN_RELATIVE_DECREASE), where
        if t["outcome"] == "ACCEPTED":
            # the step evaluator's comparisons: a cost below its minimum resets the count of
            # non-monotonic steps (and so moves the reference switch); a cost that is not
            # below it is compared with the evaluator's candidate cost
            assert _apart(t["candidate_cost"], t["evaluator_minimum_cost"]), where
            if not t["candidate_cost"] < t["evaluator_minimum_cost"]:
                assert _apart(t["candidate_cost"], t["evaluator_candidate_cost"]), where
            assert _apart(t["candidate_cost"], t["x_cost"]), where


def assert_reaches(result, branches):
    for b in branches:
        assert BRANCHES[b](result), (b, outcomes(result["trace"]), result["termination"])
    assert_margins(result)


# ---- 2D ProbabilityGrid problems --------------------------------------------------------------
def noise_cells(rng, ny, nx):
    return rng.randint(1, 32768, size=(ny, nx)).astype(np.uint16)


def problem2d(seed, n=60, size=40):
    """(cells, resolution, max_x, max_y, cloud, target_xy, initial_pose)."""
    rng = np.random.RandomState(seed)
    cells = noise_cells(rng, size, size)
    cloud = np.concatenate([rng.uniform(-0.6, 0.6, (n, 2)), np.zeros((n, 1))], 1).astype(np.float32)
    init = np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4), rng.uniform(-1, 1)])
    return cells, 0.05, size * 0.025, size * 0.025, cloud, init[:2] * 0.5, init


def far_cloud2d(n):
    """Points a grid-width outside problem2d's grid: constant residuals, a zero Jacobian."""
    k = np.arange(n, dtype=np.float64)
    return np.stack([5.0 + 0.01 * k, -7.0 - 0.02 * k, np.zeros(n)], 1).astype(np.float32)


WEAK_PRIOR = dict(occupied_space_weight=20.0, translation_weight=1e-2, rotation_weight=1e-2)

# (name, problem seed, options, the branches the trace must show)
SOLVES_2D = [
    ("rejections_rising_switch_best", 3, dict(WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=50),
     ["rejected", "two_rejections", "three_rejections", "accepted_rising", "reference_switch",
      "best_not_last", "function_tolerance"]),
    ("eight_rejections", 0, dict(WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=50),
     ["rejected", "two_rejections", "three_rejections", "accepted_rising", "reference_switch"]),
    ("rejected_first", 31, dict(WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=50),
     ["rejected", "two_rejections", "accepted_rising", "best_not_last"]),
    ("fifty_iterations", 13, dict(WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=50),
     ["accepted_rising", "reference_switch", "max_iterations"]),
    ("monotonic_rejections", 1, dict(WEAK_PRIOR, use_nonmonotonic_steps=False, max_num_iterations=50),
     ["rejected", "two_rejections", "three_rejections", "function_tolerance"]),
    ("monotonic_rejected_first", 2, dict(WEAK_PRIOR, use_nonmonotonic_steps=False, max_num_iterations=50),
     ["rejected", "two_rejections", "three_rejections"]),
    ("one_iteration", 3, dict(WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=1),
     ["max_iterations"]),
    # the unconstrained solve of seed 3 takes 20 iterations: a limit of 20 changes nothing but
    # the exit that is taken first, a limit of 19 stops one short
    ("limit_equal", 3, dict(WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=20),
     ["rejected", "best_not_last", "function_tolerance"]),
    ("limit_one_less", 3, dict(WEAK_PRIOR, use_nonmonotonic_steps=True, max_num_iterations=19),
     ["rejected", "best_not_last", "max_iterations"]),
]


# ---- TSDF2D problems --------------------------------------------------------------------------
def problem_tsdf(seed, n=60, size=40, hole=0.0):
    """(tsd cells, weight cells, resolution, max_x, max_y, truncation, max_weight, cloud,
    target_xy, initial_pose).  hole: the fraction of the grid's border cells without weight,
    which trial steps can land in."""
    rng = np.random.RandomState(seed)
    tsd = noise_cells(rng, size, size)
    wgt = noise_cells(rng, size, size)
    if hole > 0.0:
        m = int(size * hole)
        keep = np.zeros((size, size), bool)
        keep[m:size - m, m:size - m] = True
        wgt[~keep] = 0
        tsd[~keep] = 0
    spread = 0.6 if hole == 0.0 else 0.12
    cloud = np.concatenate([rng.uniform(-spread, spread, (n, 2)), np.zeros((n, 1))], 1).astype(np.float32)
    off = 0.3 if hole == 0.0 else 0.1
    init = np.array([rng.uniform(-off, off), rng.uniform(-off, off), rng.uniform(-1, 1)])
    return tsd, wgt, 0.05, size * 0.025, size * 0.025, 0.3, 10.0, cloud, init[:2] * 0.5, init


# ---- 3D problems ------------------------------------------------------------------------------
def problem3d(seed, n_hi=70, n_lo=0, size=10):
    """(resolution, indices, values, high cloud, low cloud or None, target, initial pose): a
    dense size^3 box of noise voxels around the origin."""
    rng = np.random.RandomState(seed)
    lo = -(size // 2)
    ax = np.arange(lo, lo + size)
    idx = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)
    val = rng.randint(1, 32768, size=len(idx)).astype(np.uint16)
    res = 0.1
    hi = rng.uniform(-0.35, 0.35, (n_hi, 3)).astype(np.float32)
    low = rng.uniform(-0.35, 0.35, (n_lo, 3)).astype(np.float32) if n_lo else None
    a = rng.uniform(-0.4, 0.4)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    t = rng.uniform(-0.15, 0.15, 3)
    init = np.concatenate([t, [math.cos(a / 2)], math.sin(a / 2) * axis])
    return res, idx, val, hi, low, t * 0.5, init


WEAK_PRIOR_3D = dict(translation_weight=1e-2, rotation_weight=1e-2)


def edge_cells(rng, ny, nx):
    """Noise with the values the cost conversion branches on: unknown (0), the smallest and
    largest values and cells that carry the update marker (32768 = marked unknown, 65535)."""
    cells = noise_cells(rng, ny, nx)
    special = np.array([0, 1, 32767, 32768, 65535, 32768 + 12345], np.uint16)
    flat = cells.reshape(-1)
    where = rng.permutation(flat.size)[:max(1, flat.size // 2)]
    flat[where] = special[np.arange(len(where)) % len(special)]
    return cells


# ---- solver case tables of the other three instantiations ---------------------------------------
# (name, seed, hole, nonmonotonic, max iterations, branches)
SOLVES_TSDF = [
    ("rejections_switch_best_not_last", 5, 0.3, True, 50,
     ["rejected", "two_rejections", "three_rejections", "accepted_rising", "reference_switch",
      "best_not_last", "max_iterations"]),
    ("monotonic_rejections", 3, 0.0, False, 50,
     ["rejected", "two_rejections", "three_rejections", "function_tolerance"]),
    ("function_tolerance", 0, 0.0, True, 50, ["function_tolerance"]),
    ("one_iteration", 5, 0.3, True, 1, ["max_iterations"]),
]
# A solve that must NOT be used as a parity case, kept to show that assert_margins refuses it:
# it falls into an exact 2-cycle whose lower cost converges to the last bit, so the step
# evaluator's `cost < minimum` (which resets the non-monotonic count and so places the
# reference switch) is decided by rounding, and two correct implementations that sum in a
# different order take different branches from there (poses 1.6e-5 apart after 50 iterations).
TSDF_DECIDED_BY_ROUNDING = ("two_cycle", 8, 0.0, True, 50, [])


def tsdf_want(case):
    """(oracle TSDF2D, problem, traced oracle result) of a SOLVES_TSDF entry."""
    from tests import tsdf2d_oracle as T
    name, seed, hole, nonmono, iters, branches = case
    p = problem_tsdf(seed, hole=hole)
    g = T.TSDF2D(p[0].shape[1], p[0].shape[0], p[2], p[3], p[4], p[5], p[6], p[0], p[1])
    trace = []
    want = T.match(g, p[7], p[8], p[9], 20.0, 1e-2, 1e-2, nonmono, iters, trace=trace)
    want["trace"] = trace
    return g, p, want


# (name, seed, low-resolution points, nonmonotonic, max iterations, branches)
SOLVES_3D = [
    ("rejections_switch", 1, 0, True, 50,
     ["rejected", "two_rejections", "three_rejections", "accepted_rising", "reference_switch"]),
    ("best_not_last_fifty", 5, 0, True, 50,
     ["accepted_rising", "reference_switch", "best_not_last", "max_iterations"]),
    ("rejected_first", 7, 0, True, 50, ["rejected", "two_rejections", "accepted_rising"]),
    ("monotonic", 4, 0, False, 50, ["rejected", "two_rejections", "three_rejections"]),
    ("two_clouds", 0, 33, True, 50,
     ["rejected", "two_rejections", "accepted_rising", "reference_switch", "function_tolerance"]),
    ("two_clouds_monotonic", 5, 33, False, 50, ["rejected", "three_rejections"]),
    ("one_iteration", 1, 0, True, 1, ["max_iterations"]),
]


def want3d(oracle, case):
    """(problem, traced oracle result) of a SOLVES_3D entry; oracle = oracle.pyoracle."""
    name, seed, n_lo, nonmono, iters, branches = case
    res, idx, val, hi, low, tgt, init = problem3d(seed, n_lo=n_lo)
    grid = oracle.HybridGrid(res, idx, val)
    pairs = [(hi, grid)] + ([(low, grid)] if n_lo else [])
    want = oracle.ceres3d_match(pairs, tgt, init, occupied_space_weights=(5.0, 30.0),
                                use_nonmonotonic_steps=nonmono, max_num_iterations=iters,
                                trace=True, **WEAK_PRIOR_3D)
    return (res, idx, val, hi, low, tgt, init), want


def problem_intensity(seed, n=40):
    """problem3d plus (sums, counts, intensities): a noise intensity grid over the same voxels
    and returns on both sides of the threshold 100."""
    res, idx, val, hi, _, tgt, init = problem3d(seed, n_hi=n)
    rng = np.random.RandomState(1000 + seed)
    sums = rng.uniform(10, 90, len(idx)).astype(np.float32)
    counts = np.ones(len(idx), np.int32)
    inten = rng.uniform(10, 120, n).astype(np.float32)
    return res, idx, val, hi, tgt, init, sums, counts, inten


INTENSITY_THRESHOLD = 100.0
# (name, seed, intensity weight, huber scale, prior weight, nonmonotonic, max iterations,
# branches); huber scale 0.05 puts the block's s_b above huber^2 (the square-root branch of
# HuberLoss), 50 below it (the identity branch)
SOLVES_INTENSITY = [
    ("rejections_switch_small_huber", 1, 0.5, 0.05, 1e-2, True, 40,
     ["rejected", "two_rejections", "three_rejections", "accepted_rising", "reference_switch",
      "function_tolerance"]),
    ("best_not_last_large_huber", 4, 0.5, 50.0, 1e-2, True, 40,
     ["rejected", "two_rejections", "accepted_rising", "reference_switch", "best_not_last",
      "max_iterations"]),
    ("monotonic", 3, 0.5, 50.0, 1e-2, False, 40,
     ["rejected", "two_rejections", "three_rejections", "function_tolerance"]),
    ("one_iteration", 1, 0.5, 0.05, 1e-2, True, 1, ["max_iterations"]),
    ("function_tolerance_stiff", 2, 0.5, 0.3, 1e2, True, 30, ["function_tolerance"]),
    ("parameter_tolerance_stiff", 2, 0.5, 0.3, 1e6, True, 30, ["parameter_tolerance"]),
]


def want_intensity(oracle, case):
    """(problem, traced oracle result) of a SOLVES_INTENSITY entry: (name, seed, intensity
    weight, huber scale, prior weight, nonmonotonic, max iterations, branches)."""
    from tests import intensity3d_oracle as iorc
    name, seed, weight, huber, prior, nonmono, iters, branches = case
    p = problem_intensity(seed)
    res, idx, val, hi, tgt, init, sums, counts, inten = p
    trace = []
    want = iorc.match([(hi, oracle.HybridGrid(res, idx, val),
                        iorc.IntensityHybridGrid(res, idx, sums, counts), inten)], tgt, init,
                      [(weight, huber, INTENSITY_THRESHOLD)], translation_weight=prior,
                      rotation_weight=prior, use_nonmonotonic_steps=nonmono,
                      max_num_iterations=iters, trace=trace)
    want["trace"] = trace
    return p, want
