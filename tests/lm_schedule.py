"""Step-by-step replay of the pose-graph Levenberg-Marquardt schedule (test support; importable
without a GPU).

solve.cu runs Ceres' TrustRegionMinimizer with the LevenbergMarquardtStrategy on the device
(lm_init_kernel, lm_build_kernel / lm_persist_kernel, lm_step_kernel, lm_decide_kernel,
lm_accept_kernel, and the host loop of vgx_graph_solve that runs one iteration ahead).  LM repairs a
wrong radius or a wrong step in its next iterations, so final poses cannot pin that schedule.  This
module restates it in float64, driven by an evaluation callback evaluate(x) -> (ok, cost, g, H) over
the full 4N parameter vector, with the state of LmState: radius, decrease_factor, reuse_diagonal, the
iteration-0 Jacobi scale and the clamped LM diagonal.  The linear algebra is solve_exact's
(lm_system, recover_step, backward_ratio, model_cost_change).

Every decision is recorded with its margin: the distance of the tested value from its threshold
over the uncertainty the value carries from rounding.  The replay's step solves the same system as
the device's Cholesky, but not bit for bit; a correct float64 solve is within kappa(A) gamma u of it
(the forward error that goes with the backward-error bound solve_exact checks).  That step error
moves the model cost change and the candidate cost by at most (|gs| + |Hs||y|) . |dy|; the costs
themselves carry cost_rtol.  A decision whose margin is <= 1 is ambiguous: another correct
implementation could take the other branch.  The radius follows the ratio rho through
radius / max(1/3, 1 - (2 rho - 1)^3), so the replayed radius carries a relative uncertainty eps_r,
and a backward-error check at that radius gains the term |diag / radius| eps_r |y|.

With `follow` (the device's iterates x_k and successful-step counts), the replay walks the device's
trajectory instead of its own: an accepted device step is recovered from x_{k-1} -> x_k and checked
against the LM system at the replayed radius, scale and diagonal; a rejected one must leave x
bit-unchanged, and the replay's own candidate, evaluated by the callback, must be rejected.
"""
import numpy as np
import scipy.linalg

import solve_exact as SX

U = SX.U
TWO_PI = 6.283185307179586476925286766559      # graph.h normalize_angle, as a float64

# vgx_solver_options_default / vgo_solver_options_default (pose_graph.cpp:91-97 over Ceres' defaults)
DEFAULTS = dict(max_num_iterations=50, parameter_tolerance=3e-3, function_tolerance=1e-6,
                gradient_tolerance=1e-10, initial_trust_region_radius=1e4, max_trust_region_radius=1e16,
                min_trust_region_radius=1e-32, min_relative_decrease=1e-3, min_lm_diagonal=1e-6,
                max_lm_diagonal=1e32, max_solver_time_s=4.0, jacobi_scaling=1)


def options(**kw):
    o = dict(DEFAULTS)
    for k in kw:
        assert k in o, k
    o.update(kw)
    return o


def normalize_angle(a):
    """graph.h / vgo_normalize_angle: a - 2 pi floor((a + pi) / 2 pi), in the same float64 operations."""
    return a - TWO_PI * np.floor((a + 3.14159265358979323846) / TWO_PI)


def plus(x, free, d):
    """Plus(x, d) over the free unknowns of the flat 4N vector: xyz additive, yaw wrapped."""
    xc = np.array(x, np.float64).reshape(-1)
    v = xc[free] + d
    yaw = free % 4 == 3
    v[yaw] = normalize_angle(v[yaw])
    xc[free] = v
    return xc


def step_norms(x, xc, free):
    """step_norm = |x - Plus(x, d)| (the 2 pi jump of a wrapped yaw included) and x_norm, over the free
    unknowns, as lm_step_kernel and vgo_graph_solve compute them."""
    a = np.asarray(x, np.float64).reshape(-1)[free]
    dd = a - np.asarray(xc, np.float64).reshape(-1)[free]
    return float(np.sqrt(dd @ dd)), float(np.sqrt(a @ a))


def recover_step_wrapped(x0, x1, free, scale, y_ref):
    """solve_exact.recover_step for steps that may carry a yaw across +-pi: a yaw difference is taken
    modulo 2 pi, using the representative nearest the reference step y_ref (the replay's own).
    Returns y^ = -d / scale and delta >= |y^ - y|, with the rounding of the wrap included."""
    a0 = np.asarray(x0, np.float64).reshape(-1)[free]
    a1 = np.asarray(x1, np.float64).reshape(-1)[free]
    yaw = free % 4 == 3
    d_ref = -np.asarray(y_ref, np.float64) * scale
    jump = np.zeros(len(free))
    jump[yaw] = np.round((d_ref[yaw] - (a1[yaw] - a0[yaw])) / TWO_PI)
    if not np.any(jump) and np.all(np.abs(a1[yaw]) < 3.0):
        return SX.recover_step(x0, x1, free, scale)
    ld = np.longdouble
    d = a1.astype(ld) - a0.astype(ld) + jump.astype(ld) * ld(TWO_PI)
    y = -d / scale.astype(ld)
    df = np.abs(d.astype(np.float64))
    # x1 = fl(fl(x0 + d) - k fl(2 pi)): ulp(x1) + ulp(x0 + d) (k fl(2 pi) is exact for |k| = 1); d = fl(y * scale)
    delta = (np.spacing(np.abs(a1)) + np.where(jump != 0, np.spacing(np.abs(a0 + df * np.sign(d.astype(float)))), 0.0)
             + 2.0 * U * df) / scale * (1 + 1e-9)
    return y, delta


class Margin:
    """One decision: value against threshold, with the value's rounding uncertainty."""

    def __init__(self, name, value, threshold, uncertainty):
        self.name, self.value, self.threshold = name, float(value), float(threshold)
        self.uncertainty = float(uncertainty)

    @property
    def margin(self):
        """gap / uncertainty; a comparison of exactly known values (uncertainty 0) is never ambiguous."""
        gap = abs(self.value - self.threshold)
        return np.inf if self.uncertainty == 0 else gap / self.uncertainty

    @property
    def ambiguous(self):
        return self.margin <= 1.0

    def __repr__(self):
        return "%s %.6g vs %.6g (margin %.3g)" % (self.name, self.value, self.threshold, self.margin)


class Iteration:
    """Record of one replayed iteration: outcome is 'accepted', 'rejected', 'invalid', 'parameter'
    (termination 0) or 'function' (termination 1)."""

    def __init__(self, k, radius, eps_r, decrease_factor, reuse):
        self.k, self.radius, self.eps_r = k, radius, eps_r
        self.decrease_factor, self.reuse = decrease_factor, reuse
        self.outcome = None
        self.margins = []
        self.rho = None
        self.ratio = None            # backward-error ratio of a followed (device) accepted step
        self.damping_share = None    # min over columns of (diag / radius) / A_kk
        self.clamp_lo = self.clamp_hi = 0
        self.wraps = 0               # yaws an accepted step carried across +-pi
        self.x = None                # iterate after the iteration
        self.successful = 0
        self.problems = []           # follow mode: disagreements with the device


class Run:
    def __init__(self):
        self.iters = []
        self.termination = None
        self.checks = []             # margins of the finalize checks (gradient, radius)
        self.x0 = None
        self.problems = []

    @property
    def iterations(self):
        return len(self.iters)

    @property
    def successful(self):
        return sum(it.outcome == "accepted" for it in self.iters)

    @property
    def invalid(self):
        return sum(it.outcome == "invalid" for it in self.iters)

    @property
    def rejections(self):
        return sum(it.outcome == "rejected" for it in self.iters)

    @property
    def longest_rejection_run(self):
        best = cur = 0
        for it in self.iters:
            cur = cur + 1 if it.outcome in ("rejected", "invalid") else 0
            best = max(best, cur)
        return best

    @property
    def margins(self):
        return self.checks + [m for it in self.iters for m in it.margins]

    @property
    def ambiguous(self):
        return [m for m in self.margins if m.ambiguous]

    @property
    def smallest_margin(self):
        ms = self.margins
        return min(m.margin for m in ms) if ms else np.inf

    @property
    def clamp_hits(self):
        return (max([it.clamp_lo for it in self.iters], default=0), max([it.clamp_hi for it in self.iters], default=0))

    def truncated(self, k):
        """(iterations, successful steps, termination, x) of the same solve with max_num_iterations = k."""
        K = self.iterations
        if self.termination == 4:
            return 0, 0, 4, self.x0
        if k < K or (k == K and self.termination in (2, 3, 5)):
            x = self.iters[k - 1].x if k > 0 else self.x0
            return k, sum(it.outcome == "accepted" for it in self.iters[:k]), 3, x
        x = self.iters[-1].x if K else self.x0
        return K, self.successful, self.termination, x

    def coverage(self):
        return dict(iterations=self.iterations, successful=self.successful, rejections=self.rejections,
                    invalid=self.invalid, longest_rejection_run=self.longest_rejection_run,
                    clamp_hits=self.clamp_hits, wraps=sum(it.wraps for it in self.iters),
                    largest_radius=max([it.radius for it in self.iters], default=0.0),
                    smallest_damping_share=min([it.damping_share for it in self.iters[:3]
                                                if it.damping_share is not None], default=0.0),
                    termination=self.termination,
                    smallest_margin=self.smallest_margin)


def truncations(run):
    """The max_num_iterations values that truncate run: 0 .. K, and K + 1 unless the run itself was
    cut by max_num_iterations."""
    return range(run.iterations + (1 if run.termination == 3 else 2))


def replay(evaluate, x0, free, opts, follow=None, cost_rtol=1e-12, grad_rtol=1e-10, h_rtol=0.0):
    """Ceres' LM schedule (vgo_graph_solve's order of checks) in float64 from x0 (flat 4N).

    follow: None, or (xs, successful) with xs[k] the device's poses after k iterations (k = 0..K)
    and successful[k] its successful-step count; the replay then walks that trajectory (module doc).
    cost_rtol, grad_rtol, h_rtol: the relative uncertainty of an evaluation's cost, gradient and
    Hessian against another correct implementation's (h_rtol widens the step's forward error)."""
    o = opts
    free = np.asarray(free)
    run = Run()
    x = np.array(x0, np.float64).reshape(-1)
    run.x0 = x.copy()
    ok, cost, g, H = evaluate(x)
    assert ok
    scale = None
    radius, decrease_factor, reuse, invalid = float(o["initial_trust_region_radius"]), 2.0, False, 0
    eps_r = 0.0
    while True:
        # FinalizeIterationAndCheckIfMinimizerCanContinue, in Ceres' order: time, iterations, gradient, radius
        if o["max_solver_time_s"] <= 0:
            run.termination = 4
            break
        if run.iterations >= o["max_num_iterations"]:
            run.termination = 3
            break
        gmax = float(np.max(np.abs(g[free]))) if len(free) else 0.0
        run.checks.append(Margin("gradient", gmax, o["gradient_tolerance"],
                                 grad_rtol * max(gmax, float(np.max(np.abs(g)))) + 1e-300))
        if gmax <= o["gradient_tolerance"]:
            run.termination = 2
            break
        # the radius is known to a relative interval: compare logarithms
        run.checks.append(Margin("radius", np.log(radius), np.log(o["min_trust_region_radius"]), eps_r))
        if radius <= o["min_trust_region_radius"]:
            run.termination = 5
            break
        k = run.iterations + 1
        it = Iteration(k, radius, eps_r, decrease_factor, reuse)
        run.iters.append(it)
        A, b, scale = SX.lm_system(H, g, free, radius, o["jacobi_scaling"], scale,
                                   o["min_lm_diagonal"], o["max_lm_diagonal"])
        Hf = H[np.ix_(free, free)]
        Hs = (scale[:, None] * scale[None, :]) * Hf
        v = scale * scale * np.diag(Hf)
        it.clamp_lo = int(np.sum(v < o["min_lm_diagonal"]))
        it.clamp_hi = int(np.sum(v > o["max_lm_diagonal"]))
        diag = np.clip(v, o["min_lm_diagonal"], o["max_lm_diagonal"])
        pos = np.diag(A) > 0
        it.damping_share = float(np.min((diag / radius)[pos] / np.diag(A)[pos])) if np.any(pos) else None
        y = None
        try:
            y = scipy.linalg.cho_solve(scipy.linalg.cho_factor(A, lower=True, check_finite=True), b)
        except (np.linalg.LinAlgError, ValueError):
            pass
        mcc = SX.model_cost_change(H, g, free, scale, y) if y is not None and np.all(np.isfinite(y)) else np.nan
        dev_x_prev = dev_x = None
        dev_accepted = None
        if follow is not None:
            xs, succ = follow
            if k < len(xs):
                dev_x_prev, dev_x = np.asarray(xs[k - 1]).reshape(-1), np.asarray(xs[k]).reshape(-1)
                dev_accepted = succ[k] > succ[k - 1]
        if not (mcc > 0):
            it.outcome = "invalid"
            invalid += 1
            if dev_accepted:
                it.problems.append("device accepted a step the replay finds invalid")
            if invalid >= 5:
                run.termination = 6
                it.x = x.copy()
                break
            radius /= decrease_factor   # a power of two: exact, eps_r is unchanged
            decrease_factor *= 2
            reuse = True
            it.x = x.copy()
            if dev_x is not None and not np.array_equal(dev_x.view(np.uint64), dev_x_prev.view(np.uint64)):
                it.problems.append("x moved on an invalid step")
            continue
        invalid = 0
        step_rtol = np.linalg.cond(A) * (SX.gamma_c(len(b)) * U + h_rtol)
        ay = np.abs(y)
        if dev_accepted:
            # the device's step, recovered from its poses and checked at the replayed radius
            yd, delta = recover_step_wrapped(dev_x_prev, dev_x, free, scale, y)
            it.ratio = SX.backward_ratio(A, b, yd, delta, extra=(diag / radius) * eps_r * np.abs(np.asarray(yd, np.float64)))
            y = np.asarray(yd, np.float64)
            ay = np.abs(y)
            mcc = SX.model_cost_change(H, g, free, scale, y)
            xc = dev_x.copy()
        else:
            xc = plus(x, free, -y * scale)
        e_mcc = float((np.abs(b) + np.abs(Hs) @ ay) @ (step_rtol * ay))
        ok_c, cost_c, g_c, H_c = evaluate(xc)
        assert ok_c
        sn, xn = step_norms(x, xc, free)
        e_sn = step_rtol * sn + 4 * np.sqrt(len(free)) * float(np.max(np.spacing(np.abs(x[free]) + TWO_PI)))
        thr = o["parameter_tolerance"] * (xn + o["parameter_tolerance"])
        it.margins.append(Margin("parameter", sn, thr, e_sn))
        cc = cost - cost_c
        e_cc = e_mcc + 2 * cost_rtol * max(cost, cost_c)
        it.margins.append(Margin("function", abs(cc), o["function_tolerance"] * cost, e_cc))
        rho = cc / mcc
        it.rho = rho
        if sn <= thr:
            it.outcome = "parameter"
            run.termination = 0
        elif abs(cc) <= o["function_tolerance"] * cost:
            it.outcome = "function"
            run.termination = 1
        else:
            e_rho = (e_cc + abs(rho) * e_mcc) / abs(mcc)
            it.margins.append(Margin("rho", rho, o["min_relative_decrease"], e_rho))
            if rho > o["min_relative_decrease"]:
                it.outcome = "accepted"
                yaw = free[free % 4 == 3]
                it.wraps = int(np.sum(np.abs((xc[yaw] - x[yaw]) - (-y * scale)[free % 4 == 3]) > np.pi))
                x, cost, g, H = xc, cost_c, g_c, H_c
                q = 2.0 * rho - 1.0
                den = max(1.0 / 3.0, 1.0 - q * q * q)
                r_new = radius / den
                eps_new = eps_r + 6 * q * q / den * e_rho + 4 * U
                if r_new > o["max_trust_region_radius"]:
                    # the cap decides the radius unless the uncapped value could lie below it
                    eps_new = 0.0 if r_new * (1 - eps_new) > o["max_trust_region_radius"] else eps_new
                    r_new = o["max_trust_region_radius"]
                radius, eps_r = r_new, eps_new
                decrease_factor, reuse = 2.0, False
            else:
                it.outcome = "rejected"
                radius /= decrease_factor
                decrease_factor *= 2
                reuse = True
        it.x = x.copy()
        it.successful = run.successful
        if dev_accepted is not None:
            if dev_accepted != (it.outcome == "accepted"):
                it.problems.append("device accepted=%s, replay %s" % (dev_accepted, it.outcome))
            if not dev_accepted and not np.array_equal(dev_x.view(np.uint64), dev_x_prev.view(np.uint64)):
                it.problems.append("x moved on a step that was not accepted")
        if run.termination is not None:
            break
    run.problems = ["iteration %d: %s" % (it.k, p) for it in run.iters for p in it.problems]
    return run


# ------------------------------------------------------------------ scenarios
class Scenario:
    """A pose graph (solve_exact.Spec, or RegSpec with registration constraints) and solver options,
    plus the coverage it must reach on the oracle's trajectory (tests/test_oracle_lm_schedule.py)."""

    def __init__(self, name, spec, opts, expect):
        self.name, self.spec, self.opts, self.expect = name, spec, opts, expect

    @property
    def path(self):
        return "shared memory" if self.spec.n <= SX.SMEM_MAX_N else "cooperative"

    @property
    def registration(self):
        return isinstance(self.spec, RegSpec)

    @property
    def tolerances(self):
        """replay() uncertainties: float64 rounding for relative-pose graphs; for registration graphs the
        device's per-point sums differ from the oracle's by ~1e-9 relative in H (and less in the cost)."""
        if self.registration:
            return dict(cost_rtol=1e-8, grad_rtol=1e-8, h_rtol=1e-8)
        return dict(cost_rtol=1e-12, grad_rtol=1e-10, h_rtol=0.0)

    def oracle_graph(self, oracle):
        og = SX.oracle_graph(oracle, self.spec)
        if self.registration:
            self.spec.add_oracle_registration(oracle, og)
        return og

    def pose_graph(self, ctx):
        """The scenario's api.PoseGraph on ctx, synchronised (the context's current graph)."""
        from voxgraph_b200 import api
        if self.registration:
            self.spec.upload(ctx)
        pg = SX.pose_graph(api, ctx, self.spec)
        if self.registration:
            for (i, j) in self.spec.scene.pairs:
                pg.addRegistrationConstraint(api.RegistrationConstraintConfig(i, j))
        pg._sync()
        return pg


class RegSpec(SX.Spec):
    """A synth scene as a pose graph (test_gpu_solver's layout): node 0 constant, the odometry as
    relative-pose edges, and one mirrored registration constraint (isosurface points) per
    overlapping pair, from the scene's initial poses."""

    def __init__(self, scene):
        self.scene = scene
        n = len(scene.submaps)
        edges = [(i, j, np.asarray(t, np.float64), float(y), scene.odom_information) for (i, j, t, y) in scene.odometry]
        super().__init__(list(range(n)), np.array(scene.poses_init, np.float64), [i == 0 for i in range(n)], edges)

    def add_oracle_registration(self, oracle, og):
        sc = self.scene
        layers = [oracle.Layer.from_blocks(s.voxel_size, s.vps, s.block_idx, s.distance, s.weight) for s in sc.submaps]
        for (i, j) in sc.pairs:
            a, b = sc.submaps[i], sc.submaps[j]
            og.add_registration(i, j, layers[j], a.points_xyz, a.points_distance, a.points_weight)
            og.add_registration(j, i, layers[i], b.points_xyz, b.points_distance, b.points_weight)

    def upload(self, ctx):
        for s in self.scene.submaps:
            ctx.upload_synth_submap(s)


def small_scene():
    """tests/conftest.py small_scene: a scaled-down config 2 (6 submaps, 2k points each)."""
    from voxgraph_b200 import synth
    return RegSpec(synth.make_scene(seed=2, n_submaps=6, n_points=2000, radius=8.0, size_xy=(48.0, 32.0),
                                    n_clutter=80, n_walls=6))


def far_graph(n, seed, xy=3.0, yaw=2.0, **kw):
    """solve_exact.make_graph with the free poses moved up to xy metres and yaw radians further from
    the measurements: a start where many LM steps are rejected."""
    spec = SX.make_graph(n, seed=seed, **kw)
    rng = np.random.default_rng(seed + 77)
    x0 = spec.x0.copy()
    fr = ~spec.constant
    x0[fr, :2] += rng.uniform(-xy, xy, (int(fr.sum()), 2))
    x0[fr, 3] = normalize_angle(x0[fr, 3] + rng.uniform(-yaw, yaw, int(fr.sum())))
    return SX.Spec(spec.ids, x0, spec.constant, spec.edges)


def rotated(spec, theta):
    """The same graph seen from a frame rotated by theta about z: every pose (constant ones too) is
    rotated, the relative measurements are unchanged, so the solution is the rotated one."""
    c, s = np.cos(theta), np.sin(theta)
    x0 = spec.x0.copy()
    x0[:, 0], x0[:, 1] = c * spec.x0[:, 0] - s * spec.x0[:, 1], s * spec.x0[:, 0] + c * spec.x0[:, 1]
    x0[:, 3] = normalize_angle(spec.x0[:, 3] + theta)
    return SX.Spec(spec.ids, x0, spec.constant, spec.edges)


def yaw_wrap_graph():
    """Free node 3 starts at yaw pi - 0.05 and its solution lies past pi: an accepted step wraps."""
    spec = SX.make_graph(32, seed=11)
    return rotated(spec, np.pi - 0.05 - spec.x0[3, 3])


def scenarios():
    S = []
    tight = dict(parameter_tolerance=1e-9, function_tolerance=1e-9, max_num_iterations=60)
    # min_relative_decrease 0.9: steps the quadratic model predicts to within 10 % only are accepted
    rej32 = far_graph(32, seed=1, loops=False)
    rej = dict(min_relative_decrease=0.9, max_num_iterations=200)
    S.append(Scenario("rejections_32", rej32, options(**rej),
                      dict(rejections=10, run=3, termination=(0,))))
    S.append(Scenario("rejections_260", far_graph(260, seed=0, loops=False), options(**rej),
                      dict(rejections=3, run=2, termination=(0,))))
    S.append(Scenario("function_tolerance", rej32, options(parameter_tolerance=1e-14, **rej),
                      dict(rejections=1, termination=(1,))))
    S.append(Scenario("heavy_damping", SX.make_graph(32, seed=21),
                      options(initial_trust_region_radius=1e-2, max_trust_region_radius=1.0, **tight),
                      dict(largest_radius=1.0, damping_share=0.5)))
    S.append(Scenario("clamps_jacobi0", SX.make_graph(32, seed=31),
                      options(jacobi_scaling=0, min_lm_diagonal=20.0, max_lm_diagonal=200.0, **tight),
                      dict(clamps=True)))
    S.append(Scenario("clamps_jacobi1", SX.make_graph(32, seed=32),
                      options(min_lm_diagonal=0.8, max_lm_diagonal=0.9, **tight), dict(clamps=True)))
    S.append(Scenario("yaw_wrap", yaw_wrap_graph(), options(**tight), dict(wraps=1)))
    S.append(Scenario("gradient_at_x0", SX.make_graph(32, seed=41), options(gradient_tolerance=1e6),
                      dict(termination=(2,), iterations=0)))
    S.append(Scenario("gradient_after_step", SX.make_graph(32, seed=41),
                      options(gradient_tolerance=GRADIENT_AFTER_STEP, parameter_tolerance=1e-14,
                              function_tolerance=1e-14),
                      dict(termination=(2,), successful=1)))
    S.append(Scenario("time_budget_zero", SX.make_graph(32, seed=51), options(max_solver_time_s=0.0),
                      dict(termination=(4,), iterations=0)))
    S.append(Scenario("min_radius_at_x0", SX.make_graph(32, seed=51),
                      options(initial_trust_region_radius=1e-3, min_trust_region_radius=1e-3),
                      dict(termination=(5,), iterations=0)))
    S.append(Scenario("min_radius_rejections", rej32, options(min_trust_region_radius=MIN_RADIUS_REJECTIONS, **rej),
                      dict(termination=(5,), rejections=1)))
    reg = small_scene()
    # voxgraph's options (pose_graph.cpp:91-97) and tight ones; the scene's yaws lie near +-pi
    S.append(Scenario("registration_voxgraph", reg, options(), dict(termination=(0,), accepted=3, wraps=1)))
    S.append(Scenario("registration_tight", reg, options(**REGISTRATION_TIGHT),
                      dict(termination=(0,), accepted=5, wraps=1)))
    for n in (32, 260):
        S.append(Scenario("invalid_steps_%d" % n, SX.make_graph(n, seed=61 + n, untouched=True),
                          options(min_lm_diagonal=0.0), dict(termination=(6,), invalid=5)))
    return S


# thresholds chosen on the oracle's trajectories of the graphs above (tests/test_oracle_lm_schedule.py
# checks the coverage they give, with every decision clear of its rounding uncertainty)
GRADIENT_AFTER_STEP = 1.0      # met after the second accepted step
REGISTRATION_TIGHT = dict(parameter_tolerance=1e-6, function_tolerance=1e-9, max_num_iterations=100)
MIN_RADIUS_REJECTIONS = 12.0   # below every radius before the first run of 4 rejections ends at 9.77


def report(request, lines):
    """Write lines to the terminal past pytest's output capture, so a passing run shows them."""
    cap = request.config.pluginmanager.getplugin("capturemanager")
    tr = request.config.pluginmanager.getplugin("terminalreporter")
    if tr is None:
        return
    with cap.global_and_fixture_disabled():
        tr.write_line("")
        for line in lines:
            tr.write_line(line)


# ------------------------------------------------------------------ device runs
def device_solve(ctx, spec, opts, k=None):
    """vgx_graph_solve from spec.x0 on the context's current graph (max_num_iterations = k if given):
    (return code, (iterations, successful, residual evals, termination, initial cost, final cost),
    poses (N, 4)).  The summary and poses are read even when the solve fails (termination 6)."""
    import ctypes as C
    from voxgraph_b200 import _lib
    ctx.graph_set_poses(spec.x0)
    o = ctx.solver_options(**opts)
    if k is not None:
        o.max_num_iterations = k
    s = _lib.SolverSummary()
    x = np.zeros((spec.N, 4))
    rc = ctx._L.vgx_graph_solve(ctx._h, C.byref(o), x.ctypes.data_as(C.POINTER(C.c_double)), C.byref(s))
    return rc, (s.iterations, s.num_successful_steps, s.num_residual_evals, s.termination,
                s.initial_cost, s.final_cost), x


def device_trajectory(ctx, sc):
    """The pose graph of scenario sc on ctx, and its device solves at every truncation of the device's
    own full run: [(rc, summary, x) for k in truncations]."""
    pg = sc.pose_graph(ctx)
    full = device_solve(ctx, sc.spec, sc.opts)
    it, term = full[1][0], full[1][3]
    ks = range(it + (1 if term == 3 else 2))
    return pg, [device_solve(ctx, sc.spec, sc.opts, k) for k in ks] + [full]


def _main(out):
    """Every scenario's device trajectory into the npz `out` (run in a fresh process, e.g. with
    VGX_LM_NO_RUNAHEAD=1, which solve.cu reads once per process)."""
    from voxgraph_b200 import api
    ctx = api.Context(0)
    res = {}
    for sc in scenarios():
        _, runs = device_trajectory(ctx, sc)
        res[sc.name + ".rc"] = np.array([r[0] for r in runs])
        res[sc.name + ".summary"] = np.array([r[1] for r in runs], np.float64)
        res[sc.name + ".x"] = np.array([r[2] for r in runs])
    ctx.close()
    np.savez(out, **res)


if __name__ == "__main__":
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    _main(sys.argv[1])
