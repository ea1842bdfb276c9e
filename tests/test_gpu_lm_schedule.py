"""The device's Levenberg-Marquardt schedule, step by step (tests/lm_schedule.py).

Every scenario is solved from x0 with max_num_iterations = k for every k up to the length of its full
run.  A: each truncated solve reports the oracle's (iterations, successful steps, termination), with
poses within 1e-9 of the oracle's for relative-pose graphs and at test_gpu_solver's tolerances for
registration graphs.  B: the float64 replay walks the device's own trajectory on the device's own
evaluations, which pins the registration scenarios at full precision (there the device's H differs
from the oracle's by ~1e-9): each accepted step passes the backward-error bound of the LM system at
the replayed radius, Jacobi scale and diagonal, and each rejected step leaves x bit-unchanged while
the replay's candidate is rejected too.  Also: the speculative iteration the host enqueues ahead is a
no-op (VGX_LM_NO_RUNAHEAD=1 gives the same bits), and a solve leaves no state behind for the next."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import lm_schedule as LS
import solve_exact as SX
from support import ctx  # noqa: F401

pytestmark = pytest.mark.gpu

SCENARIOS = {s.name: s for s in LS.scenarios()}
TRAJ = {}        # scenario -> [(rc, summary, x)], the in-process (run-ahead) solves
WORST = {}       # largest backward-error ratio per Cholesky path
MARGIN = {}      # smallest decision margin per scenario


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    LS.report(request, ["LM schedule: largest backward-error ratio, %-14s %.3g" % (k, WORST[k]) for k in sorted(WORST)]
              + ["LM schedule: smallest decision margin, %-22s %.3g" % (k, MARGIN[k]) for k in sorted(MARGIN)])


def _trajectory(ctx, name):
    sc = SCENARIOS[name]
    pg, runs = LS.device_trajectory(ctx, sc)
    TRAJ[name] = runs
    return sc, pg, runs


def _wrapped_diff(a, b):
    d = (np.asarray(a) - np.asarray(b)).reshape(-1, 4)
    d[:, 3] = LS.normalize_angle(d[:, 3])
    return np.abs(d).max()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_schedule_matches_oracle_and_replay(ctx, oracle, name):
    sc, pg, runs = _trajectory(ctx, name)
    spec = sc.spec
    full = runs[-1]
    runs = runs[:-1]
    # poses: 1e-9 of the pose scale for relative-pose graphs; registration graphs at test_gpu_solver's
    # tolerances (the device's per-point sums differ from the oracle's in the last digits)
    if not sc.registration:
        pose_tol = 1e-9 * max(1.0, float(np.abs(spec.x0).max()))
    else:
        pose_tol = 1e-4 if sc.opts["parameter_tolerance"] < 3e-3 else 3e-3
    # A: schedule parity with the oracle at every truncation
    for k, (rc, s, x) in enumerate(runs):
        og = sc.oracle_graph(oracle)
        orc, so = og.solve(oracle.solver_options(num_threads=1, **dict(sc.opts, max_num_iterations=k)))
        assert (s[0], s[1], s[3]) == (so.iterations, so.num_successful_steps, so.termination), k
        assert _wrapped_diff(x, og.poses()) <= pose_tol, (k, _wrapped_diff(x, og.poses()))
        assert (rc == 0) == (so.termination != 6), (k, rc)
    assert full[1][:4] == runs[-1][1][:4] and np.array_equal(_bits(full[2]), _bits(runs[-1][2]))
    # B: the replay on the device's own evaluations, following the device's trajectory
    xs = [r[2].reshape(-1) for r in runs]
    succ = [r[1][1] for r in runs]

    def evaluate(x):
        ctx.graph_set_poses(np.asarray(x).reshape(spec.N, 4))
        return pg.evaluate()
    try:
        run = LS.replay(evaluate, spec.x0, spec.free, sc.opts, follow=(xs, succ), **sc.tolerances)
    finally:
        ctx.graph_set_poses(spec.x0)
    assert not run.problems, run.problems
    assert (run.iterations, run.successful, run.termination) == (full[1][0], full[1][1], full[1][3])
    assert not run.ambiguous, run.ambiguous
    MARGIN[name] = run.smallest_margin
    for it in run.iters:
        if it.ratio is not None:
            WORST[sc.path] = max(WORST.get(sc.path, 0.0), it.ratio)
            assert it.ratio <= 1, (it.k, it.ratio)
    # the residual evaluations the device counts: the start plus one per candidate of a valid step
    for k, (rc, s, x) in enumerate(runs):
        invalid = sum(it.outcome == "invalid" for it in run.iters[:k])
        assert s[2] == 1 + s[0] - invalid, (k, s)
    # a solve that takes no step leaves the poses and the cost as they were
    if full[1][0] == 0:
        assert np.array_equal(_bits(full[2]), _bits(spec.x0.reshape(-1, 4)))
        assert full[1][5] == full[1][4]
    if sc.opts["max_solver_time_s"] == 0:
        assert full[1][3] == 4 and full[1][0] == 0
    if run.termination == 6:
        from voxgraph_b200 import api, _lib
        assert full[0] == _lib.VGX_ERR_INVALID and full[1][3] == 6
        assert np.array_equal(_bits(full[2]), _bits(spec.x0.reshape(-1, 4)))
        ctx.graph_set_poses(spec.x0)
        pg.solver_options = ctx.solver_options(**sc.opts)
        with pytest.raises(api.VgxError, match="invalid steps"):
            pg.optimize()


def test_runahead_is_a_no_op(ctx):
    """The whole matrix again in a fresh process that waits for each iteration's outcome before it
    enqueues the next (VGX_LM_NO_RUNAHEAD=1): bit-identical poses and summaries for every k."""
    missing = sorted(set(SCENARIOS) - set(TRAJ))
    for name in missing:
        _trajectory(ctx, name)
    env = dict(os.environ, VGX_LM_NO_RUNAHEAD="1")
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "no_runahead.npz")
        subprocess.run([sys.executable, "-s", os.path.join(os.path.dirname(__file__), "lm_schedule.py"), out],
                       check=True, env=env, timeout=1200)
        with np.load(out) as ref:
            for name, runs in TRAJ.items():
                assert np.array_equal(ref[name + ".rc"], [r[0] for r in runs]), name
                assert np.array_equal(_bits(ref[name + ".summary"]),
                                      _bits(np.array([r[1] for r in runs], np.float64))), name
                assert np.array_equal(_bits(ref[name + ".x"]), _bits(np.array([r[2] for r in runs]))), name


@pytest.mark.parametrize("name,k", [("rejections_32", 4), ("rejections_32", 7), ("rejections_260", 6),
                                    ("clamps_jacobi0", 2)])
def test_no_state_leaks_between_solves(ctx, name, k):
    """A solve on tables a previous solve used (its scale, diagonal and radius still in d_scale, d_diag
    and d_state) gives the same bits as a fresh graph's solve from the same poses."""
    from voxgraph_b200 import api
    sc = SCENARIOS[name]
    pg = SX.pose_graph(api, ctx, sc.spec)
    pg._sync()
    _, _, xk = LS.device_solve(ctx, sc.spec, sc.opts, k)     # stops mid-run, after rejections
    spec_k = SX.Spec(sc.spec.ids, xk, sc.spec.constant, sc.spec.edges)
    second = LS.device_solve(ctx, spec_k, sc.opts)
    fresh_pg = SX.pose_graph(api, ctx, spec_k)
    fresh_pg._sync()
    fresh = LS.device_solve(ctx, spec_k, sc.opts)
    assert second[0] == fresh[0] and second[1] == fresh[1]
    assert np.array_equal(_bits(second[2]), _bits(fresh[2]))
