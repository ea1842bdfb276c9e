"""The float64 LM replay of tests/lm_schedule.py against the oracle's vgo_graph_solve (CPU).

Driven by the oracle's own evaluations, the replay must reproduce the oracle's solve at every
truncation max_num_iterations = k: the same iterations, successful steps and termination, and the
same poses to 1e-12.  Each scenario must also reach the coverage it exists for, with no decision on
its trajectory inside the rounding uncertainty.  tests/test_gpu_lm_schedule.py relies on both."""
import numpy as np
import pytest

import lm_schedule as LS
import solve_exact as SX

SCENARIOS = {s.name: s for s in LS.scenarios()}
RUNS = {}        # scenario -> the replay on the oracle's evaluations (computed once per process)
COVERAGE = {}    # scenario -> coverage counts, reported at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    LS.report(request, ["LM schedule coverage, %-22s %s" % (k, COVERAGE[k]) for k in sorted(COVERAGE)])


def _oracle_opts(oracle, opts):
    return oracle.solver_options(num_threads=1, **opts)


def _replay(oracle, sc):
    if sc.name not in RUNS:
        og = sc.oracle_graph(oracle)

        def evaluate(x):
            og.set_poses(np.asarray(x).reshape(sc.spec.N, 4))
            return og.eval()
        RUNS[sc.name] = LS.replay(evaluate, sc.spec.x0, sc.spec.free, sc.opts, **sc.tolerances)
    return RUNS[sc.name]


def test_defaults_match_oracle(oracle):
    o = oracle.solver_options()
    for k, v in LS.DEFAULTS.items():
        assert getattr(o, k) == v, k


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_replay_reproduces_oracle_at_every_truncation(oracle, name):
    sc = SCENARIOS[name]
    run = _replay(oracle, sc)
    scale = max(1.0, float(np.abs(sc.spec.x0).max()))
    for k in LS.truncations(run):
        og = sc.oracle_graph(oracle)
        rc, s = og.solve(_oracle_opts(oracle, dict(sc.opts, max_num_iterations=k)))
        it, succ, term, x = run.truncated(k)
        assert (s.iterations, s.num_successful_steps, s.termination) == (it, succ, term), k
        assert rc == (-1 if term == 6 else 0)
        d = og.poses().reshape(-1) - x
        d[3::4] = LS.normalize_angle(d[3::4])
        assert np.abs(d).max() <= 1e-12 * scale, (k, np.abs(d).max())
    # the untruncated solve
    og = sc.oracle_graph(oracle)
    rc, s = og.solve(_oracle_opts(oracle, sc.opts))
    assert (s.iterations, s.num_successful_steps, s.termination) == (run.iterations, run.successful, run.termination)


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_scenario_coverage(oracle, name):
    sc = SCENARIOS[name]
    run = _replay(oracle, sc)
    cov = run.coverage()
    COVERAGE[name] = "rejections %d, longest run %d, invalid %d, clamp hits %s, wraps %d, termination %d" % (
        cov["rejections"], cov["longest_rejection_run"], cov["invalid"], cov["clamp_hits"], cov["wraps"],
        cov["termination"])
    assert not run.ambiguous, run.ambiguous
    e = sc.expect
    if "termination" in e:
        assert run.termination in e["termination"]
    if "iterations" in e:
        assert run.iterations == e["iterations"]
    if "rejections" in e:
        assert run.rejections >= e["rejections"]
        if run.termination == 5:   # reached through a run of rejections
            assert run.iters[-1].outcome == "rejected"
    if "run" in e:
        assert run.longest_rejection_run >= e["run"]
        assert max(it.decrease_factor for it in run.iters) >= 2 ** e["run"]
    if "accepted" in e:
        assert run.successful >= e["accepted"]
    if "successful" in e:
        assert run.successful >= e["successful"] and run.iters[-1].outcome == "accepted"
    if "invalid" in e:
        assert run.invalid == e["invalid"] and run.successful == 0
    if "largest_radius" in e:   # the cap binds
        assert cov["largest_radius"] == e["largest_radius"] == sc.opts["max_trust_region_radius"]
        assert any(it.radius == sc.opts["max_trust_region_radius"] for it in run.iters)
    if "damping_share" in e:
        assert cov["smallest_damping_share"] >= e["damping_share"]
    if "clamps" in e:
        lo, hi = cov["clamp_hits"]
        assert lo > 0 and hi > 0
    if "wraps" in e:
        assert cov["wraps"] >= e["wraps"]
        if name == "yaw_wrap":
            assert sc.spec.x0[3, 3] == pytest.approx(np.pi - 0.05, abs=1e-12)
    if run.termination in (0, 1) and "rejections" in e:
        assert run.rejections >= 1


def test_cholesky_paths_covered():
    """Rejections and invalid steps on both of solve.cu's LM Cholesky paths."""
    paths = {(s.path, s.expect.get("termination", (None,))[0] == 6) for s in SCENARIOS.values()}
    assert {("shared memory", True), ("cooperative", True), ("shared memory", False), ("cooperative", False)} <= paths
    assert SCENARIOS["rejections_260"].spec.n >= SX.COOP_MIN_N


def test_registration_scenarios_have_one_constant_node():
    for name in ("registration_voxgraph", "registration_tight"):
        sc = SCENARIOS[name]
        assert sc.registration and int(sc.spec.constant.sum()) == 1 and len(sc.spec.scene.pairs) > 0
