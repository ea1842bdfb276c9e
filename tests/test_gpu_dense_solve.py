"""The device's dense solves against a backward-error bound (tests/solve_exact.py).

LM first and second steps at sizes straddling the dispatch edge of solve.cu (shared-memory FP64-MMA
Cholesky up to n = 232, the cooperative grid from 236), edge covariances (always on the cooperative
grid) and the rank rule of getEdgeCovarianceMap."""
import numpy as np
import pytest

import solve_exact as SX
from support import ctx  # noqa: F401

pytestmark = pytest.mark.gpu

RADII = [1e4, 1.0, 1e-3]       # nearly Gauss-Newton .. heavy damping
ANCHORS = ["first", "interleaved", "frame"]
WORST = {}                     # largest ratio to the bound per path, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for k in sorted(WORST):
        print("dense solve: largest ratio to the bound, %-36s %.3g" % (k, WORST[k]))


def _note(path, ratio):
    WORST[path] = max(WORST.get(path, 0.0), ratio)


def _lm_path(n):
    return "LM shared memory" if n <= SX.SMEM_MAX_N else "LM cooperative"


def _graph(ctx, spec):
    from voxgraph_b200 import api
    pg = SX.pose_graph(api, ctx, spec)
    ok, cost, g, H = pg.evaluate()
    assert ok
    return pg, cost, g, H


def _solve(ctx, pg, spec, x_start, iterations, radius, jacobi, **kw):
    """Forced-accept solve of `iterations` steps from x_start; the poses it returns."""
    ctx.graph_set_poses(x_start)
    pg.solver_options = ctx.solver_options(max_num_iterations=iterations, initial_trust_region_radius=radius,
                                           jacobi_scaling=jacobi, **SX.FORCED, **kw)
    s = pg.optimize()
    assert s.num_successful_steps == iterations and s.iterations == iterations, (s.iterations, s.termination)
    return ctx.graph_get_poses(spec.N)


@pytest.mark.parametrize("n", SX.LM_SIZES)
def test_lm_first_step_backward_error(ctx, n):
    spec = SX.make_graph(n, anchor=ANCHORS[SX.LM_SIZES.index(n) % 3], seed=n)
    pg, _, g, H = _graph(ctx, spec)
    for jacobi in (0, 1):
        for radius in RADII:
            x1 = _solve(ctx, pg, spec, spec.x0, 1, radius, jacobi)
            ratio, _ = SX.step_ratio(H, g, spec.x0, x1, spec.free, radius, jacobi)
            _note(_lm_path(n) + (", radius 1e-3" if radius < 1 else ""), ratio)
            assert ratio < 1, (jacobi, radius, ratio)


@pytest.mark.parametrize("n", [232, 796])
def test_lm_first_step_ill_conditioned_chain(ctx, n):
    """Anchored chains without loop closures (condition numbers of J^T J 2e7 and 2e8)."""
    spec = SX.make_graph(n, anchor="first", loops=False, seed=7 + n, info=SX.INFO_ODOM)
    pg, _, g, H = _graph(ctx, spec)
    Hf = H[np.ix_(spec.free, spec.free)]
    assert np.linalg.cond(Hf) > 1e7
    for radius in RADII:
        x1 = _solve(ctx, pg, spec, spec.x0, 1, radius, 1)
        ratio, _ = SX.step_ratio(H, g, spec.x0, x1, spec.free, radius, 1)
        _note(_lm_path(n) + (", radius 1e-3" if radius < 1 else ""), ratio)
        assert ratio < 1, (radius, ratio)


@pytest.mark.parametrize("n", [12, 36, 232, 236, 260, 796])
@pytest.mark.parametrize("jacobi", [0, 1])
def test_lm_second_step_keeps_iteration_0_scale(ctx, n, jacobi):
    """Two forced steps with max radius = initial radius.  Step 1 decreases the cost by more than half
    the model's prediction, so the radius stays at its maximum; step 2 must then solve the system built
    from H and g at x1 with the Jacobi scale of iteration 0 (scale_ready, lm_persist_kernel)."""
    spec = SX.make_graph(n, anchor="interleaved", seed=1000 + n)
    pg, cost0, g0, H0 = _graph(ctx, spec)
    for radius in (1e4, 1.0):
        x1 = _solve(ctx, pg, spec, spec.x0, 1, radius, jacobi, max_trust_region_radius=radius)
        ok, cost1, g1, H1 = pg.evaluate()
        ratio1, (_, _, y1, scale0) = SX.step_ratio(H0, g0, spec.x0, x1, spec.free, radius, jacobi)
        assert ratio1 < 1
        rel = (cost0 - cost1) / SX.model_cost_change(H0, g0, spec.free, scale0, y1)
        assert rel > 0.5, rel
        x2 = _solve(ctx, pg, spec, spec.x0, 2, radius, jacobi, max_trust_region_radius=radius)
        ratio2, _ = SX.step_ratio(H1, g1, x1, x2, spec.free, radius, jacobi, scale=scale0)
        _note(_lm_path(n), ratio2)
        assert ratio2 < 1, (radius, ratio2)


def _red(spec):
    red, o = {}, 0
    for i, nid in enumerate(spec.ids):
        if not spec.constant[i]:
            red[nid] = o
            o += 4
    return red


def _check_covariances(ctx, spec, path):
    pg, _, _, H = _graph(ctx, spec)
    Hf = H[np.ix_(spec.free, spec.free)]
    red = _red(spec)
    free_ids = list(red)
    const_ids = [nid for i, nid in enumerate(spec.ids) if spec.constant[i]]
    col_ids = sorted({free_ids[0], free_ids[len(free_ids) // 2], free_ids[-1]})
    pairs = [(a, b) for b in col_ids for a in free_ids]           # whole columns, (b, b) included
    pairs += [(col_ids[0], a) for a in free_ids[1:3]]             # (b, a): other columns, one block
    pairs += [(c, col_ids[-1]) for c in const_ids[:2]] + [(col_ids[0], c) for c in const_ids[:2]]
    got = pg.getEdgeCovarianceMap(pairs)
    X = np.zeros((spec.n, 4 * len(col_ids)))
    for k, b in enumerate(col_ids):
        for a in free_ids:
            X[red[a]:red[a] + 4, 4 * k:4 * k + 4] = got[(a, b)]
    cols = [red[b] + q for b in col_ids for q in range(4)]
    ratio = SX.covariance_ratio(Hf, X, cols)
    _note(path, ratio)
    assert ratio < 1, ratio
    scale = np.abs(X).max()
    for a in free_ids[1:3]:
        assert np.abs(got[(col_ids[0], a)] - got[(a, col_ids[0])].T).max() <= 1e-8 * scale
    for c in const_ids[:2]:
        assert np.all(got[(c, col_ids[-1])] == 0) and np.all(got[(col_ids[0], c)] == 0)


def _cov_path(n):
    return "covariance n <= 256" if n <= 256 else "covariance n > 256"


@pytest.mark.parametrize("n", SX.COV_SIZES)
def test_covariance_columns_backward_error(ctx, n):
    _check_covariances(ctx, SX.make_graph(n, anchor="interleaved", seed=2000 + n), _cov_path(n))


@pytest.mark.parametrize("n", [252, 796])
def test_covariance_ill_conditioned_chain(ctx, n):
    """Anchored chains without loop closures are full rank: no error, and the bound holds."""
    _check_covariances(ctx, SX.make_graph(n, anchor="first", loops=False, seed=3000 + n, info=SX.INFO_ODOM),
                       _cov_path(n))


@pytest.mark.parametrize("n,kind", [(32, "gauge"), (252, "gauge"), (260, "gauge"), (796, "gauge"),
                                    (36, "untouched"), (260, "untouched")])
def test_covariance_rank_deficient_raises(ctx, n, kind):
    """ceres::Covariance::Compute fails on a rank-deficient J^T J: a graph without a constant node
    (4-dimensional gauge freedom) or with a free node no constraint touches."""
    from voxgraph_b200 import api
    if kind == "gauge":
        spec = SX.make_graph(n, anchor="none", seed=4017 + n)
    else:
        spec = SX.make_graph(n, anchor="first", seed=4000 + n, untouched=True)
    pg, _, _, _ = _graph(ctx, spec)
    free_ids = list(_red(spec))
    with pytest.raises(api.VgxError, match="rank deficient"):
        pg.getEdgeCovarianceMap([(free_ids[0], free_ids[-1]), (free_ids[-1], free_ids[-1])])


@pytest.mark.parametrize("n", [32, 260])
def test_lm_on_gauge_free_graph(ctx, n):
    """The LM damping makes A positive definite without a constant node: the step passes the bound
    and a default solve ends normally."""
    spec = SX.make_graph(n, anchor="none", seed=5000 + n)
    pg, cost0, g, H = _graph(ctx, spec)
    for radius in (1e4, 1.0):
        x1 = _solve(ctx, pg, spec, spec.x0, 1, radius, 1)
        ratio, _ = SX.step_ratio(H, g, spec.x0, x1, spec.free, radius, 1)
        _note(_lm_path(n), ratio)
        assert ratio < 1, (radius, ratio)
    ctx.graph_set_poses(spec.x0)
    pg.solver_options = ctx.solver_options()
    s = pg.optimize()
    assert s.termination in (0, 1, 2) and s.final_cost < cost0
