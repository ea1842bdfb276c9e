"""GPU parity: device-resident Levenberg-Marquardt vs the oracle's Ceres-default LM."""
import numpy as np
import pytest

from support import ctx, oracle_layer  # noqa: F401
from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu


def _wrap(a):
    return a - 2 * np.pi * np.floor((a + np.pi) / (2 * np.pi))


def test_relative_pose_loop_ka12(ctx, oracle):
    from voxgraph_b200 import api
    rs = np.random.RandomState(1)
    n = 8
    gt = np.stack([3 * np.cos(np.linspace(0, 2 * np.pi, n, endpoint=False)),
                   3 * np.sin(np.linspace(0, 2 * np.pi, n, endpoint=False)),
                   np.linspace(0, 0.5, n), np.linspace(-2.5, 2.5, n)], -1)
    pg = api.PoseGraph(ctx)
    og = oracle.Graph()
    info = np.diag([1.0, 1.0, 2500.0, 2500.0])
    L = oracle.sqrt_information(info)
    for i in range(n):
        init = gt[i] + (0 if i == 0 else rs.normal(0, 0.3, 4))
        pg.addSubmapNode(api.SubmapNodeConfig(i, init, set_constant=(i == 0)))
        og.add_node(i, init, constant=(i == 0))
    for i in range(n):
        j = (i + 1) % n
        t, y = synth.relative_pose(gt[i], gt[j])
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(i, j, np.array([*t, y]), info))
        og.add_relative(i, j, t, y, L)
    # per-evaluation parity first
    ok, cost_g, g_g, H_g = pg.evaluate()
    ok, cost_o, g_o, H_o = og.eval()
    np.testing.assert_allclose(cost_g, cost_o, rtol=1e-12)
    np.testing.assert_allclose(g_g, g_o, rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(H_g, H_o, rtol=1e-10, atol=1e-9)
    pg.solver_options = ctx.solver_options(parameter_tolerance=1e-12, function_tolerance=1e-16,
                                           max_num_iterations=100)
    s = pg.optimize()
    rc, so = og.solve(oracle.solver_options(parameter_tolerance=1e-12, function_tolerance=1e-16,
                                            max_num_iterations=100))
    x = np.array([pg.getSubmapPoses()[i] for i in range(n)])
    np.testing.assert_allclose(x[:, :3], gt[:, :3], atol=1e-7)
    np.testing.assert_allclose(_wrap(x[:, 3] - gt[:, 3]), 0, atol=1e-7)
    assert s.final_cost < 1e-15
    # same trust-region schedule: identical iteration count and termination
    assert (s.iterations, s.termination) == (so.iterations, so.termination)
    assert s.num_successful_steps == so.num_successful_steps


@pytest.mark.parametrize("pert", [(0.3, 0.0, 0.0, 0.0), (0.0, -0.6, 0.0, 0.0), (0.0, 0.0, 0.3, 0.0),
                                  (0.0, 0.0, 0.0, 0.1), (0.3, -0.6, 0.3, -0.2)])
def test_self_registration_ka5(ctx, oracle, pair_scene, pert):
    """registration_test_bench protocol on the GPU, against the oracle solve of the same problem."""
    from voxgraph_b200 import api
    s = pair_scene.submaps[0]
    ctx.submap_upload(10, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
    ctx.submap_upload(11, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
    ctx.submap_upload_points(10, 1, s.points_xyz, s.points_distance, s.points_weight)
    pg = api.PoseGraph(ctx)
    pg.addSubmapNode(api.SubmapNodeConfig(10, s.pose_gt, set_constant=True))
    pg.addSubmapNode(api.SubmapNodeConfig(11, s.pose_gt + np.array(pert), set_constant=False))
    # test-bench mode: a single (reference -> reading) residual block, no mirroring
    ctx_cfg = api.RegistrationConstraintConfig(10, 11, registration_point_type=api.K_VOXELS)
    ctx.submap_upload_points(10, api.K_VOXELS, s.points_xyz, s.points_distance, s.points_weight)
    pg.addRegistrationConstraint(ctx_cfg)
    pg.solver_options = ctx.solver_options(parameter_tolerance=3e-9, max_num_iterations=40)
    summ = pg.optimize()
    og = oracle.Graph()
    og.add_node(0, s.pose_gt, constant=True)
    og.add_node(1, s.pose_gt + np.array(pert))
    og.add_registration(0, 1, oracle_layer(oracle, s), s.points_xyz, s.points_distance, s.points_weight)
    rc, so = og.solve(oracle.solver_options(parameter_tolerance=3e-9, max_num_iterations=40))
    xg = pg.getSubmapPoses()[11]; xo = og.poses()[1]
    err = xg - s.pose_gt
    assert np.abs(err[:3]).max() < 0.02 and abs(err[3]) < 0.005
    # both at a tight tolerance: 1e-5 (BASELINE.md parity gate)
    assert np.abs(xg[:3] - xo[:3]).max() < 1e-5 and abs(_wrap(xg[3] - xo[3])) < 1e-5
    assert abs(summ.final_cost - so.final_cost) <= 1e-6 * max(so.final_cost, 1e-12) + 1e-12


def _graphs(ctx, oracle, sc, api):
    for s in sc.submaps:
        ctx.upload_synth_submap(s)
    pg = api.PoseGraph(ctx); og = oracle.Graph()
    layers = [oracle_layer(oracle, s) for s in sc.submaps]
    for i in range(len(sc.submaps)):
        pg.addSubmapNode(api.SubmapNodeConfig(i, sc.poses_init[i], set_constant=(i == 0)))
        og.add_node(i, sc.poses_init[i], constant=(i == 0))
    L = oracle.sqrt_information(sc.odom_information)
    for (i, j, t, y) in sc.odometry:
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(i, j, np.array([*t, y]),
                                                                      sc.odom_information))
        og.add_relative(i, j, t, y, L)
    for (i, j) in sc.pairs:
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(i, j))
        a, b = sc.submaps[i], sc.submaps[j]
        og.add_registration(i, j, layers[j], a.points_xyz, a.points_distance, a.points_weight)
        og.add_registration(j, i, layers[i], b.points_xyz, b.points_distance, b.points_weight)
    return pg, og


def test_config1_pair_solve(ctx, oracle, pair_scene):
    """BASELINE config 1 (2 submaps, 1k points, one mirrored registration constraint + odometry)
    at the reference's solver options (pose_graph.cpp:91-97)."""
    from voxgraph_b200 import api
    pg, og = _graphs(ctx, oracle, pair_scene, api)
    s = pg.optimize()
    rc, so = og.solve(oracle.solver_options(num_threads=4))
    assert rc == 0
    xg = np.array([pg.getSubmapPoses()[i] for i in range(2)]); xo = og.poses()
    assert np.abs(xg[:, :3] - xo[:, :3]).max() < 3e-3
    assert np.abs(_wrap(xg[:, 3] - xo[:, 3])).max() < 3e-3
    assert s.final_cost < s.initial_cost
    assert abs(s.initial_cost - so.initial_cost) <= 1e-8 * so.initial_cost


def test_small_graph_solve_matches_oracle(ctx, oracle, small_scene):
    from voxgraph_b200 import api
    sc = small_scene
    pg, og = _graphs(ctx, oracle, sc, api)
    s = pg.optimize()
    rc, so = og.solve(oracle.solver_options(num_threads=4))
    assert rc == 0
    n = len(sc.submaps)
    xg = np.array([pg.getSubmapPoses()[i] for i in range(n)]); xo = og.poses()
    assert np.abs(xg[:, :3] - xo[:, :3]).max() < 3e-3
    assert np.abs(_wrap(xg[:, 3] - xo[:, 3])).max() < 3e-3
    assert abs(s.final_cost - so.final_cost) <= 1e-3 * so.final_cost
    # tight tolerance from the same start
    pg2, og2 = _graphs(ctx, oracle, sc, api)
    pg2.solver_options = ctx.solver_options(parameter_tolerance=1e-9, function_tolerance=1e-12,
                                            max_num_iterations=200)
    s2 = pg2.optimize()
    rc, so2 = og2.solve(oracle.solver_options(parameter_tolerance=1e-9, function_tolerance=1e-12,
                                              max_num_iterations=200, num_threads=4))
    xg = np.array([pg2.getSubmapPoses()[i] for i in range(n)]); xo = og2.poses()
    assert np.abs(xg[:, :3] - xo[:, :3]).max() < 1e-4
    assert np.abs(_wrap(xg[:, 3] - xo[:, 3])).max() < 1e-4
    # excluded registration (pre-optimisation after loop closures, pose_graph_interface.cpp:182-188)
    pg3, og3 = _graphs(ctx, oracle, sc, api)
    s3 = pg3.optimize(exclude_registration_constraints=True)
    rc, so3 = og3.solve(oracle.solver_options(exclude_registration=1))
    xg = np.array([pg3.getSubmapPoses()[i] for i in range(n)]); xo = og3.poses()
    assert np.abs(xg - xo).max() < 1e-6


@pytest.mark.parametrize("n", [9, 40, 200])
def test_large_relative_pose_graph(ctx, oracle, n):
    """Dense-solver sizes up to BASELINE configs[3] (200 nodes -> 796 unknowns): chain + random
    loop closures with noisy measurements; GPU LM == oracle LM (same schedule, same solution)."""
    from voxgraph_b200 import api
    rs = np.random.RandomState(n)
    gt = np.cumsum(np.concatenate([np.zeros((1, 4)), rs.normal(0, 1, (n - 1, 4)) * [2, 2, 0.1, 0.3]]), 0)
    gt[:, 3] = _wrap(gt[:, 3])
    info = np.diag([1.0, 1.0, 2500.0, 2500.0])
    L = oracle.sqrt_information(info)
    pg = api.PoseGraph(ctx); og = oracle.Graph()
    for i in range(n):
        init = gt[i] + (0 if i == 0 else rs.normal(0, 0.2, 4) * [1, 1, 0.1, 0.1])
        pg.addSubmapNode(api.SubmapNodeConfig(i, init, set_constant=(i == 0)))
        og.add_node(i, init, constant=(i == 0))
    edges = [(i, i + 1) for i in range(n - 1)] + [tuple(sorted(rs.choice(n, 2, replace=False))) for _ in range(3 * n)]
    for (i, j) in edges:
        if i == j:
            continue
        t, y = synth.relative_pose(gt[i], gt[j])
        t = t + rs.normal(0, 0.02, 3); y = y + rs.normal(0, 0.002)
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(int(i), int(j), np.array([*t, y]), info))
        og.add_relative(int(i), int(j), t, y, L)
    ok, cg_, gg, Hg = pg.evaluate()
    ok, co, go_, Ho = og.eval()
    np.testing.assert_allclose(cg_, co, rtol=1e-11)
    np.testing.assert_allclose(Hg, Ho, rtol=1e-9, atol=1e-9 * np.abs(Ho).max())
    opts = dict(parameter_tolerance=1e-10, function_tolerance=1e-14, max_num_iterations=100)
    pg.solver_options = ctx.solver_options(**opts)
    s = pg.optimize()
    rc, so = og.solve(oracle.solver_options(num_threads=1, **opts))
    assert rc == 0
    xg = np.array([pg.getSubmapPoses()[i] for i in range(n)]); xo = og.poses()
    assert np.abs(xg[:, :3] - xo[:, :3]).max() < 1e-7
    assert np.abs(_wrap(xg[:, 3] - xo[:, 3])).max() < 1e-7
    assert abs(s.final_cost - so.final_cost) <= 1e-8 * max(so.final_cost, 1e-9)
    assert abs(s.iterations - so.iterations) <= 1


def test_height_constraints_via_reference_frame(ctx, oracle):
    """AbsolutePoseConstraint (height measurement, information only on z; LDLT sqrt) between a
    constant reference-frame node and submap nodes, mixed with odometry."""
    from voxgraph_b200 import api
    rs = np.random.RandomState(5)
    n = 6
    gt = np.stack([np.arange(n) * 2.0, np.sin(np.arange(n)), np.linspace(0.5, 1.5, n), np.linspace(0, 1, n)], -1)
    info_odo = np.diag([1.0, 1.0, 2500.0, 2500.0])
    info_h = np.zeros((4, 4)); info_h[2, 2] = 2500.0
    pg = api.PoseGraph(ctx); og = oracle.Graph()
    pg.addReferenceFrameNode(api.ReferenceFrameNodeConfig(0))
    og.add_node(api.FRAME_NODE_ID_BASE, np.zeros(4), constant=True)
    for i in range(n):
        init = gt[i] + (0 if i == 0 else rs.normal(0, 0.2, 4) * [1, 1, 1, 0.1])
        pg.addSubmapNode(api.SubmapNodeConfig(i, init, set_constant=(i == 0)))
        og.add_node(i, init, constant=(i == 0))
    L = oracle.sqrt_information(info_odo); Lh = oracle.sqrt_information_ldlt(info_h)
    for i in range(n - 1):
        t, y = synth.relative_pose(gt[i], gt[i + 1])
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(i, i + 1, np.array([*t, y]), info_odo))
        og.add_relative(i, i + 1, t, y, L)
    for i in range(1, n):
        pg.addAbsolutePoseConstraint(api.AbsolutePoseConstraintConfig(
            0, i, np.array([0.0, 0.0, gt[i, 2] + 0.01, 0.0]), info_h,
            allow_semi_definite_information_matrix=True))
        og.add_relative(api.FRAME_NODE_ID_BASE, i, np.array([0.0, 0.0, gt[i, 2] + 0.01]), 0.0, Lh)
    ok, cg_, gg, Hg = pg.evaluate()
    ok, co, go_, Ho = og.eval()
    # node order: the mirror sorts by id (submaps, then the frame node); the oracle has the frame first
    perm = np.r_[np.arange(4, 4 * (n + 1)), np.arange(4)]
    np.testing.assert_allclose(cg_, co, rtol=1e-12)
    np.testing.assert_allclose(gg, go_[perm], rtol=1e-10, atol=1e-9)
    np.testing.assert_allclose(Hg, Ho[np.ix_(perm, perm)], rtol=1e-10, atol=1e-9)
    opts = dict(parameter_tolerance=1e-10, function_tolerance=1e-14, max_num_iterations=100)
    pg.solver_options = ctx.solver_options(**opts)
    s = pg.optimize()
    rc, so = og.solve(oracle.solver_options(**opts))
    xg = np.array([pg.getSubmapPoses()[i] for i in range(n)]); xo = og.poses()[1:]
    assert np.abs(xg - xo).max() < 1e-7
    assert np.abs(xg[1:, 2] - (gt[1:, 2] + 0.01)).max() < 0.02   # heights pulled to the measurements


def test_solver_errors(ctx, oracle):
    from voxgraph_b200 import api
    pg = api.PoseGraph(ctx)
    pg.addSubmapNode(api.SubmapNodeConfig(0, np.zeros(4), True))
    with pytest.raises(ValueError):
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(0, 0))
    with pytest.raises(ValueError):
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(0, 5))
    with pytest.raises(ValueError):
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(0, 1, np.zeros(4), -np.eye(4)))


def test_edge_covariances_match_inverse_normal_matrix(ctx, oracle, small_scene):
    """PoseGraph::getEdgeCovarianceMap (pose_graph.cpp:117-163): blocks of (J^T J)^-1 over the free
    nodes, as ceres::Covariance reports them, vs numpy on the oracle's J^T J."""
    from voxgraph_b200 import api
    sc = small_scene
    for s in sc.submaps:
        ctx.upload_synth_submap(s)
    pg = api.PoseGraph(ctx); og = oracle.Graph()
    layers = [oracle.Layer.from_blocks(s.voxel_size, s.vps, s.block_idx, s.distance, s.weight) for s in sc.submaps]
    n = len(sc.submaps)
    for i in range(n):
        pg.addSubmapNode(api.SubmapNodeConfig(i, sc.poses_init[i], set_constant=(i == 0)))
        og.add_node(i, sc.poses_init[i], constant=(i == 0))
    L = oracle.sqrt_information(sc.odom_information)
    for (i, j, t, y) in sc.odometry:
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(i, j, np.array([*t, y]), sc.odom_information))
        og.add_relative(i, j, t, y, L)
    for (i, j) in sc.pairs:
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(i, j))
        a, b = sc.submaps[i], sc.submaps[j]
        og.add_registration(i, j, layers[j], a.points_xyz, a.points_distance, a.points_weight)
        og.add_registration(j, i, layers[i], b.points_xyz, b.points_distance, b.points_weight)
    ok, cost, g, H = og.eval(num_threads=2)
    free = np.arange(4, 4 * n)                      # node 0 is constant
    Cov = np.linalg.inv(H[np.ix_(free, free)])
    pairs = [(1, 2), (2, 1), (3, 3), (1, n - 1), (0, 2), (2, 0)]
    got = pg.getEdgeCovarianceMap(pairs)
    scale = np.abs(Cov).max()
    for (a, b) in pairs:
        if a == 0 or b == 0:
            assert np.all(got[(a, b)] == 0)          # constant block: zero covariance
            continue
        want = Cov[4 * (a - 1):4 * a, 4 * (b - 1):4 * b]
        assert np.abs(got[(a, b)] - want).max() <= 1e-7 * scale, (a, b)
    assert np.allclose(got[(1, 2)], got[(2, 1)].T, atol=1e-9 * scale)
    with pytest.raises(api.VgxError):
        ctx.graph_edge_covariances([1], [99])
