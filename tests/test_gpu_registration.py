"""GPU parity: CUDA registration path (through the C-ABI) vs the CPU oracle."""
import numpy as np
import pytest

from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu

VS, VPS = 0.2, 16


@pytest.fixture(scope="module")
def ctx():
    from voxgraph_b200 import api
    c = api.Context(0)
    yield c
    c.close()


def _olayer(oracle, s):
    return oracle.Layer.from_blocks(s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)


def _bit_equal(a, b):
    return np.array_equal(a, b)  # -0.0 == 0.0


def test_emit_bit_exact_pair_scene(ctx, oracle, pair_scene):
    """Config 1: single registration constraint, Ceres layout, bit-exact vs the oracle."""
    for s in pair_scene.submaps:
        ctx.upload_synth_submap(s)
    s0, s1 = pair_scene.submaps
    for (a, b) in ((s0, s1), (s1, s0)):
        layer = _olayer(oracle, b)
        ia, ib = a.submap_id, b.submap_id
        ref, read = pair_scene.poses_init[ia], pair_scene.poses_init[ib]
        ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(layer, a.points_xyz, a.points_distance,
                                                    a.points_weight, ref, read)
        ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(ia, ib, ref, read)
        assert ok_o and ok_g
        assert (np.abs(jr_o).sum(1) > 0).sum() > 500  # most points have a correspondence
        assert _bit_equal(r_g, r_o)
        assert _bit_equal(jr_g, jr_o)
        assert _bit_equal(je_g, je_o)
        # residual-only call (jacobians == nullptr)
        ok_g2, r_g2, _, _ = ctx.reg_eval_emit(ia, ib, ref, read, jacobians=False)
        assert ok_g2 and _bit_equal(r_g2, r_o)


def test_emit_bit_exact_many_poses(ctx, oracle, small_scene):
    """Scaled-down config 2: every pair, both directions, at perturbed poses incl. yaw near +-pi."""
    sc = small_scene
    for s in sc.submaps:
        ctx.upload_synth_submap(s)
    layers = [_olayer(oracle, s) for s in sc.submaps]
    rs = np.random.RandomState(0)
    n_checked = 0
    for (i, j) in sc.pairs:
        for (a, b) in ((i, j), (j, i)):
            ref = sc.poses_init[a] + rs.normal(0, 0.05, 4)
            read = sc.poses_init[b] + rs.normal(0, 0.05, 4)
            sa = sc.submaps[a]
            ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(layers[b], sa.points_xyz, sa.points_distance,
                                                        sa.points_weight, ref, read)
            ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(a, b, ref, read)
            assert ok_o == ok_g
            assert _bit_equal(r_g, r_o) and _bit_equal(jr_g, jr_o) and _bit_equal(je_g, je_o)
            n_checked += len(r_o)
    assert n_checked >= 10000


def test_emit_plane_closed_form_and_edges(ctx, oracle):
    """KA1/KA7 on the GPU: plane field, missing blocks, unobserved voxel, block-face crossings,
    negative block indices, ragged point counts (1, 255, 257, 2049)."""
    n = np.array([0.3, -0.5, 0.81]); n /= np.linalg.norm(n)
    idx, d, w = synth.plane_layer_blocks(n, 0.17, VS, VPS, ((-2, 1), (-2, 1), (-1, 0)))
    w = w.copy()
    w[3, 5 + 16 * (5 + 16 * 5)] = 0.0     # one unobserved voxel
    w[7, :64] = 1e-7                      # weights below the isObserved threshold
    layer = oracle.Layer.from_blocks(VS, VPS, idx, d, w)
    ctx.submap_upload(100, VS, VPS, idx, d, w)
    rs = np.random.RandomState(1)
    for k in (1, 255, 257, 2049):
        xyz = rs.uniform(-7.5, 4.5, (k, 3)).astype(np.float32)   # some fall outside the layer
        xyz[:, 2] = rs.uniform(-3.5, 0.5, k)
        # a few exactly on voxel / block boundaries
        xyz[: min(k, 8)] = np.round(xyz[: min(k, 8)] / 0.2) * 0.2
        dist = rs.uniform(-0.1, 0.1, k).astype(np.float32)
        wt = rs.uniform(0.5, 2.0, k).astype(np.float32)
        ctx.submap_upload(101, VS, VPS, idx[:1], d[:1], w[:1])
        ctx.submap_upload_points(101, 1, xyz, dist, wt)
        ref = np.array([0.4, -0.2, 0.1, 3.1]); read = np.array([-0.3, 0.5, -0.05, -3.0])
        cfg = ctx.reg_config(no_correspondence_cost=0.3)
        ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(layer, xyz, dist, wt, ref, read,
                                                    no_correspondence_cost=0.3)
        ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(101, 100, ref, read, cfg)
        assert ok_o and ok_g
        assert _bit_equal(r_g, r_o) and _bit_equal(jr_g, jr_o) and _bit_equal(je_g, je_o)
    no_corr = (np.abs(jr_o).sum(1) == 0)
    assert 0 < no_corr.sum() < len(no_corr)


@pytest.mark.parametrize("voxel_size,vps", [(0.1, 16), (0.05, 8), (0.4, 32)])
def test_emit_other_voxel_sizes_and_block_sizes(ctx, oracle, voxel_size, vps):
    """BASELINE configs[3..4] voxel sizes (0.10 m, 0.05 m) and non-default voxels_per_side."""
    world = synth.make_world(7, size_xy=(16.0, 14.0), n_clutter=20, n_walls=2)
    r = 3.0 if voxel_size < 0.2 else 6.0
    a = synth.make_submap(world, 400, np.array([8.0, 7.0, 1.0, 0.2]), voxel_size, vps, r, n_points=3000)
    b = synth.make_submap(world, 401, np.array([8.6, 7.3, 1.0, -0.4]), voxel_size, vps, r, n_points=3000)
    for s_ in (a, b):
        ctx.upload_synth_submap(s_)
    layer = oracle.Layer.from_blocks(b.voxel_size, b.vps, b.block_idx, b.distance, b.weight)
    ref = a.pose_gt + np.array([0.03, -0.02, 0.01, 0.01]); read = b.pose_gt
    ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(layer, a.points_xyz, a.points_distance, a.points_weight, ref, read)
    ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(400, 401, ref, read)
    assert ok_o and ok_g and (np.abs(jr_o).sum(1) > 0).sum() > 300
    assert _bit_equal(r_g, r_o) and _bit_equal(jr_g, jr_o) and _bit_equal(je_g, je_o)
    # and through the fused path (shared-memory block grid + octets)
    from voxgraph_b200 import api
    pg = api.PoseGraph(ctx); og = oracle.Graph()
    la = oracle.Layer.from_blocks(a.voxel_size, a.vps, a.block_idx, a.distance, a.weight)
    for sid, pose, cst in ((400, ref, True), (401, read, False)):
        pg.addSubmapNode(api.SubmapNodeConfig(sid, pose, set_constant=cst)); og.add_node(sid, pose, constant=cst)
    pg.addRegistrationConstraint(api.RegistrationConstraintConfig(400, 401))
    og.add_registration(400, 401, layer, a.points_xyz, a.points_distance, a.points_weight)
    og.add_registration(401, 400, la, b.points_xyz, b.points_distance, b.points_weight)
    ok, cg_, gg, Hg = pg.evaluate(); ok, co, go_, Ho = og.eval()
    assert abs(cg_ - co) <= 1e-9 * co and np.abs(Hg - Ho).max() <= 1e-7 * np.abs(Ho).max()


def test_esdf_style_layer_observed_flag(ctx, oracle):
    """Default voxgraph registers against the ESDF (use_esdf_distance = true): the layer is uploaded
    with weight = observed ? 1 : 0 and euclidean (untruncated) distances."""
    rs = np.random.RandomState(11)
    fn = lambda p: np.linalg.norm(p - np.array([1.0, 0.5, 0.2]), axis=1) - 1.5   # sphere ESDF
    idx, d, w = synth.field_layer_blocks(fn, VS, VPS, ((-1, 1), (-1, 1), (-1, 0)))
    w = (rs.uniform(size=w.shape) > 0.02).astype(np.float32)      # 2 % unobserved voxels
    layer = oracle.Layer.from_blocks(VS, VPS, idx, d, w)
    ctx.submap_upload(410, VS, VPS, idx, d, w)
    xyz = rs.uniform(-3.0, 4.0, (4000, 3)).astype(np.float32); xyz[:, 2] = rs.uniform(-2.5, 1.0, 4000)
    ctx.submap_upload(411, VS, VPS, idx[:1], d[:1], w[:1])
    ctx.submap_upload_points(411, 0, xyz, np.zeros(4000, np.float32), np.ones(4000, np.float32))
    cfg = ctx.reg_config(registration_point_type=0)
    ref = np.array([0.1, 0.0, 0.05, 0.3]); read = np.array([0.0, 0.1, 0.0, -0.2])
    ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(layer, xyz, np.zeros(4000, np.float32),
                                                np.ones(4000, np.float32), ref, read)
    ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(411, 410, ref, read, cfg)
    assert ok_o and ok_g
    nz = (np.abs(jr_o).sum(1) > 0)
    assert 500 < nz.sum() < 3990          # some points hit unobserved corners / leave the layer
    assert _bit_equal(r_g, r_o) and _bit_equal(jr_g, jr_o) and _bit_equal(je_g, je_o)


def test_emit_zero_weight_and_errors(ctx, oracle):
    from voxgraph_b200 import api
    idx, d, w = synth.plane_layer_blocks([0, 0, 1.0], 0.0, VS, VPS, ((0, 0), (0, 0), (0, 0)))
    ctx.submap_upload(200, VS, VPS, idx, d, w)
    ctx.submap_upload(201, VS, VPS, idx, d, w)
    xyz = np.array([[1.0, 1.0, 1.0], [2.0, 2.0, 2.0]], np.float32)
    ctx.submap_upload_points(201, 1, xyz, np.zeros(2, np.float32), np.zeros(2, np.float32))
    ok, r, _, _ = ctx.reg_eval_emit(201, 200, np.zeros(4), np.zeros(4))
    assert not ok   # Evaluate returns false on zero summed weight (cpp:273)
    # no points at all
    ctx.submap_upload_points(201, 1, np.zeros((0, 3), np.float32), np.zeros(0, np.float32),
                             np.zeros(0, np.float32))
    assert ctx.reg_num_residuals(201) == 0
    ok, r, _, _ = ctx.reg_eval_emit(201, 200, np.zeros(4), np.zeros(4))
    assert not ok
    with pytest.raises(api.VgxError):
        ctx.reg_eval_emit(201, 999, np.zeros(4), np.zeros(4))       # unknown submap
    with pytest.raises(api.VgxError):
        ctx.reg_eval_emit(200, 200, np.zeros(4), np.zeros(4))       # submap against itself
    with pytest.raises(api.VgxError):
        ctx.reg_eval_emit(201, 200, np.zeros(4), np.zeros(4), ctx.reg_config(sampling_ratio=-0.5))


def _build_graphs(ctx, oracle, sc, api):
    for s in sc.submaps:
        ctx.upload_synth_submap(s)
    pg = api.PoseGraph(ctx)
    og = oracle.Graph()
    layers = [_olayer(oracle, s) for s in sc.submaps]
    for i, s in enumerate(sc.submaps):
        pg.addSubmapNode(api.SubmapNodeConfig(i, sc.poses_init[i], set_constant=(i == 0)))
        og.add_node(i, sc.poses_init[i], constant=(i == 0))
    L = oracle.sqrt_information(sc.odom_information)
    for (i, j, t, y) in sc.odometry:
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(
            i, j, np.array([t[0], t[1], t[2], y]), sc.odom_information))
        og.add_relative(i, j, t, y, L)
    for (i, j) in sc.pairs:
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(i, j))
        a, b = sc.submaps[i], sc.submaps[j]
        og.add_registration(i, j, layers[j], a.points_xyz, a.points_distance, a.points_weight)
        og.add_registration(j, i, layers[i], b.points_xyz, b.points_distance, b.points_weight)
    return pg, og


def test_reduce_mode_matches_oracle(ctx, oracle, small_scene):
    """Fused J^T J / J^T r / cost of the whole problem vs what Ceres would assemble."""
    from voxgraph_b200 import api
    pg, og = _build_graphs(ctx, oracle, small_scene, api)
    ok_g, cost_g, g_g, H_g = pg.evaluate()
    ok_o, cost_o, g_o, H_o = og.eval(num_threads=4)
    assert ok_g and ok_o
    # tolerance: BASELINE.md parity gate is 1e-4 relative; device trig may differ from libm by 1 ulp
    assert abs(cost_g - cost_o) <= 1e-9 * abs(cost_o)
    scale_g = np.abs(g_o).max(); scale_H = np.abs(H_o).max()
    assert np.abs(g_g - g_o).max() <= 1e-7 * scale_g
    assert np.abs(H_g - H_o).max() <= 1e-7 * scale_H
    # per-edge residual sums (pose_graph.cpp:194-207)
    per_g = pg.getVisualizationEdgeResiduals()
    per_o = og.registration_costs(len(per_g))
    np.testing.assert_allclose(per_g, per_o, rtol=1e-9)
    # excluding registration constraints (PoseGraph::optimize(true))
    ok_g, cost_g2, g_g2, H_g2 = pg.evaluate(exclude_registration_constraints=True)
    ok_o, cost_o2, g_o2, H_o2 = og.eval(exclude_registration=True)
    assert abs(cost_g2 - cost_o2) <= 1e-12 * max(1.0, abs(cost_o2))
    np.testing.assert_allclose(H_g2, H_o2, rtol=1e-10, atol=1e-10 * np.abs(H_o2).max())
    # run-to-run bit reproducibility of the fused reduction
    ok_g, cost_g3, g_g3, H_g3 = pg.evaluate()
    assert cost_g3 == cost_g and np.array_equal(g_g3, g_g) and np.array_equal(H_g3, H_g)


def test_device_pose_setup_matches_host(ctx, oracle, pair_scene):
    """Reduce mode computes the float pose block on the device (double trig rounded once),
    emit mode on the host with libm: the two must agree to ~1 ulp in the sums.  At arbitrary poses
    only; tests/test_gpu_reduce_exact.py pins the fused sums to the exact sum of the oracle's terms
    at poses whose pose blocks agree bit for bit."""
    from voxgraph_b200 import api
    sc = pair_scene
    for s in sc.submaps:
        ctx.upload_synth_submap(s)
    pg = api.PoseGraph(ctx)
    for i in range(2):
        pg.addSubmapNode(api.SubmapNodeConfig(i, sc.poses_init[i], set_constant=(i == 0)))
    pg.addRegistrationConstraint(api.RegistrationConstraintConfig(0, 1))
    ok, cost, g, H = pg.evaluate()
    tot = 0.0
    Hx = np.zeros((8, 8)); gx = np.zeros(8)
    for (a, b) in ((0, 1), (1, 0)):
        ok2, r, jr, je = ctx.reg_eval_emit(a, b, sc.poses_init[a], sc.poses_init[b])
        J = np.zeros((len(r), 8)); J[:, 4 * a:4 * a + 4] = jr; J[:, 4 * b:4 * b + 4] = je
        tot += 0.5 * r @ r; Hx += J.T @ J; gx += J.T @ r
    assert abs(cost - tot) <= 1e-6 * tot
    assert np.abs(H - Hx).max() <= 1e-6 * np.abs(Hx).max()
    assert np.abs(g - gx).max() <= 1e-6 * np.abs(gx).max()


# --------------------------------------------------------------------------- sampling mode
def test_draw_samples_match_reference_golden(ctx):
    """vgx_submap_draw_samples == voxgraph::WeightedSampler::getRandomItem of the reference itself
    (golden generated from the compiled reference header, tests/golden/make_sampler_golden.py)."""
    import json
    import os
    cases = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "weighted_sampler.json")))["cases"]
    idx, d, w = synth.plane_layer_blocks([0, 0, 1.0], 0.0, VS, VPS, ((0, 0), (0, 0), (0, 0)))
    for k, case in enumerate(cases):
        wts = np.array(case["weights"], np.float32)
        sid = 300 + k
        ctx.submap_upload(sid, VS, VPS, idx, d, w)
        n = len(wts)
        ctx.submap_upload_points(sid, 1, np.zeros((n, 3), np.float32), np.zeros(n, np.float32), wts)
        assert ctx.submap_draw_samples(sid, 1, 64).tolist() == case["draw_0_64"]
        assert ctx.submap_draw_samples(sid, 1, 64).tolist() == case["draw_64_128"]


def test_emit_sampling_mode_bit_exact(ctx, oracle, pair_scene):
    """sampling_ratio = 0.2 (registration_test_bench.yaml:27) and 0.05 (voxgraph_mapper.yaml:34):
    every Evaluate draws int(ratio*K) points from the reference submap's generator, weight 1."""
    for s in pair_scene.submaps:
        ctx.upload_synth_submap(s)      # fresh upload = fresh default-seeded generator
    s0, s1 = pair_scene.submaps
    layer = _olayer(oracle, s1)
    sampler = oracle.WeightedSampler(s0.points_weight)
    ref, read = pair_scene.poses_init[0], pair_scene.poses_init[1]
    for ratio in (0.2, 0.05, 0.2):
        cfg = ctx.reg_config(sampling_ratio=ratio)
        K = oracle.sampled_num_residuals(ratio, len(s0.points_weight))
        assert ctx.reg_num_residuals(0, cfg) == K
        idx = sampler.draw(K)           # the oracle's generator advances in lock-step
        ok_o, r_o, jr_o, je_o = oracle.reg_evaluate_sampled(layer, s0.points_xyz, s0.points_distance,
                                                            idx, ref, read)
        ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(0, 1, ref, read, cfg)
        assert ok_o and ok_g and len(r_g) == K
        assert _bit_equal(r_g, r_o) and _bit_equal(jr_g, jr_o) and _bit_equal(je_g, je_o)


def test_graph_sampling_mode_matches_oracle(ctx, oracle, small_scene):
    """The reference's production configuration (sampling_ratio 0.05) through the fused path: the
    indices the library drew (one draw per constraint-list build) feed the oracle."""
    from voxgraph_b200 import api
    sc = small_scene
    for s in sc.submaps:
        ctx.upload_synth_submap(s)
    pg = api.PoseGraph(ctx)
    og = oracle.Graph()
    layers = [_olayer(oracle, s) for s in sc.submaps]
    for i, s in enumerate(sc.submaps):
        pg.addSubmapNode(api.SubmapNodeConfig(i, sc.poses_init[i], set_constant=(i == 0)))
        og.add_node(i, sc.poses_init[i], constant=(i == 0))
    L = oracle.sqrt_information(sc.odom_information)
    for (i, j, t, y) in sc.odometry:
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(
            i, j, np.array([t[0], t[1], t[2], y]), sc.odom_information))
        og.add_relative(i, j, t, y, L)
    ratios = [0.05, 0.5]
    for k, (i, j) in enumerate(sc.pairs):
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(i, j, sampling_ratio=ratios[k % 2]))
    pg._sync()
    samplers = {i: oracle.WeightedSampler(s.points_weight) for i, s in enumerate(sc.submaps)}
    keep = []
    for k, (a, b) in enumerate(pg.registration_blocks):
        ratio = ratios[(k // 2) % 2]
        K = oracle.sampled_num_residuals(ratio, len(sc.submaps[a].points_weight))
        idx = ctx.graph_get_sample_indices(k, K)
        assert len(idx) == K
        # the library's draw is the reference sampler's stream of submap a, in list order
        assert np.array_equal(idx, samplers[a].draw(K))
        sa = sc.submaps[a]
        xyz = np.ascontiguousarray(sa.points_xyz[idx]); dd = np.ascontiguousarray(sa.points_distance[idx])
        ww = np.ones(K, np.float32)
        keep.append((xyz, dd, ww))
        og.add_registration(a, b, layers[b], xyz, dd, ww)
    ok_g, cost_g, g_g, H_g = pg.evaluate()
    ok_o, cost_o, g_o, H_o = og.eval(num_threads=2)
    assert ok_g and ok_o
    assert abs(cost_g - cost_o) <= 1e-9 * abs(cost_o)
    assert np.abs(g_g - g_o).max() <= 1e-7 * np.abs(g_o).max()
    assert np.abs(H_g - H_o).max() <= 1e-7 * np.abs(H_o).max()
    # the sample is frozen within a solve: evaluating again gives the identical numbers
    ok_g, cost_g2, g_g2, H_g2 = pg.evaluate()
    assert cost_g2 == cost_g and np.array_equal(H_g2, H_g)
    # explicit index list (vgx_graph_set_sample_indices)
    K0 = oracle.sampled_num_residuals(ratios[0], len(sc.submaps[pg.registration_blocks[0][0]].points_weight))
    ctx.graph_set_sample_indices(0, np.arange(K0, dtype=np.int32))
    assert np.array_equal(ctx.graph_get_sample_indices(0, K0), np.arange(K0))
    summ = pg.optimize()
    assert summ.final_cost <= summ.initial_cost
