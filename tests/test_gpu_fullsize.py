"""Full-size (BASELINE configs[1]: 50 submaps / 200 pairs / 10 k points, 4 M residuals) property
checks of the CUDA path — sizes where running the oracle on everything would take too long for a
unit test, so parity is established through size-independent properties:
  * the fused reduce path equals the sum of J^T J / J^T r / r^2 over the Ceres-layout output of the
    emit path (itself bit-exact against the oracle at small sizes), constraint by constraint;
  * a sample of constraints is checked against the oracle directly;
  * run-to-run bit reproducibility;
  * TSDF: the ray-ordered integrator is a pure function of its inputs (two fresh submaps agree
    bit for bit) and does exactly the work the lock-free one does.
"""
import numpy as np
import pytest

from support import ctx  # noqa: F401
from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def config2_scene():
    return synth.make_scene(seed=2, n_submaps=50, n_points=10000, voxel_size=0.2, max_pairs=200,
                            trunc=0.6, drift=(0.03, 0.005, 0.002))


def test_config2_fused_equals_sum_of_emit(ctx, oracle, config2_scene):
    from voxgraph_b200 import api
    sc = config2_scene
    assert len(sc.pairs) == 200
    for s in sc.submaps:
        ctx.upload_synth_submap(s)
    pg = api.PoseGraph(ctx)
    n = len(sc.submaps)
    for i in range(n):
        pg.addSubmapNode(api.SubmapNodeConfig(i, sc.poses_init[i], set_constant=(i == 0)))
    for (i, j) in sc.pairs:
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(i, j))
    ok, cost, g, H = pg.evaluate()
    assert ok
    local, glob = ctx.graph_num_registration_residuals()
    assert glob == 4_000_000 and local == glob
    # ---- sum of the emit path, block by block
    dim = 4 * n
    Hx = np.zeros((dim, dim)); gx = np.zeros(dim); cx = 0.0
    per_edge = []
    for (a, b) in pg.registration_blocks:
        ok2, r, jr, je = ctx.reg_eval_emit(a, b, sc.poses_init[a], sc.poses_init[b])
        assert ok2
        J = np.concatenate([jr, je], axis=1)          # K x 8
        blk = J.T @ J; gb = J.T @ r
        ia = slice(4 * a, 4 * a + 4); ib = slice(4 * b, 4 * b + 4)
        Hx[ia, ia] += blk[:4, :4]; Hx[ib, ib] += blk[4:, 4:]
        Hx[ia, ib] += blk[:4, 4:]; Hx[ib, ia] += blk[4:, :4]
        gx[ia] += gb[:4]; gx[ib] += gb[4:]
        cx += 0.5 * float(r @ r)
        per_edge.append(float(r @ r))
    # device pose set-up rounds the float trig from double, the host emit path uses libm: <= 1 ulp
    assert abs(cost - cx) <= 1e-5 * cx
    assert np.abs(H - Hx).max() <= 1e-5 * np.abs(Hx).max()
    assert np.abs(g - gx).max() <= 1e-5 * np.abs(gx).max()
    np.testing.assert_allclose(pg.getVisualizationEdgeResiduals(), per_edge, rtol=1e-5)
    assert np.allclose(H, H.T, rtol=0, atol=1e-9 * np.abs(H).max())
    # ---- a sample of residual blocks against the oracle (bit-exact emit path)
    for (a, b) in pg.registration_blocks[::67]:
        sa, sb = sc.submaps[a], sc.submaps[b]
        layer = oracle.Layer.from_blocks(sb.voxel_size, sb.vps, sb.block_idx, sb.distance, sb.weight)
        ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(layer, sa.points_xyz, sa.points_distance,
                                                    sa.points_weight, sc.poses_init[a], sc.poses_init[b])
        ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(a, b, sc.poses_init[a], sc.poses_init[b])
        assert ok_o and ok_g
        assert np.array_equal(r_g, r_o) and np.array_equal(jr_g, jr_o) and np.array_equal(je_g, je_o)
    # ---- bit reproducibility of the fused path at full size
    ok, cost2, g2, H2 = pg.evaluate()
    assert cost2 == cost and np.array_equal(g2, g) and np.array_equal(H2, H)


def test_full_scan_ray_ordered_is_deterministic(ctx):
    """64 x 1024 LiDAR scan (BASELINE configs[2] shape): two fresh submaps integrated with the
    ray-ordered path agree bit for bit."""
    world = synth.make_world(2, size_xy=(120.0, 80.0), n_clutter=400, n_walls=24)
    pts = synth.lidar_scan(world, np.array([60.0, 40.0, 1.2, 0.3]), n_beams=64, n_azimuth=1024, seed=3,
                           miss_range=40.0)
    assert pts.shape[0] == 65536
    T = synth.pose_to_T([0, 0, 0, 0])
    out = []
    stats = []
    for sid, det in ((500, 1), (501, 1), (502, 0)):
        ctx.submap_create(sid, 0.2, 16, 8192)
        st = ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(mode=0, deterministic=det))
        assert st.saturated_batches > 1000
        stats.append((st.rays_valid, st.rays_cast, st.voxel_updates, st.blocks_allocated))
        out.append(ctx.submap_download(sid))
    assert stats[0] == stats[1] == stats[2]
    assert stats[0][2] > 3_000_000
    (i0, d0, w0), (i1, d1, w1), (i2, d2, w2) = out
    # block allocation order is racy (atomic counter): compare by block index
    def by_block(idx, d, w):
        order = np.lexsort((idx[:, 0], idx[:, 1], idx[:, 2]))
        return idx[order], d[order], w[order]
    a = by_block(i0, d0, w0); b = by_block(i1, d1, w1); c = by_block(i2, d2, w2)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert np.array_equal(a[0], c[0]) and np.array_equal(a[2] > 0, c[2] > 0)
    for sid in (500, 501, 502):
        ctx.submap_free(sid)
