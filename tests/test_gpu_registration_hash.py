"""GPU parity of the fused registration reduction on its hash path: reading submaps whose block
AABB is too large for the shared-memory block grid look their blocks up in the hash instead."""
import numpy as np
import pytest

from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu

GRID_MAX_CELLS = 4096   # larger block AABBs get no block grid (submap.cu, VGX_GRID_MAX_CELLS)


def test_reduce_hash_path_matches_oracle(oracle):
    from voxgraph_b200 import api
    world = synth.make_world(7, size_xy=(16.0, 14.0), n_clutter=20, n_walls=2)
    a = synth.make_submap(world, 420, np.array([8.0, 7.0, 1.0, 0.2]), 0.05, 8, 6.0, n_points=3000)
    b = synth.make_submap(world, 421, np.array([8.6, 7.3, 1.0, -0.4]), 0.05, 8, 6.0, n_points=3000)
    for s in (a, b):
        cells = int(np.prod(s.block_idx.max(0) - s.block_idx.min(0) + 1))
        assert cells > GRID_MAX_CELLS
    ctx = api.Context(0)
    try:
        for s in (a, b):
            ctx.upload_synth_submap(s)
        ref = a.pose_gt + np.array([0.03, -0.02, 0.01, 0.01]); read = b.pose_gt
        pg = api.PoseGraph(ctx); og = oracle.Graph()
        la = oracle.Layer.from_blocks(a.voxel_size, a.vps, a.block_idx, a.distance, a.weight)
        lb = oracle.Layer.from_blocks(b.voxel_size, b.vps, b.block_idx, b.distance, b.weight)
        for sid, pose, cst in ((420, ref, True), (421, read, False)):
            pg.addSubmapNode(api.SubmapNodeConfig(sid, pose, set_constant=cst))
            og.add_node(sid, pose, constant=cst)
        pg.addRegistrationConstraint(api.RegistrationConstraintConfig(420, 421))
        og.add_registration(420, 421, lb, a.points_xyz, a.points_distance, a.points_weight)
        og.add_registration(421, 420, la, b.points_xyz, b.points_distance, b.points_weight)
        ok_g, cost_g, g_g, H_g = pg.evaluate()
        ok_o, cost_o, g_o, H_o = og.eval(num_threads=4)
        assert ok_g and ok_o and cost_o > 0
        # tolerances of test_reduce_mode_matches_oracle
        assert abs(cost_g - cost_o) <= 1e-9 * abs(cost_o)
        assert np.abs(g_g - g_o).max() <= 1e-7 * np.abs(g_o).max()
        assert np.abs(H_g - H_o).max() <= 1e-7 * np.abs(H_o).max()
    finally:
        ctx.close()
