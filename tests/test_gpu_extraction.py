"""GPU parity: registration-point extraction on resident bricks (vgx_submap_extract_points) vs the
oracle's findRelevantVoxelIndices / findIsosurfaceVertices / surface OBB - bit-exact, same order."""
import numpy as np
import pytest

from support import ctx  # noqa: F401
from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu

VS, VPS = 0.2, 16


def _check(ctx, oracle, sid, voxel_size, vps, idx, d, w, min_w=1.0, max_d=0.3):
    from voxgraph_b200 import api
    ctx.submap_upload(sid, voxel_size, vps, idx, d, w)
    ctx.submap_extract_points(sid, ctx.registration_filter(min_voxel_weight=min_w, max_voxel_distance=max_d))
    L = oracle.Layer.from_blocks(voxel_size, vps, idx, d, w)
    # relevant voxels: same points, same order
    xo, do_, wo = oracle.find_relevant_voxels(L, min_w, max_d)
    xg, dg, wg = ctx.submap_download_points(sid, api.K_VOXELS)
    assert xg.shape == xo.shape
    assert np.array_equal(xg, xo) and np.array_equal(dg, do_) and np.array_equal(wg, wo)
    ok_o, mn_o, mx_o = oracle.surface_obb(L, min_w, max_d)
    ok_g, mn_g, mx_g = ctx.submap_surface_obb(sid)
    assert ok_o == ok_g
    if ok_o:
        assert np.array_equal(mn_g, mn_o) and np.array_equal(mx_g, mx_o)
    # isosurface vertices
    xo, do_, wo, blk = oracle.find_isosurface_vertices(L, min_w)
    xg, dg, wg = ctx.submap_download_points(sid, api.K_ISOSURFACE_POINTS)
    assert xg.shape == xo.shape
    assert np.array_equal(xg, xo) and np.array_equal(dg, do_) and np.array_equal(wg, wo)
    return len(xo)


def test_plane_and_min_weight(ctx, oracle):
    idx, d, w = synth.plane_layer_blocks([0, 0, 1.0], 0.37, VS, VPS, ((0, 1), (0, 1), (-1, 0)))
    assert _check(ctx, oracle, 700, VS, VPS, idx, d, 2.0 * w) == 31 * 31
    assert _check(ctx, oracle, 701, VS, VPS, idx, d, w) == 0          # weight 1 is not > min_weight 1
    assert _check(ctx, oracle, 702, VS, VPS, idx, d, w, min_w=0.5) == 31 * 31


def test_tilted_plane_and_sphere(ctx, oracle):
    idx, d, w = synth.plane_layer_blocks([0.3, -0.2, 0.93], 1.1, VS, VPS, ((-1, 1), (-1, 1), (-1, 1)))
    assert _check(ctx, oracle, 703, VS, VPS, idx, d, 3.0 * w) > 1000
    c = np.array([1.7, 1.5, 1.6]); R = 1.3
    idx, d, w = synth.field_layer_blocks(lambda p: np.linalg.norm(p - c, axis=-1) - R, VS, VPS,
                                         ((0, 1), (0, 1), (0, 1)), weight=3.0)
    d = np.clip(d, -0.6, 0.6).astype(np.float32)
    assert _check(ctx, oracle, 704, VS, VPS, idx, d, w) > 500


@pytest.mark.parametrize("voxel_size,vps", [(0.1, 16), (0.15, 8), (0.05, 32)])
def test_scene_submap_other_resolutions(ctx, oracle, voxel_size, vps):
    world = synth.make_world(5, size_xy=(30.0, 24.0), n_clutter=60, n_walls=4)
    s = synth.make_submap(world, 0, np.array([14.0, 12.0, 1.0, 0.3]), voxel_size=voxel_size, vps=vps,
                          radius=3.0 if voxel_size < 0.1 else 5.0, n_points=None)
    n = _check(ctx, oracle, 705, voxel_size, vps, s.block_idx, s.distance, s.weight)
    assert n > 200


def test_extracted_points_feed_registration(ctx, oracle, pair_scene):
    """The points extracted on the device are what the cost function consumes: emit-mode residuals
    of (device-extracted reference points -> reading submap) are bit-exact vs the oracle fed with
    the oracle's own extraction."""
    from voxgraph_b200 import api
    s0, s1 = pair_scene.submaps
    for s in (s0, s1):
        ctx.submap_upload(710 + s.submap_id, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
        ctx.submap_extract_points(710 + s.submap_id, None)
    L0 = oracle.Layer.from_blocks(s0.voxel_size, s0.vps, s0.block_idx, s0.distance, s0.weight)
    L1 = oracle.Layer.from_blocks(s1.voxel_size, s1.vps, s1.block_idx, s1.distance, s1.weight)
    xo, do_, wo, _ = oracle.find_isosurface_vertices(L0, 1.0)
    assert len(xo) > 100
    ref, read = pair_scene.poses_init[0], pair_scene.poses_init[1]
    ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(L1, xo, do_, wo, ref, read)
    ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(710, 711, ref, read)
    assert ok_o and ok_g
    assert np.array_equal(r_g, r_o) and np.array_equal(jr_g, jr_o) and np.array_equal(je_g, je_o)
    # and through the fused graph path
    pg = api.PoseGraph(ctx)
    for i in range(2):
        pg.addSubmapNode(api.SubmapNodeConfig(710 + i, pair_scene.poses_init[i], set_constant=(i == 0)))
    pg.addRegistrationConstraint(api.RegistrationConstraintConfig(710, 711))
    ok, cost, g, H = pg.evaluate()
    assert ok and cost > 0


def test_overlapping_pairs_match_oracle(ctx, oracle, small_scene):
    """vgx_find_overlapping_pairs == updateOverlappingSubmapList over the oracle's overlapsWith
    (AABB from the extracted surface OBB, isosurface blocks from the extracted vertices)."""
    sc = small_scene
    ids = [800 + i for i in range(len(sc.submaps))]
    layers, obbs, isos = [], [], []
    for sid, s in zip(ids, sc.submaps):
        ctx.submap_upload(sid, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
        ctx.submap_extract_points(sid, None)
        L = oracle.Layer.from_blocks(s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
        layers.append(L)
        obbs.append(oracle.surface_obb(L, 1.0, 0.3))
        isos.append(oracle.find_isosurface_vertices(L, 1.0)[3])
    rs = np.random.RandomState(3)
    for trial in range(3):
        poses = sc.poses_init + (rs.normal(0, 0.5, sc.poses_init.shape) * np.array([1, 1, 0.05, 0.1]) if trial else 0)
        T = np.array([synth.pose_to_T(p) for p in poses], np.float32)
        got = ctx.find_overlapping_pairs(ids, T)
        want = []
        aabbs = [oracle.aabb_from_obb_and_pose(o[1], o[2], T[k]) for k, o in enumerate(obbs)]
        for i in range(len(ids)):
            for j in range(i + 1, len(ids)):
                bs = sc.submaps[i].voxel_size * sc.submaps[i].vps
                if oracle.submaps_overlap(aabbs[i], aabbs[j], T[i], T[j], isos[i], np.float32(bs), layers[j]):
                    want.append((ids[i], ids[j]))
        assert got == want
        assert len(want) >= 3
