"""GPU parity: ESDF generation on resident bricks (vgx_submap_generate_esdf) vs the oracle's fixed
point, and the use_esdf_distance registration branch (registration_cost_function.cpp:133-140)."""
import numpy as np
import pytest

from support import ctx  # noqa: F401
from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu
VS, VPS = 0.2, 16


def _esdf_check(ctx, oracle, sid, vs, vps, idx, d, w, **cfg):
    ctx.submap_upload(sid, vs, vps, idx, d, w)
    sweeps = ctx.submap_generate_esdf(sid, ctx.esdf_config(**cfg) if cfg else None)
    L = oracle.Layer.from_blocks(vs, vps, idx, d, w)
    eo, obo, _ = oracle.generate_esdf(L, oracle.esdf_config(**cfg) if cfg else None)
    eg, obg = ctx.submap_download_esdf(sid)
    assert np.array_equal(obg, obo)
    assert np.array_equal(eg, eo)        # the fixed point does not depend on the update order
    assert sweeps >= 2
    return L, eo, obo


def test_plane_and_sphere_bit_exact(ctx, oracle):
    idx, d, w = synth.plane_layer_blocks([0, 0, 1.0], 0.37, VS, VPS, ((0, 1), (0, 1), (-1, 1)), trunc=0.6)
    _esdf_check(ctx, oracle, 900, VS, VPS, idx, d, w)
    c = np.array([1.7, 1.5, 1.6]); R = 0.9
    idx, d, w = synth.field_layer_blocks(lambda p: np.linalg.norm(p - c, axis=-1) - R, VS, VPS,
                                         ((0, 1), (0, 1), (0, 1)), weight=1.0)
    _esdf_check(ctx, oracle, 901, VS, VPS, idx, np.clip(d, -0.6, 0.6).astype(np.float32), w)
    _esdf_check(ctx, oracle, 902, VS, VPS, idx, np.clip(d, -0.6, 0.6).astype(np.float32), w,
                max_distance_m=1.0, default_distance_m=1.0, min_distance_m=0.1)


def test_scene_submap_esdf_and_registration_branch(ctx, oracle, pair_scene):
    """finishSubmap's ESDF feeds Evaluate's default branch: emit-mode residuals against the reading
    submap's ESDF are bit-exact vs the oracle evaluating the oracle's ESDF layer."""
    from voxgraph_b200 import api
    s0, s1 = pair_scene.submaps
    L1, e1, ob1 = _esdf_check(ctx, oracle, 911, s1.voxel_size, s1.vps, s1.block_idx, s1.distance, s1.weight)
    ctx.submap_upload(910, s0.voxel_size, s0.vps, s0.block_idx, s0.distance, s0.weight)
    ctx.submap_upload_points(910, api.K_ISOSURFACE_POINTS, s0.points_xyz, s0.points_distance, s0.points_weight)
    # the oracle's ESDF as a layer: weight = observed ? 1 : 0 (SURVEY: observed <=> weight > 1e-6)
    Le = oracle.Layer.from_blocks(s1.voxel_size, s1.vps, s1.block_idx, e1, ob1)
    ref, read = pair_scene.poses_init[0], pair_scene.poses_init[1]
    ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(Le, s0.points_xyz, s0.points_distance, s0.points_weight, ref, read)
    ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(910, 911, ref, read, ctx.reg_config(use_esdf_distance=1))
    assert ok_o and ok_g and (np.abs(jr_o).sum(1) > 0).sum() > 300
    assert np.array_equal(r_g, r_o) and np.array_equal(jr_g, jr_o) and np.array_equal(je_g, je_o)
    # the TSDF branch differs (the ESDF extends beyond the truncation band)
    ok_t, r_t, _, _ = ctx.reg_eval_emit(910, 911, ref, read)
    assert ok_t and not np.array_equal(r_t, r_g)
    # without an ESDF the branch is refused
    with pytest.raises(api.VgxError):
        ctx.reg_eval_emit(911, 910, read, ref, ctx.reg_config(use_esdf_distance=1))
    # relevant voxels carry the ESDF distance when the filter asks for it (cpp:185-189)
    ctx.submap_extract_points(911, ctx.registration_filter(use_esdf_distance=1))
    xg, dg, wg = ctx.submap_download_points(911, api.K_VOXELS)
    xo, do_, wo = oracle.find_relevant_voxels(L1, 1.0, 0.3)
    assert np.array_equal(xg, xo) and np.array_equal(wg, wo)
    flat_e = e1.reshape(-1); flat_d = s1.distance.reshape(-1); flat_w = s1.weight.reshape(-1)
    sel = (flat_w.astype(np.float64) > 1.0) & (np.abs(flat_d.astype(np.float64)) < 0.3)
    assert np.array_equal(dg, flat_e[sel])
