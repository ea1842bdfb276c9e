"""TSDF integration on the device: the Fast schedule against the oracle's restatement of it, capacity overflow,
and an integrated submap as the reading submap of a registration constraint.  Ray-ordered (mode 0) parity with
the oracle is pinned in test_gpu_tsdf_exact.py."""
import numpy as np
import pytest

from support import ctx, world  # noqa: F401
from voxgraph_b200 import _lib, synth

pytestmark = pytest.mark.gpu

VS = 0.2
IDENT = np.array([1, 0, 0, 0, 0, 0, 0], np.float32)


def _as_dict(idx, d, w):
    return {tuple(b): (d[k], w[k]) for k, b in enumerate(idx)}


def test_fast_mode_properties(ctx, oracle, world):
    """FastTsdfIntegrator scheduling is race dependent in the reference; check its invariants."""
    pose = np.array([15.0, 15.0, 1.2, 0.4])
    pts = synth.lidar_scan(world, pose, n_beams=32, n_azimuth=512, seed=1)
    T = synth.pose_to_T([0, 0, 0, 0])
    ctx.submap_create(303, VS, 16, 4096); ctx.submap_create(304, VS, 16, 4096)
    s_simple = ctx.tsdf_integrate(303, T, pts, ctx.tsdf_config(mode=0))
    s_fast = ctx.tsdf_integrate(304, T, pts, ctx.tsdf_config(mode=1))
    assert s_fast.rays_valid == s_simple.rays_valid
    assert s_fast.rays_cast < s_simple.rays_cast and s_fast.voxel_updates < s_simple.voxel_updates
    lay_fast = oracle.Layer(VS, 16)
    so = oracle.tsdf_integrate(lay_fast, oracle.tsdf_config(mode=1), T, pts)
    # same order of magnitude of work as the single-threaded restatement of the Fast rule
    assert 0.5 * so.voxel_updates < s_fast.voxel_updates < 2.0 * so.voxel_updates
    gs = _as_dict(*ctx.submap_download(303)); gf = _as_dict(*ctx.submap_download(304))
    agree = tot = 0
    for b in gf:
        assert b in gs
        m = (gf[b][1] > 0) & (np.abs(gf[b][0]) < 0.3) & (gs[b][1] > 0)
        agree += (np.sign(gf[b][0][m]) == np.sign(gs[b][0][m])).sum(); tot += m.sum()
    assert tot > 100 and agree / tot > 0.9
    # blocks are allocated on demand, only where a voxel is actually visited (as
    # allocateStorageAndGetVoxelPtr does; a visit whose update weight drops to zero still allocates):
    # a subset of the Simple set, and about as many as the single-threaded restatement of the Fast
    # rule allocates
    assert sum((gf[b][1] > 0).any() for b in gf) >= 0.9 * len(gf)
    assert len(gf) <= len(gs)
    go = _as_dict(*lay_fast.export())
    assert abs(len(gf) - len(go)) <= 0.1 * len(go)
    assert len(set(gf) & set(go)) >= 0.85 * len(go)


def test_fast_mode_sparse_rays_match_oracle_exactly(ctx, oracle):
    """Rays that share no voxel and no de-duplication bucket make the Fast schedule deterministic:
    block set, visited voxels, distances and weights equal the oracle's Fast restatement."""
    rs = np.random.RandomState(5)
    dirs = []
    for az in np.linspace(-3.0, 3.0, 24):
        for el in (-0.5, 0.0, 0.45):
            dirs.append([np.cos(az) * np.cos(el), np.sin(az) * np.cos(el), np.sin(el)])
    pts = (np.array(dirs) * rs.uniform(4.0, 9.0, (len(dirs), 1))).astype(np.float32)
    T = synth.pose_to_T([0.13, -0.27, 0.31, 0.2])
    lay = oracle.Layer(VS, 16)
    so = oracle.tsdf_integrate(lay, oracle.tsdf_config(mode=1), T, pts)
    ctx.submap_create(308, VS, 16, 4096)
    sg = ctx.tsdf_integrate(308, T, pts, ctx.tsdf_config(mode=1))
    go = _as_dict(*lay.export()); gg = _as_dict(*ctx.submap_download(308))
    # rays leave the sensor through shared voxels, where the race-free schedules may differ: compare
    # beyond 1.5 m from the sensor origin only (no voxel is shared there)
    assert (sg.rays_valid, sg.rays_cast) == (so.rays_valid, so.rays_cast)
    assert set(gg) == set(go)
    origin = np.array([0.13, -0.27, 0.31])
    checked = 0
    for b in go:
        lin = np.arange(16 ** 3)
        c = (np.stack([lin % 16, (lin // 16) % 16, lin // 256], -1) + 0.5) * VS + np.array(b) * 16 * VS
        far = np.linalg.norm(c - origin, axis=1) > 1.5
        assert np.array_equal(go[b][1][far] > 0, gg[b][1][far] > 0)
        assert np.array_equal(go[b][0][far], gg[b][0][far]) and np.array_equal(go[b][1][far], gg[b][1][far])
        checked += int((go[b][1][far] > 0).sum())
    assert checked > 500


def test_capacity_overflow_reports_error(ctx):
    from voxgraph_b200 import api
    ctx.submap_create(305, VS, 16, 2)
    pts = np.array([[10.0, 3.0, 1.0], [-8.0, 2.0, 0.5]], np.float32)
    with pytest.raises(api.VgxError) as e:
        ctx.tsdf_integrate(305, IDENT, pts, ctx.tsdf_config())
    assert e.value.code == _lib.VGX_ERR_CAPACITY
    # the overflow leaves a consistent submap behind (hash rebuilt from the blocks that exist):
    # further calls keep failing cleanly instead of hanging on a full table, in both modes
    assert ctx.submap_block_count(305) == 2
    for mode in (1, 0, 1):
        with pytest.raises(api.VgxError) as e:
            ctx.tsdf_integrate(305, IDENT, pts, ctx.tsdf_config(mode=mode))
        assert e.value.code == _lib.VGX_ERR_CAPACITY
    far = np.array([[60.0, 3.0, 1.0], [-70.0, 2.0, 0.5], [5.0, 80.0, 9.0]], np.float32)
    with pytest.raises(api.VgxError):
        ctx.tsdf_integrate(305, IDENT, far, ctx.tsdf_config(mode=1, max_ray_length_m=100.0))
    idx, d, w = ctx.submap_download(305)
    assert idx.shape[0] == 2


def test_integrate_then_register(ctx, oracle):
    """HP1 -> HP2 hand-over: a submap filled by the integrator is finished and used as the
    reading submap of a registration constraint; emit-mode parity vs the oracle on the
    downloaded layer."""
    world = synth.make_world(5, size_xy=(24.0, 24.0), n_clutter=30, n_walls=3)
    pose = np.array([12.0, 12.0, 1.2, 0.0])
    pts = synth.lidar_scan(world, pose, n_beams=32, n_azimuth=512, seed=2)
    T = synth.pose_to_T([0, 0, 0, 0])
    ctx.submap_create(306, VS, 16, 4096)
    for _ in range(2):
        ctx.tsdf_integrate(306, T, pts, ctx.tsdf_config())
    ctx.submap_finish(306)
    idx, d, w = ctx.submap_download(306)
    layer = oracle.Layer.from_blocks(VS, 16, idx, d, w)
    # reference points: the scan end points themselves (on the surface), in the same frame
    sel = pts[:: 7][:2000]
    ctx.submap_upload(307, VS, 16, idx[:1], d[:1], w[:1])
    ctx.submap_upload_points(307, 1, sel, np.zeros(len(sel), np.float32), np.ones(len(sel), np.float32))
    ref = np.array([0.05, -0.03, 0.02, 0.01]); read = np.zeros(4)
    ok_o, r_o, jr_o, je_o = oracle.reg_evaluate(layer, sel, np.zeros(len(sel), np.float32),
                                                np.ones(len(sel), np.float32), ref, read)
    ok_g, r_g, jr_g, je_g = ctx.reg_eval_emit(307, 306, ref, read)
    assert ok_o and ok_g
    assert (np.abs(jr_o).sum(1) > 0).sum() > 500
    assert np.array_equal(r_g, r_o) and np.array_equal(jr_g, jr_o) and np.array_equal(je_g, je_o)
