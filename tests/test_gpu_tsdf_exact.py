"""TSDF integration pinned to the oracle (tests/tsdf_exact.py) across its configuration, resolutions,
ray edges and segment lengths, and the Fast schedule checked for lost or duplicated updates.

Mode 0 (ray ordered): identical stats, block set, and every voxel's distance and weight bit for bit,
and the number of closed-form batches of tsdf_apply_long_kernel equal to the exact model's count.
Mode 1 with every ray cast (start keys all distinct, unlimited ray collisions): the set of updates is
fixed; tsdf_exact.check_fast checks the order-independent parts exactly and the rest against the
running-mean rounding bound."""
import itertools

import numpy as np
import pytest

import tsdf_exact as tx
from support import ctx  # noqa: F401
from voxgraph_b200 import _lib, synth

pytestmark = pytest.mark.gpu

_ids = itertools.count(2000)
FAST_ALL = dict(mode=1, start_voxel_subsampling_factor=1e3, max_consecutive_ray_collisions=1 << 30)


@pytest.fixture(scope="module")
def world():
    return synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)


def _run_mode0(ctx, oracle, vs, vps, scans, capacity=None, **kw):
    """Integrate `scans` = [(T, points[, cfg overrides])] on both sides; returns per-scan stats and the
    model's closed-form batch counts.  Capacity defaults to the oracle's final block count."""
    layer = oracle.Layer(vs, vps)
    state = tx.State()
    exp = []
    for sc in scans:
        T, pts = sc[0], sc[1]
        ocfg = oracle.tsdf_config(**{**kw, **(sc[2] if len(sc) > 2 else {})})
        st, g, s, u = oracle.tsdf_integrate_trace(layer, ocfg, T, pts)
        sat = tx.replay(tx.voxel_keys(g), s, u, ocfg.default_truncation_distance, ocfg.max_weight, state)[3]
        exp.append((st.rays_valid, st.rays_cast, st.voxel_updates, st.blocks_allocated, sat))
    sid = next(_ids)
    ctx.submap_create(sid, vs, vps, layer.num_blocks if capacity is None else capacity)
    try:
        got = []
        for sc in scans:
            gcfg = ctx.tsdf_config(**{**kw, **(sc[2] if len(sc) > 2 else {})})
            sg = ctx.tsdf_integrate(sid, sc[0], sc[1], gcfg)
            got.append((sg.rays_valid, sg.rays_cast, sg.voxel_updates, sg.blocks_allocated, sg.saturated_batches))
        assert got == exp
        tx.assert_layers_bit_equal(layer.export(), ctx.submap_download(sid))
    finally:
        ctx.submap_free(sid)
    return exp


@pytest.mark.parametrize("kw", tx.CONFIGS, ids=tx.config_id)
def test_simple_bit_exact_config_matrix(ctx, oracle, world, kw):
    exp = _run_mode0(ctx, oracle, 0.2, 16, tx.scans(world), **kw)
    sat = sum(e[4] for e in exp)
    if kw.get("use_const_weight", 1) and kw.get("max_weight", 1e4) <= 2.0 ** 20 and kw.get("voxel_carving_enabled", 1):
        assert sat > 0     # integer weights >= 2^-20 max_weight: the closed form runs
    if kw.get("max_weight", 0) >= tx.MW24 - 8:
        assert sat == 0


@pytest.mark.parametrize("mw", [3.0, 40.0, 100.5, 1e4, tx.MW24 - 8, tx.MW24])
def test_saturated_batches_cross_the_cap(ctx, oracle, mw):
    """Integer update weights of 2^14 (|z| = 2^-7, use_const_weight=0) reach 2^24 within 1024 rays:
    the cap is crossed inside a closed-form batch at small, fractional and near-2^24 caps.  At 2^24
    the integer closed form is refused and only the batches after a voxel sits at the cap collapse."""
    pts = tx.ring(1100, [2.0 ** -7, -2.0 ** -7], [3.0, 4.5, 6.0])
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.3])
    exp = _run_mode0(ctx, oracle, 0.2, 16, [(T, pts)], use_const_weight=0, max_weight=mw)
    assert exp[0][4] > 0


@pytest.mark.parametrize("vs,vps", [(0.05, 8), (0.1, 16), (0.15, 8), (0.05, 32), (0.2, 16)])
def test_simple_bit_exact_resolutions(ctx, oracle, world, vs, vps):
    """Other voxel sizes and block sizes (key = slot << 3 log2(vps), sort end bit, sentinel), a sensor
    at negative coordinates, one 2 km from the origin, and a float quaternion that is not exactly unit."""
    scans = tx.scans(world, n_beams=8, n_azimuth=128)
    T_neg = scans[0][0].copy(); T_neg[4:] = [-7.3, -11.9, -2.05]
    T_far = scans[1][0].copy(); T_far[4:] += np.array([2000.0, -1312.5, 3.0], np.float32)
    q = np.array([0.71, 0.12, -0.2, 0.67], np.float32)        # |q|^2 = 0.9894
    T_q = np.concatenate([q, np.float32([0.4, -0.3, 0.2])]).astype(np.float32)
    cfg = dict(max_ray_length_m=6.0)
    _run_mode0(ctx, oracle, vs, vps, [(T_neg, scans[0][1]), (T_q, scans[2][1])], **cfg)
    _run_mode0(ctx, oracle, vs, vps, [(T_far, scans[1][1]), (T_far, scans[0][1])], **cfg)


def test_ray_edges_simple_bit_exact(ctx, oracle):
    """Crafted points at 0.25 m voxels (faces exactly representable) from a sensor on a block corner
    and from one inside a voxel, under four configurations, accumulated in one submap."""
    pts = tx.edge_points()
    scans = []
    for t in ([0.0, 0.0, 0.0], [0.3, -0.45, 0.1]):
        T = np.array([1, 0, 0, 0, *t], np.float32)
        scans += [(T, pts, c) for c in tx.EDGE_CFGS]
    exp = _run_mode0(ctx, oracle, 0.25, 8, scans)
    assert all(e[0] == e[1] for e in exp)
    # 15 axis points within or beyond the lengths, 4 huge finite, 5 on faces, 5 in one voxel, 3 clearing
    assert exp[0][0] == 32


def _run_fast(ctx, oracle, vs, vps, T, pts, **kw):
    ocfg = oracle.tsdf_config(**{**FAST_ALL, **kw})
    layer = oracle.Layer(vs, vps)
    st, g, s, u = oracle.tsdf_integrate_trace(layer, ocfg, T, pts)
    assert st.rays_cast == st.rays_valid            # every ray is cast: the update set is fixed
    sid = next(_ids)
    ctx.submap_create(sid, vs, vps, layer.num_blocks)
    try:
        sg = ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(**{**FAST_ALL, **kw}))
        assert (sg.rays_valid, sg.rays_cast, sg.voxel_updates, sg.blocks_allocated) == \
            (st.rays_valid, st.rays_cast, st.voxel_updates, st.blocks_allocated)
        gi, gd, gw = ctx.submap_download(sid)
    finally:
        ctx.submap_free(sid)
    oi, od, ow = layer.export()
    assert np.array_equal(np.unique(gi, axis=0), np.unique(oi, axis=0))
    return tx.check_fast(tx.layer_voxels(gi, gd, gw, vps), tx.voxel_keys(g), s, u,
                         ocfg.default_truncation_distance, ocfg.max_weight, tx.layer_voxels(oi, od, ow, vps))


def test_fast_serialisation_dense_scan(ctx, oracle, world):
    """32 x 512 scan, constant weight, no drop-off (uw = 1 or 20): tens of thousands of CAS updates
    on the sensor voxels and racing on-demand allocation of fresh blocks."""
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=32, n_azimuth=512, seed=1,
                           miss_range=40.0)
    info = _run_fast(ctx, oracle, 0.2, 16, synth.pose_to_T([0.3, -0.2, 0.1, 0.4]), pts, use_weight_dropoff=0)
    assert info["max_updates"] > 10000 and info["inner"] > 1000 and info["single"] > 1000


def test_fast_serialisation_ray_edges(ctx, oracle):
    """The crafted points in the Fast schedule.  The one-ulp neighbours of the length limits are left
    out: after the sensor translation they can land on the same float point, and the Fast schedule
    then rightly casts only one of them."""
    pts = tx.edge_points()
    keep = np.ones(len(pts), bool); keep[[0, 1, 2, 6, 7, 8, 9, 10, 11, 15, 16, 17]] = False
    for c in tx.EDGE_CFGS:
        _run_fast(ctx, oracle, 0.25, 8, np.array([1, 0, 0, 0, 0.3, -0.45, 0.1], np.float32), pts[keep],
                  **{**c, "use_weight_dropoff": 0})


@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 128, 129])
def test_segment_lengths(ctx, oracle, n):
    """N rays with carving from one sensor: the sensor voxel's segment has exactly N tuples (short
    path up to 64, warp path with 32-tuple batches and a tail beyond).  Saturated stream: integer
    weights 2^6 far behind the sensor; mixed stream: some sdf below 2 trunc at the sensor voxel and
    fractional weights."""
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.0])
    sat_pts = tx.ring(n, 0.125, [3.0, 4.2, 5.5])
    mixed = tx.ring(n, [0.125, 0.3, 0.125, -0.2, 0.125, 0.125, 0.125], [3.0, 1.0, 4.2, 5.5, 1.1])
    for pts in (sat_pts, mixed):
        layer = oracle.Layer(0.2, 16)
        st, g, s, u = oracle.tsdf_integrate_trace(layer, oracle.tsdf_config(use_const_weight=0), T, pts)
        keys = tx.voxel_keys(g)
        assert np.count_nonzero(keys == tx.voxel_keys([[0, 0, 0]])[0]) == n
        exp = _run_mode0(ctx, oracle, 0.2, 16, [(T, pts), (T, pts)], use_const_weight=0)
        if pts is sat_pts and n >= 65:
            assert exp[1][4] > 0
        if n <= 64:
            assert exp[0][4] == exp[1][4] == 0


@pytest.mark.parametrize("mode", [0, 1])
def test_capacity_at_the_edge(ctx, oracle, world, mode):
    """Capacity equal to the oracle's block count succeeds; one block less fails with
    VGX_ERR_CAPACITY and leaves exactly `capacity` blocks, all of them in the oracle's set."""
    from voxgraph_b200 import api
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=8, n_azimuth=128, seed=3)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    kw = FAST_ALL if mode == 1 else {}
    layer = oracle.Layer(0.2, 16)
    oracle.tsdf_integrate(layer, oracle.tsdf_config(**kw), T, pts)
    nb = layer.num_blocks
    oset = set(map(tuple, layer.export()[0].tolist()))
    for cap in (nb, nb - 1):
        sid = next(_ids)
        ctx.submap_create(sid, 0.2, 16, cap)
        try:
            if cap == nb:
                ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(**kw))
            else:
                with pytest.raises(api.VgxError) as e:
                    ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(**kw))
                assert e.value.code == _lib.VGX_ERR_CAPACITY
            assert ctx.submap_block_count(sid) == cap
            gi = ctx.submap_download(sid)[0]
            assert len(gi) == cap and set(map(tuple, gi.tolist())) <= oset
        finally:
            ctx.submap_free(sid)
