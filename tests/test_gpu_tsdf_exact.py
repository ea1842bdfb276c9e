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


def _scans(world, n_beams=16, n_azimuth=256, origin=(0.0, 0.0, 0.0)):
    """Three scans from different poses (two with clearing rays), sensor poses offset by `origin`."""
    out = []
    for k, (px, py, yaw) in enumerate([(15.0, 15.0, 0.4), (16.5, 14.0, 1.9), (13.0, 16.0, -2.6)]):
        pts = synth.lidar_scan(world, np.array([px, py, 1.2, yaw]), n_beams=n_beams, n_azimuth=n_azimuth,
                               seed=k, miss_range=40.0 if k != 1 else None)
        T = synth.pose_to_T([px - 15.0 + origin[0], py - 15.0 + origin[1], 0.1 * k + origin[2], yaw])
        out.append((T, pts))
    return out


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


MW24 = 2.0 ** 24
CONFIGS = [
    dict(),
    dict(use_const_weight=0),
    dict(use_weight_dropoff=0),
    dict(use_sparsity_compensation_factor=0),
    dict(sparsity_compensation_factor=1.0),
    dict(sparsity_compensation_factor=2.5),
    dict(allow_clear=0),
    dict(voxel_carving_enabled=0),
    dict(use_const_weight=0, use_weight_dropoff=0),
    dict(use_const_weight=0, sparsity_compensation_factor=2.5, allow_clear=0),
    dict(voxel_carving_enabled=0, use_weight_dropoff=0, use_sparsity_compensation_factor=0),
    dict(min_ray_length_m=1.5, max_ray_length_m=9.0),
    dict(default_truncation_distance=0.1),
    dict(default_truncation_distance=0.2),    # = voxel size: the drop-off denominator is 0
    dict(default_truncation_distance=2.0),
    dict(max_weight=3.0),
    dict(max_weight=40.0),
    dict(max_weight=100.5),
    dict(max_weight=MW24 - 8),
    dict(max_weight=MW24),
]


@pytest.mark.parametrize("kw", CONFIGS, ids=lambda kw: ",".join("%s=%r" % i for i in kw.items()) or "default")
def test_simple_bit_exact_config_matrix(ctx, oracle, world, kw):
    exp = _run_mode0(ctx, oracle, 0.2, 16, _scans(world), **kw)
    sat = sum(e[4] for e in exp)
    if kw.get("use_const_weight", 1) and kw.get("max_weight", 1e4) <= 2.0 ** 20 and kw.get("voxel_carving_enabled", 1):
        assert sat > 0     # integer weights >= 2^-20 max_weight: the closed form runs
    if kw.get("max_weight", 0) >= MW24 - 8:
        assert sat == 0


def _ring(n, z, ranges, az0=0.1):
    """n points around the sensor at height z (sensor frame) and the given horizontal ranges."""
    a = az0 + 2 * np.pi * np.arange(n) / n
    r = np.resize(np.asarray(ranges, np.float64), n)
    zz = np.resize(np.asarray(z, np.float64), n)
    return np.stack([r * np.cos(a), r * np.sin(a), zz], -1).astype(np.float32)


@pytest.mark.parametrize("mw", [3.0, 40.0, 100.5, 1e4, MW24 - 8, MW24])
def test_saturated_batches_cross_the_cap(ctx, oracle, mw):
    """Integer update weights of 2^14 (|z| = 2^-7, use_const_weight=0) reach 2^24 within 1024 rays:
    the cap is crossed inside a closed-form batch at small, fractional and near-2^24 caps.  At 2^24
    the integer closed form is refused and only the batches after a voxel sits at the cap collapse."""
    pts = _ring(1100, [2.0 ** -7, -2.0 ** -7], [3.0, 4.5, 6.0])
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.3])
    exp = _run_mode0(ctx, oracle, 0.2, 16, [(T, pts)], use_const_weight=0, max_weight=mw)
    assert exp[0][4] > 0


@pytest.mark.parametrize("vs,vps", [(0.05, 8), (0.1, 16), (0.15, 8), (0.05, 32), (0.2, 16)])
def test_simple_bit_exact_resolutions(ctx, oracle, world, vs, vps):
    """Other voxel sizes and block sizes (key = slot << 3 log2(vps), sort end bit, sentinel), a sensor
    at negative coordinates, one 2 km from the origin, and a float quaternion that is not exactly unit."""
    scans = _scans(world, n_beams=8, n_azimuth=128)
    T_neg = scans[0][0].copy(); T_neg[4:] = [-7.3, -11.9, -2.05]
    T_far = scans[1][0].copy(); T_far[4:] += np.array([2000.0, -1312.5, 3.0], np.float32)
    q = np.array([0.71, 0.12, -0.2, 0.67], np.float32)        # |q|^2 = 0.9894
    T_q = np.concatenate([q, np.float32([0.4, -0.3, 0.2])]).astype(np.float32)
    cfg = dict(max_ray_length_m=6.0)
    _run_mode0(ctx, oracle, vs, vps, [(T_neg, scans[0][1]), (T_q, scans[2][1])], **cfg)
    _run_mode0(ctx, oracle, vs, vps, [(T_far, scans[1][1]), (T_far, scans[0][1])], **cfg)


def _edge_points():
    f = np.float32
    up = lambda v: np.nextafter(f(v), f(np.inf)); dn = lambda v: np.nextafter(f(v), f(-np.inf))
    p = []
    for r in (0.5, 8.0):                       # min / max ray length exactly, and one ulp either side
        for v in (dn(r), f(r), up(r)):
            p += [[v, 0, 0], [0, -v, 0], [0, 0, v]]     # axis-aligned: t = 2 on the degenerate axes
    p += [[0, 0, 0]]                           # sdf = 0/0 at the sensor voxel when min_ray_length_m = 0
    p += [[np.nan, 0, 0], [1, np.nan, 2], [np.inf, 0, 0], [-np.inf, 0, 0], [0, np.inf, 1]]
    p += [[3e19, 0, 0], [-2e19, 2e19, 0], [1.1e19, 1.1e19, 1.1e19], [1e19, -1e19, 1e19]]
    p += [[2.0, 0.5, 0.25], [4.0, -2.0, 1.0], [-2.0, 2.0, -0.75], [6.0, 4.0, 0.0], [0.0, -4.0, 2.0]]
    p += [[3.1 + 0.02 * k, 1.3 + 0.01 * k, -0.6 + 0.015 * k] for k in range(5)]   # one voxel
    p += [[12.0, 3.0, -1.0], [-9.0, 10.0, 0.5], [0.3, -15.0, 2.0]]             # clearing rays
    return np.array(p, np.float32)


EDGE_CFGS = [dict(min_ray_length_m=0.5, max_ray_length_m=8.0),
             dict(min_ray_length_m=0.0, max_ray_length_m=8.0, voxel_carving_enabled=0),
             dict(min_ray_length_m=0.0, max_ray_length_m=8.0, allow_clear=0),
             dict(min_ray_length_m=0.0, max_ray_length_m=8.0, use_weight_dropoff=0)]


def test_ray_edges_simple_bit_exact(ctx, oracle):
    """Crafted points at 0.25 m voxels (faces exactly representable) from a sensor on a block corner
    and from one inside a voxel, under four configurations, accumulated in one submap."""
    pts = _edge_points()
    scans = []
    for t in ([0.0, 0.0, 0.0], [0.3, -0.45, 0.1]):
        T = np.array([1, 0, 0, 0, *t], np.float32)
        scans += [(T, pts, c) for c in EDGE_CFGS]
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
    pts = _edge_points()
    keep = np.ones(len(pts), bool); keep[[0, 1, 2, 6, 7, 8, 9, 10, 11, 15, 16, 17]] = False
    for c in EDGE_CFGS:
        _run_fast(ctx, oracle, 0.25, 8, np.array([1, 0, 0, 0, 0.3, -0.45, 0.1], np.float32), pts[keep],
                  **{**c, "use_weight_dropoff": 0})


@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 128, 129])
def test_segment_lengths(ctx, oracle, n):
    """N rays with carving from one sensor: the sensor voxel's segment has exactly N tuples (short
    path up to 64, warp path with 32-tuple batches and a tail beyond).  Saturated stream: integer
    weights 2^6 far behind the sensor; mixed stream: some sdf below 2 trunc at the sensor voxel and
    fractional weights."""
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.0])
    sat_pts = _ring(n, 0.125, [3.0, 4.2, 5.5])
    mixed = _ring(n, [0.125, 0.3, 0.125, -0.2, 0.125, 0.125, 0.125], [3.0, 1.0, 4.2, 5.5, 1.1])
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
