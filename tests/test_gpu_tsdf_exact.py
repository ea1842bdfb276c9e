"""TSDF integration pinned to the oracle (tests/tsdf_exact.py, tests/colour_exact.py) across its configuration,
resolutions, ray edges and segment lengths, and the Fast schedule checked for lost or duplicated updates.

Mode 0 (ray ordered): every case runs into a coloured submap, every ray with a colour of its own whose four
channels differ, and into a colourless twin.  Both have the exact model's stats and number of closed-form batches
of tsdf_apply_long_kernel, the same launch counts, and the oracle's block set and every voxel's distance and weight
bit for bit; every colour word equals the sequential coloured replay, and only the coloured submap has a channel.
Mode 1 with every ray cast (start keys all distinct, unlimited ray collisions): the set of updates is
fixed; tsdf_exact.check_fast checks the order-independent parts exactly and the rest against the
running-mean rounding bound."""
import itertools

import numpy as np
import pytest

import colour_exact as cx
import tsdf_exact as tx
from support import ctx, world  # noqa: F401
from voxgraph_b200 import _lib, api, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
_ids = itertools.count(2000)


def _mode0(ctx, oracle, vs, vps, scans, seed=0, then=None, **kw):
    """Integrate scans [(T, points[, cfg overrides])] ray ordered, every point with a colour of its own, into a
    coloured submap and a colourless twin, and check both against the models; then(coloured id, its colour words)
    runs before the submaps are freed.  -> (per-scan model stats with saturated batches, [(voxel key, ray index,
    sdf, uw) per tuple] per scan, number of non-zero expected colour words)."""
    rs = np.random.RandomState(seed)
    layer = oracle.Layer(vs, vps)
    st_c, st_t = cx.State(), tx.State()
    exp, calls, traces = [], [], []
    for sc in scans:
        T, pts = sc[0], np.asarray(sc[1], F32)
        kwc = {**kw, **(sc[2] if len(sc) > 2 else {})}
        ocfg = oracle.tsdf_config(**kwc)
        trunc, M = ocfg.default_truncation_distance, ocfg.max_weight
        rgba = cx.colours(rs, len(pts))
        stats, g, s, u, r = cx.trace_rays(oracle, layer, ocfg, T, pts)
        keys = tx.voxel_keys(g)
        sat = tx.replay(keys, s, u, trunc, M, st_t)[3]
        cx.replay(keys, s, u, cx.pack(rgba)[r], trunc, M, st_c)
        exp.append(stats + (sat,))
        calls.append((T, pts, rgba, kwc))
        traces.append((keys, r, s, u))
    plain, col = next(_ids), next(_ids)
    try:
        for sid in (plain, col):
            ctx.submap_create(sid, vs, vps, layer.num_blocks)
        got = {plain: [], col: []}
        for (T, pts, rgba, kwc) in calls:
            cfg = ctx.tsdf_config(**kwc)
            for sid in (plain, col):
                before = ctx.launch_count
                sg = ctx.tsdf_integrate(sid, T, pts, cfg, rgba=rgba if sid == col else None)
                got[sid].append((sg.rays_valid, sg.rays_cast, sg.voxel_updates, sg.blocks_allocated,
                                 sg.saturated_batches, ctx.launch_count - before))
        assert [g[:5] for g in got[col]] == exp, (got[col], exp)
        assert got[col] == got[plain]
        assert ctx.submap_has_colour(col) and not ctx.submap_has_colour(plain)
        assert not ctx.submap_download_colour(plain).any()
        lay = ctx.submap_download(col)
        tx.assert_layers_bit_equal(layer.export(), lay)
        tx.assert_layers_bit_equal(ctx.submap_download(plain), lay)
        words = ctx.submap_download_colour(col)
        gk, gc = cx.layer_colours(lay[0], words, vps)
        want = cx.expected_words(lay[0], vps, st_c)
        bad = np.nonzero(gc != want)[0]
        assert bad.size == 0, (len(bad), gk[bad[0]], hex(int(gc[bad[0]])), hex(int(want[bad[0]])))
        if then is not None:
            then(col, words)
    finally:
        for sid in (plain, col):
            ctx.submap_free(sid)
    return exp, traces, int(np.count_nonzero(want))


def test_single_rays_bit_exact(ctx, oracle):
    """Forty rays without carving from a rotated sensor, 4-15 m long in random directions: only +-trunc around
    each end point is touched."""
    rs = np.random.RandomState(0)
    dirs = rs.normal(size=(40, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    pts = (dirs * rs.uniform(4.0, 15.0, (40, 1))).astype(F32)
    T = np.array([np.cos(0.35), 0, 0, np.sin(0.35), 0.13, -0.27, 0.41], F32)
    _mode0(ctx, oracle, 0.2, 16, [(T, pts)], voxel_carving_enabled=0)


def test_single_carving_ray_bit_exact(ctx, oracle):
    """One carving ray three times: repeated scans accumulate weight as the oracle does."""
    T = np.array([1, 0, 0, 0, 0.1, 0.1, 0.1], F32)
    _mode0(ctx, oracle, 0.2, 16, [(T, np.array([[7.3, 2.1, -1.4]], F32))] * 3)


def test_lidar_scan_vs_oracle(ctx, oracle, world):
    """Dense scan (config-3 shaped, scaled down).  `deterministic` = 0 changes nothing: the device ignores it
    (kept in the struct for layout compatibility) and the oracle's config has no such field."""
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=32, n_azimuth=512, seed=1,
                           miss_range=40.0)
    assert pts.shape[0] == 32 * 512
    exp = _mode0(ctx, oracle, 0.2, 16, [(synth.pose_to_T([0.3, -0.2, 0.1, 0.4]), pts)], deterministic=0)[0]
    # the voxels around the sensor collect one update per ray: their replay collapses in closed form
    assert exp[0][4] > 100


def test_finished_submap_refuses_integration(ctx):
    """Finishing a submap builds its registration view; integrating into it afterwards is refused."""
    T = np.array([1, 0, 0, 0, 0.1, 0.1, 0.1], F32)
    pts = np.array([[7.3, 2.1, -1.4]], F32)
    sid = next(_ids)
    ctx.submap_create(sid, 0.2, 16, 64)
    try:
        ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config())
        ctx.submap_finish(sid)
        with pytest.raises(api.VgxError) as e:
            ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config())
        assert e.value.code == _lib.VGX_ERR_INVALID
    finally:
        ctx.submap_free(sid)


def test_dense_scans_bit_exact(ctx, oracle, world):
    """Three 32 x 512 scans from different poses, two with clearing rays: thousands of rays through the same
    voxels, accumulated in one submap."""
    exp = _mode0(ctx, oracle, 0.2, 16, tx.scans(world, 32, 512))[0]
    assert sum(e[2] for e in exp) > 500000
    assert sum(e[4] for e in exp) > 300      # the closed-form replay of saturated batches was exercised


@pytest.mark.parametrize("vs,vps,max_ray", [(0.2, 16, 16.0), (0.05, 8, 5.0)])
def test_scans_and_ring_bit_exact(ctx, oracle, world, vs, vps, max_ray):
    """Three overlapping scans, then a 200-ray ring twice from one pose: its sensor voxel takes the long-segment
    path, and the closed-form batches the second time.  A later colourless scan leaves the colour channel
    untouched, and finishing keeps it."""
    scans = tx.scans(world, 16, 256) if vps == 16 else tx.scans(world, 8, 128)
    ring = (synth.pose_to_T([0.1, 0.1, 0.1, 0.0]), tx.ring(200, 0.125, [3.0, 4.2, 5.5]))
    scans += [ring, ring]
    cfg = dict(max_ray_length_m=max_ray)

    def then(sid, words):
        ctx.tsdf_integrate(sid, scans[0][0], scans[0][1], ctx.tsdf_config(**cfg))
        assert np.array_equal(ctx.submap_download_colour(sid), words)
        ctx.submap_finish_ex(sid)
        assert ctx.submap_has_colour(sid) and np.array_equal(ctx.submap_download_colour(sid), words)

    exp, _, n_col = _mode0(ctx, oracle, vs, vps, scans, then=then, **cfg)
    assert exp[-1][4] > 0 and n_col > 1000        # the closed-form batches are still taken with colours


@pytest.mark.parametrize("kw", tx.CONFIGS, ids=tx.config_id)
def test_simple_bit_exact_config_matrix(ctx, oracle, world, kw):
    exp, _, n_col = _mode0(ctx, oracle, 0.2, 16, tx.scans(world), **kw)
    assert n_col > 1000
    sat = sum(e[4] for e in exp)
    if kw.get("use_const_weight", 1) and kw.get("max_weight", 1e4) <= 2.0 ** 20 and kw.get("voxel_carving_enabled", 1):
        assert sat > 0     # integer weights >= 2^-20 max_weight: the closed form runs
    if kw.get("max_weight", 0) >= tx.MW24 - 8:
        assert sat == 0


def _band_at_cap(keys, s, u, trunc, M):
    """Band updates of the most-updated voxel that find it at the weight cap (sequential replay)."""
    k, c = np.unique(keys, return_counts=True)
    sel = keys == k[np.argmax(c)]
    d, w, n = F32(0), F32(0), 0
    for ss, uu in zip(s[sel], u[sel]):
        n += bool(w == F32(M) and abs(ss) < F32(trunc))
        d, w = tx.apply_update(ss, uu, d, w, F32(trunc), F32(M))
    return n


@pytest.mark.parametrize("mw", [3.0, 40.0, 100.5, 1e4, tx.MW24 - 8, tx.MW24])
@pytest.mark.parametrize("stream", ["far", "near"])
def test_saturated_batches_cross_the_cap(ctx, oracle, stream, mw):
    """Integer update weights of 2^14 (|z| = 2^-7, use_const_weight=0) reach 2^24 within 1024 rays:
    the cap is crossed inside a closed-form batch at small, fractional and near-2^24 caps.  At 2^24
    the integer closed form is refused and only the batches after a voxel sits at the cap collapse.
    'near' mixes in points 0.3-0.45 m from the sensor, which give the sensor voxel band updates (sdf ~ range <
    trunc), some between the far rays and the rest after them, so the colour step runs at the capped weight in
    full and partial batches."""
    pts = tx.ring(1100, [2.0 ** -7, -2.0 ** -7], [3.0, 4.5, 6.0])
    if stream == "near":
        near = tx.ring(80, [2.0 ** -7, -2.0 ** -7], [0.3, 0.45], az0=0.2)
        pts = np.concatenate([pts[:600], near[:13], pts[600:], near[13:]])
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.3])
    exp, traces, _ = _mode0(ctx, oracle, 0.2, 16, [(T, pts)], use_const_weight=0, max_weight=mw)
    assert exp[0][4] > 0
    if stream == "near":
        keys, _, s, u = traces[0]
        assert _band_at_cap(keys, s, u, 0.6, mw) >= 60


@pytest.mark.parametrize("vs,vps", [(0.05, 8), (0.1, 16), (0.15, 8), (0.05, 32), (0.2, 16)])
def test_simple_bit_exact_resolutions(ctx, oracle, world, vs, vps):
    """Other voxel sizes and block sizes (key = slot << 3 log2(vps), sort end bit, sentinel), a sensor
    at negative coordinates, one 2 km from the origin, and a float quaternion that is not exactly unit."""
    scans = tx.scans(world, n_beams=8, n_azimuth=128)
    T_neg = scans[0][0].copy(); T_neg[4:] = [-7.3, -11.9, -2.05]
    T_far = scans[1][0].copy(); T_far[4:] += np.array([2000.0, -1312.5, 3.0], F32)
    q = np.array([0.71, 0.12, -0.2, 0.67], F32)        # |q|^2 = 0.9894
    T_q = np.concatenate([q, F32([0.4, -0.3, 0.2])]).astype(F32)
    cfg = dict(max_ray_length_m=6.0)
    assert _mode0(ctx, oracle, vs, vps, [(T_neg, scans[0][1]), (T_q, scans[2][1])], **cfg)[2] > 100
    assert _mode0(ctx, oracle, vs, vps, [(T_far, scans[1][1]), (T_far, scans[0][1])], seed=1, **cfg)[2] > 100


def _ray_edges(ctx, oracle, second):
    """The crafted points from the first sensor and `second` (the same points in some order) from the second,
    under the four edge configurations, accumulated in one submap."""
    scans = []
    for t, p in (([0.0, 0.0, 0.0], tx.edge_points()), ([0.3, -0.45, 0.1], second)):
        T = np.array([1, 0, 0, 0, *t], F32)
        scans += [(T, p, c) for c in tx.EDGE_CFGS]
    exp, _, n_col = _mode0(ctx, oracle, 0.25, 8, scans)
    assert all(e[0] == e[1] for e in exp)
    # 15 axis points within or beyond the lengths, 4 huge finite, 5 on faces, 5 in one voxel, 3 clearing
    assert exp[0][0] == 32 and n_col > 20


def test_ray_edges_simple_bit_exact(ctx, oracle):
    """Crafted points at 0.25 m voxels (faces exactly representable) from a sensor on a block corner
    and from one inside a voxel, under four configurations, accumulated in one submap."""
    _ray_edges(ctx, oracle, tx.edge_points())


def test_ray_edges_permuted_bit_exact(ctx, oracle):
    """The same, with the second sensor's points in an order that interleaves the valid points with the NaN,
    inf and huge ones, so a ray colour taken from the wrong point index shows."""
    pts = tx.edge_points()
    _ray_edges(ctx, oracle, pts[np.random.RandomState(4).permutation(len(pts))])


def _segment_streams(n):
    """Saturated (integer 2^6 weights far behind the sensor), mixed (sdf below 2 trunc at the sensor voxel,
    fractional weights) and band (points 1, 3 and 4 of every 5 lie 0.35-0.5 m away: band updates at the sensor
    voxel, in every batch and in the one-tuple tails at 65, 97 and 129)."""
    return {"saturated": tx.ring(n, 0.125, [3.0, 4.2, 5.5]),
            "mixed": tx.ring(n, [0.125, 0.3, 0.125, -0.2, 0.125, 0.125, 0.125], [3.0, 1.0, 4.2, 5.5, 1.1]),
            "band": tx.ring(n, [0.125, 0.3, -0.2], [3.0, 0.35, 4.2, 0.5, 0.42])}


@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 128, 129])
def test_segment_lengths(ctx, oracle, n):
    """N rays with carving from one sensor, each stream integrated twice: the sensor voxel's segment has
    exactly N tuples per call (short path up to 64, warp path with 32-tuple batches and a tail beyond)."""
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.0])
    sensor = tx.voxel_keys([[0, 0, 0]])[0]
    for name, pts in _segment_streams(n).items():
        exp, traces, _ = _mode0(ctx, oracle, 0.2, 16, [(T, pts), (T, pts)], seed=n, use_const_weight=0)
        keys, _, s, _ = traces[0]
        at = keys == sensor
        assert np.count_nonzero(at) == n
        if name == "band":
            assert np.count_nonzero(np.abs(s[at]) < F32(0.6)) == sum(i % 5 in (1, 3, 4) for i in range(n))
        if name == "saturated" and n >= 65:
            assert exp[1][4] > 0
        if n <= 64:
            assert exp[0][4] == exp[1][4] == 0


@pytest.mark.parametrize("vs,vps", [(0.2, 16), (0.05, 8)])
def test_clearing_rays_in_the_band(ctx, oracle, vs, vps):
    """Clearing rays whose last voxels lie inside the band, twice from one pose."""
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.3])
    exp, traces, n_col = _mode0(ctx, oracle, vs, vps, [(T, tx.clearing_points(vs))] * 2, max_ray_length_m=8.0)
    assert exp[0][:2] == (400, 400)
    _, r, s, _ = traces[0]
    assert len(np.unique(r[np.abs(s) < F32(0.6)])) > 100 and n_col > 100


def _run_fast(ctx, oracle, vs, vps, T, pts, **kw):
    ocfg = oracle.tsdf_config(**{**tx.FAST_ALL, **kw})
    layer = oracle.Layer(vs, vps)
    st, g, s, u = oracle.tsdf_integrate_trace(layer, ocfg, T, pts)
    assert st.rays_cast == st.rays_valid            # every ray is cast: the update set is fixed
    sid = next(_ids)
    ctx.submap_create(sid, vs, vps, layer.num_blocks)
    try:
        sg = ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(**{**tx.FAST_ALL, **kw}))
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
    info = _run_fast(ctx, oracle, 0.2, 16, synth.pose_to_T([0.3, -0.2, 0.1, 0.4]), pts)
    assert info["max_updates"] > 10000 and info["inner"] > 1000 and info["single"] > 1000


def test_fast_serialisation_ray_edges(ctx, oracle):
    """The crafted points in the Fast schedule.  The one-ulp neighbours of the length limits are left
    out: after the sensor translation they can land on the same float point, and the Fast schedule
    then rightly casts only one of them."""
    pts = tx.edge_points()
    keep = np.ones(len(pts), bool); keep[[0, 1, 2, 6, 7, 8, 9, 10, 11, 15, 16, 17]] = False
    for c in tx.EDGE_CFGS:
        _run_fast(ctx, oracle, 0.25, 8, np.array([1, 0, 0, 0, 0.3, -0.45, 0.1], F32), pts[keep], **c)


@pytest.mark.parametrize("mode", [0, 1])
def test_capacity_at_the_edge(ctx, oracle, world, mode):
    """Capacity equal to the oracle's block count succeeds; one block less fails with
    VGX_ERR_CAPACITY and leaves exactly `capacity` blocks, all of them in the oracle's set."""
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=8, n_azimuth=128, seed=3)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    kw = tx.FAST_ALL if mode == 1 else {}
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
