"""The Fast TSDF schedule (mode 1, what voxgraph runs) on the device, checked against the race-aware model
tests/fast_schedule.py: start-voxel de-duplication, the consecutive-collision cut-off, the ~0 marker
rule and the clearing of both approximate sets between calls.

Rays are made readable by their weights: with constant weights, drop-off and sparsity compensation off,
a ray's update weight is 1/z^2, and every ray of a call gets a distinct power of four, so a voxel's
weight spells out which rays updated it.  Micro scenes (2-3 rays) must give an outcome of the exact
interleaving search; random scenes of up to 11 rays pass the checker's rules.  The real rays sit at
chosen places in a list padded with NaN points (invalid: they touch neither set), in one warp, in
several warps or in several CTAs."""
import itertools

import numpy as np
import pytest

import fast_schedule as fs
import tsdf_exact as tx
from support import ctx  # noqa: F401
from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
_ids = itertools.count(4000)
N_PAD = 400
LAYOUTS = {"warp": lambda k: [3 + 9 * i for i in range(k)],
           "warps": lambda k: [5 + 37 * i for i in range(k)],
           "ctas": lambda k: [2 + 131 * i for i in range(k)]}


def _device(ctx, sc, positions):
    """Integrate the scene's points at `positions` of a NaN-padded list into a fresh submap ->
    (stats tuple, layer)."""
    pts = np.full((N_PAD, 3), np.nan, F32)
    pts[positions] = sc.pts
    cap = len({sc.block(g) for i in sc.valid for g in sc.rays[i].seq}) + 1
    sid = next(_ids)
    ctx.submap_create(sid, sc.vs, sc.vps, cap)
    try:
        st = ctx.tsdf_integrate(sid, sc.T, pts, ctx.tsdf_config(**dict(sc.kw, max_consecutive_ray_collisions=sc.m)))
        lay = ctx.submap_download(sid)
    finally:
        ctx.submap_free(sid)
    return (st.rays_valid, st.rays_cast, st.voxel_updates, st.blocks_allocated), lay


def _add(total, info):
    for k in ("breaks", "skips", "marker"):
        total[k] += info[k]


@pytest.mark.parametrize("sensor", ["origin", "negative"])
@pytest.mark.parametrize("vs,vps", fs.RES)
def test_micro_scenes(ctx, oracle, vs, vps, sensor):
    """Every micro scene at collision limits 0, 1, 2, 7 and start-cell factors 1, 2, 4: the decoded
    outcome is one of the interleavings, and every voxel's distance is one of its update orders."""
    names = fs.MICRO_NAMES + (["marker_block"] if sensor == "origin" else [])
    total = dict(breaks=0, skips=0, marker=0)
    multi = 0
    for n, (factor, name) in enumerate(itertools.product(fs.FACTORS, names)):
        T, pts, cfg = fs.micro_scene(name, vs, factor, sensor)
        sc = fs.Scene(oracle, vs, vps, T, pts, **cfg)
        fs.assert_micro_property(sc, name, sensor)
        for k, m in enumerate(fs.MS):
            sc.m = m
            reach = {sc.canonical(o) for o in sc.reachable()}
            multi += len(reach) > 1
            layout = list(LAYOUTS)[(n + k) % 3]
            st, lay = _device(ctx, sc, LAYOUTS[layout](len(pts)))
            try:
                _add(total, sc.check(lay, st, reach))
            except AssertionError as e:
                raise AssertionError((name, factor, m, layout, st, str(e)))
    print("micro %s %s: device breaks %d, skips %d, ~0 collisions %d; %d runs with races possible"
          % ((vs, vps), sensor, total["breaks"], total["skips"], total["marker"], multi))
    assert total["breaks"] > 0 and total["skips"] > 0 and multi > 0
    if sensor == "origin":
        assert total["marker"] > 0


def test_decoded_random_scenes(ctx, oracle):
    """300 calls of 2-11 rays (random geometry, resolution, factor, collision limit, carving, sensor)
    at random places of the padded list, through the checker."""
    rs = np.random.RandomState(5)
    total = dict(breaks=0, skips=0, marker=0)
    for k in range(300):
        sc = fs.random_scene(oracle, rs)
        positions = np.sort(rs.choice(N_PAD, len(sc.pts), replace=False))
        st, lay = _device(ctx, sc, positions)
        try:
            _add(total, sc.check(lay, st))
        except AssertionError as e:
            raise AssertionError((k, sc.m, sc.kw, st, str(e)))
    print("random scenes: device breaks %d, skips %d, ~0 collisions %d"
          % (total["breaks"], total["skips"], total["marker"]))
    assert total["breaks"] > 0 and total["skips"] > 0


def test_sets_are_cleared_between_calls(ctx, oracle):
    """A scene with one reachable outcome (a duplicate pair, a ray through voxel (-1, 0, 0) at the
    identity, separate truncation bands) integrated twice into one submap: the same rays are cast and
    update the same voxels both times, so every weight doubles exactly."""
    u = 0.1
    z8, z9, z10, z7 = 2.0 ** -8, 2.0 ** -9, 2.0 ** -10, 2.0 ** -7
    pts = np.array([(8 * u, 0.3 * u, z8), (8 * u, 0.3 * u, z8), (0.2 * u, 9 * u, z9), (-7 * u, -3 * u, z10),
                    (-2.3 * u, 0.45 * u, z7)], F32)
    for m in (0, 2):
        sc = fs.Scene(oracle, u, 16, fs.pose((0.0, 0.0, 0.0)), pts, **fs.BASE, default_truncation_distance=3 * u,
                      voxel_carving_enabled=0, max_consecutive_ray_collisions=m)
        reach = {sc.canonical(o) for o in sc.reachable()}
        assert len(reach) == 1 and fs.MARKER in sc.rays[4].vh
        exp = sc.simulate()
        cfg = ctx.tsdf_config(**dict(sc.kw, max_consecutive_ray_collisions=m))
        sid = next(_ids)
        ctx.submap_create(sid, u, 16, 64)
        try:
            s1 = ctx.tsdf_integrate(sid, sc.T, pts, cfg)
            l1 = ctx.submap_download(sid)
            s2 = ctx.tsdf_integrate(sid, sc.T, pts, cfg)
            l2 = ctx.submap_download(sid)
        finally:
            ctx.submap_free(sid)
        st = (s1.rays_valid, s1.rays_cast, s1.voxel_updates, s1.blocks_allocated)
        assert st == sc.stats(exp)
        sc.check(l1, st, reach)
        assert (s2.rays_valid, s2.rays_cast, s2.voxel_updates, s2.blocks_allocated) == st[:3] + (0,)
        assert np.array_equal(l1[0], l2[0])
        assert np.array_equal(l2[2], 2 * l1[2])


def test_dense_scan_voxgraph_schedule(ctx, oracle):
    """A 32 x 512 scan at voxgraph's schedule (start-cell factor 2, two collisions) with constant
    weights, no drop-off and no sparsity factor, so a voxel's weight counts its updates: the weights
    add up to voxel_updates, every updated voxel lies on the full sequences of at least w rays,
    rays_cast is what the start keys allow, and every block holds a voxel of some sequence."""
    world = synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=32, n_azimuth=512, seed=1,
                           miss_range=40.0)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    vs, vps = 0.2, 16
    kw = dict(mode=1, use_const_weight=1, use_weight_dropoff=0, use_sparsity_compensation_factor=0,
              max_weight=1e7, start_voxel_subsampling_factor=2.0, max_consecutive_ray_collisions=2)
    # full sequences of every ray: the oracle with every ray cast and no cut-off
    layer = oracle.Layer(vs, vps)
    ost, g, _, _ = oracle.tsdf_integrate_trace(
        layer, oracle.tsdf_config(**dict(kw, start_voxel_subsampling_factor=1e3, max_consecutive_ray_collisions=1 << 30)),
        T, pts)
    assert ost.rays_cast == ost.rays_valid
    seq_keys, seq_count = np.unique(tx.voxel_keys(g), return_counts=True)
    seq_blocks = {tuple(b) for b in np.unique(g >> 4, axis=0).tolist()}    # vps = 16
    # start keys of the valid points
    cfg = oracle.tsdf_config(**kw)
    inv = F32(F32(2.0) * F32(layer.voxel_size_inv))
    keys = {}
    for p in pts:
        if not np.all(np.isfinite(p)):
            continue
        rd = np.sqrt(F32(F32(F32(p[0] * p[0]) + F32(p[1] * p[1])) + F32(p[2] * p[2])))
        if rd < F32(cfg.min_ray_length_m) or (rd > F32(cfg.max_ray_length_m) and not cfg.allow_clear):
            continue
        h = fs.any_index_hash(*fs.start_key(oracle.T_transform(T, p), inv))
        keys.setdefault(h & fs.MASK, {}).setdefault(h, 0)
        keys[h & fs.MASK][h] += 1
    assert sum(sum(k.values()) for k in keys.values()) == ost.rays_valid
    lo = hi = 0
    for k in keys.values():
        assert fs.MARKER not in k
        n = sorted(k.values())
        lo += len(n)
        big, rest = n[-1], sum(n[:-1])
        hi += len(n) if len(n) == 1 else (sum(n) if big <= rest + 1 else 2 * rest + 1)
    sid = next(_ids)
    ctx.submap_create(sid, vs, vps, len(seq_blocks) + 1)
    try:
        st = ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(**kw))
        gi, gd, gw = ctx.submap_download(sid)
    finally:
        ctx.submap_free(sid)
    assert st.rays_valid == ost.rays_valid
    assert lo <= st.rays_cast <= hi, (lo, st.rays_cast, hi)
    assert 0 < st.voxel_updates < ost.voxel_updates
    assert float(gw.astype(np.float64).sum()) == st.voxel_updates
    vk, vd, vw = tx.layer_voxels(gi, gd, gw, vps)
    upd = vw > 0
    pos = np.searchsorted(seq_keys, vk[upd])
    assert np.all(pos < len(seq_keys)) and np.array_equal(seq_keys[pos], vk[upd]), "voxel off every ray"
    assert np.all(vw[upd] <= seq_count[pos]) and np.all(vw[upd] == np.rint(vw[upd]))
    assert not np.any(vd[~upd])
    assert {tuple(b) for b in gi.tolist()} <= seq_blocks
    assert st.blocks_allocated == len(gi)
    print("dense scan: rays valid %d, cast %d (start keys allow %d..%d), updates %d of %d"
          % (st.rays_valid, st.rays_cast, lo, hi, st.voxel_updates, ost.voxel_updates))

