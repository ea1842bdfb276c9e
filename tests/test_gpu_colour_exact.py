"""Voxel colour pinned across the matrices the colourless kernels are pinned on (tests/test_gpu_fast_schedule.py,
tests/test_gpu_colour_map.py), against the exact models of tests/colour_exact.py.  Ray-ordered (mode 0) colour is
pinned with distance and weight in tests/test_gpu_tsdf_exact.py.

Every ray carries a colour of its own whose four channels differ, so an update applied out of order, with the
wrong weight or with another ray's colour changes the bytes.

* Clearing rays whose last voxels lie inside the band, in mode 1 with every ray cast.
* Fast scheduling (mode 1) at voxgraph's schedule (start-cell factor 2, two collisions): the race-aware model of
  tests/fast_schedule.py decodes which rays updated each voxel, and the colour contract of csrc/tsdf.cu is
  checked on that decoding; a one-colour scan at the default configuration.
* Projection colour at three resolutions against tests/project_colour_oracle.c, with poses that put sample points
  on voxel centres, in three id orders.
* Mesh vertex colours on crafted layers whose vertices sit exactly on voxel and block faces, against the
  containing-voxel rule, and in the PLY."""
import itertools

import numpy as np
import pytest

import colour_exact as cx
import fast_schedule as fs
import mesh_exact as me
import project_colour_oracle as pco
import project_oracle as po
import tsdf_exact as tx
from support import ctx, world, yaw_T  # noqa: F401
from voxgraph_b200 import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
_ids = itertools.count(11000)
VOXGRAPH = dict(start_voxel_subsampling_factor=2.0, max_consecutive_ray_collisions=2)


# ---------------------------------------------------------------------- clearing rays
def _contract(ctx, oracle, vs, vps, T, pts, rgba, **kw):
    """One mode-1 call with every ray cast into an empty coloured submap and its colourless twin: statistics,
    block set and the order-free integer weights equal; a voxel with one update holds the exact rule, one with
    more lies channel-wise within black and its band rays' colours, one without a band update stays 0.
    -> (ray index, sdf) of every tuple."""
    ocfg = oracle.tsdf_config(**{**tx.FAST_ALL, **kw})
    layer = oracle.Layer(vs, vps)
    _, g, s, u, r = cx.trace_rays(oracle, layer, ocfg, T, pts)
    cfg = ctx.tsdf_config(**{**tx.FAST_ALL, **kw})
    plain, col = next(_ids), next(_ids)
    try:
        res = {}
        for sid in (plain, col):
            ctx.submap_create(sid, vs, vps, layer.num_blocks)
            sg = ctx.tsdf_integrate(sid, T, pts, cfg, rgba=rgba if sid == col else None)
            res[sid] = (sg.rays_valid, sg.rays_cast, sg.voxel_updates, sg.blocks_allocated)
        assert res[col] == res[plain]
        kp, _, wp = tx.layer_voxels(*ctx.submap_download(plain), vps)
        idx, d, w = ctx.submap_download(col)
        k_all, _, w_all = tx.layer_voxels(idx, d, w, vps)
        c_all = cx.layer_colours(idx, ctx.submap_download_colour(col), vps)[1]
    finally:
        for sid in (plain, col):
            ctx.submap_free(sid)
    assert np.array_equal(kp, k_all) and np.array_equal(wp.view(np.uint32), w_all.view(np.uint32))
    trunc = F32(ocfg.default_truncation_distance)
    keys = tx.voxel_keys(g)
    o = np.argsort(keys, kind="stable")
    ks, ss, us, rws = keys[o], s[o], u[o], cx.pack(rgba)[r][o]
    uniq, start, cnt = np.unique(ks, return_index=True, return_counts=True)
    at = np.searchsorted(k_all, uniq)
    assert np.array_equal(k_all[at], uniq)
    rest = np.ones(len(k_all), bool); rest[at] = False
    assert not c_all[rest].any()
    one = cnt == 1
    j = start[one]
    zero_w, zero_c = np.zeros(len(j), F32), np.zeros(len(j), np.uint32)
    assert np.array_equal(c_all[at[one]], cx.colour_step(trunc, ss[j], us[j], zero_w, rws[j], zero_c))
    band = np.abs(ss) < trunc
    seg = np.repeat(np.arange(len(uniq)), cnt)
    hi = np.zeros((len(uniq), 4), np.int64)
    ch = cx.unpack(rws).astype(np.int64)
    for c4 in range(4):
        np.maximum.at(hi[:, c4], seg[band], ch[band, c4])
    assert (cx.unpack(c_all[at]).astype(np.int64) <= hi).all()
    has_band = np.zeros(len(uniq), bool); has_band[seg[band]] = True
    assert not c_all[at[~has_band]].any()
    return r, s


@pytest.mark.parametrize("vs,vps", [(0.2, 16), (0.05, 8)])
def test_mode1_clearing_rays_in_the_band(ctx, oracle, vs, vps):
    pts = tx.clearing_points(vs, seed=1)
    rgba = cx.colours(np.random.RandomState(2), len(pts))
    r, s = _contract(ctx, oracle, vs, vps, synth.pose_to_T([0.1, 0.1, 0.1, 0.3]), pts, rgba, max_ray_length_m=8.0)
    assert len(np.unique(r[np.abs(s) < F32(0.6)])) > 100


# ---------------------------------------------------------------------- mode 1 at voxgraph's schedule
N_PAD = 400
LAYOUTS = {"warp": lambda k: [3 + 9 * i for i in range(k)],          # where the real rays sit in the padded
           "warps": lambda k: [5 + 37 * i for i in range(k)],        # list: one warp, several warps, several
           "ctas": lambda k: [2 + 131 * i for i in range(k)]}        # CTAs


def _fast_colour(ctx, sc, positions, slot_rgba, reach=None):
    """The scene's points at `positions` of a NaN-padded list (every entry with a colour; equal points share
    their slot's colour) into a fresh coloured submap; the race-aware checker on the layer, then the colour
    contract on the decoded updates (previous weight and colour 0): one update -> the exact rule, several ->
    every channel at most the largest of the band rays' channels, no band update -> 0.  -> checker info."""
    pts = np.full((N_PAD, 3), np.nan, F32)
    pts[positions] = sc.pts
    rgba = cx.colours(np.random.RandomState(len(positions)), N_PAD)
    for i in sc.valid:
        rgba[positions[i]] = slot_rgba[sc.rays[i].slot]
    cap = len({sc.block(g) for i in sc.valid for g in sc.rays[i].seq}) + 1
    sid = next(_ids)
    ctx.submap_create(sid, sc.vs, sc.vps, cap)
    try:
        st = ctx.tsdf_integrate(sid, sc.T, pts, ctx.tsdf_config(**dict(sc.kw, max_consecutive_ray_collisions=sc.m)),
                                rgba=rgba)
        lay = ctx.submap_download(sid)
        words = ctx.submap_download_colour(sid)
    finally:
        ctx.submap_free(sid)
    info = sc.check(lay, (st.rays_valid, st.rays_cast, st.voxel_updates, st.blocks_allocated), reach)
    _, ps = sc.decode(lay)
    per = {}
    for slot, p in enumerate(ps):
        ray = sc.rays[sc.slots[slot][0]]
        word = cx.pack(slot_rgba[slot:slot + 1])[0]
        for k in range(p):
            per.setdefault(ray.seq[k], []).append((ray.sdf[k], ray.uw[k], word))
    k_all, c_all = cx.layer_colours(lay[0], words, sc.vps)
    for g, ups in per.items():
        c = c_all[np.searchsorted(k_all, tx.voxel_keys([g])[0])]
        band = [w for s, _, w in ups if abs(s) < sc.trunc]
        if len(ups) == 1:
            s, u, w = ups[0]
            exp = cx.colour_step(sc.trunc, np.array([s], F32), np.array([u], F32), np.zeros(1, F32),
                                 np.array([w], np.uint32), np.zeros(1, np.uint32))[0]
            assert c == exp, ("one update", g, hex(int(c)), hex(int(exp)))
        elif band:
            hi = cx.unpack(np.array(band, np.uint32)).max(0)
            assert (cx.unpack(np.array([c], np.uint32))[0] <= hi).all(), ("range", g, hex(int(c)))
        else:
            assert c == 0, ("no band update", g, hex(int(c)))
    touched = np.isin(k_all, tx.voxel_keys(list(per)) if per else np.zeros(0, np.int64))
    assert not c_all[~touched].any()
    info["single_band"] = sum(1 for ups in per.values() if len(ups) == 1 and abs(ups[0][0]) < sc.trunc)
    info["multi_band"] = sum(1 for ups in per.values() if len(ups) > 1 and any(abs(s) < sc.trunc for s, _, _ in ups))
    return info


def _voxgraph_scene(oracle, vs, vps, T, pts, cfg):
    sc = fs.Scene(oracle, vs, vps, T, pts, **dict(cfg, **VOXGRAPH))
    assert sc.m == 2
    return sc


@pytest.mark.parametrize("sensor", ["origin", "negative"])
@pytest.mark.parametrize("vs,vps", fs.RES)
def test_mode1_voxgraph_schedule_micro_scenes(ctx, oracle, vs, vps, sensor):
    """Every micro scene built for start-cell factor 2, run at two collisions: the outcome is one of the
    interleavings and the colours keep the contract on the decoded updates."""
    names = fs.MICRO_NAMES + (["marker_block"] if sensor == "origin" else [])
    rs = np.random.RandomState(int(vs * 100) + vps)
    tot = dict(single_band=0, multi_band=0, breaks=0)
    for n, name in enumerate(names):
        T, pts, cfg = fs.micro_scene(name, vs, 2, sensor)
        sc = _voxgraph_scene(oracle, vs, vps, T, pts, cfg)
        fs.assert_micro_property(sc, name, sensor)
        reach = {sc.canonical(o) for o in sc.reachable()}
        layout = list(LAYOUTS)[n % 3]
        try:
            info = _fast_colour(ctx, sc, LAYOUTS[layout](len(pts)), cx.colours(rs, len(sc.slots)), reach)
        except AssertionError as e:
            raise AssertionError((name, layout, str(e)))
        for k in tot:
            tot[k] += info[k]
    assert tot["single_band"] > 0 and tot["multi_band"] > 0


def test_mode1_voxgraph_schedule_random_scenes(ctx, oracle):
    """120 decoded random scenes (2-11 rays) rebuilt at start-cell factor 2 and two collisions, at random
    places of the padded list."""
    rs = np.random.RandomState(8)
    tot = dict(single_band=0, multi_band=0, breaks=0, skips=0)
    for k in range(120):
        base = fs.random_scene(oracle, rs)
        sc = _voxgraph_scene(oracle, base.vs, base.vps, base.T, base.pts, base.kw)
        assert sc.decodable()
        positions = np.sort(rs.choice(N_PAD, len(sc.pts), replace=False))
        try:
            info = _fast_colour(ctx, sc, positions, cx.colours(rs, len(sc.slots)))
        except AssertionError as e:
            raise AssertionError((k, sc.kw, str(e)))
        for key in tot:
            tot[key] += info[key]
    print("random scenes at voxgraph's schedule:", tot)
    assert tot["single_band"] > 100 and tot["multi_band"] > 20 and tot["breaks"] > 0 and tot["skips"] > 0


def test_mode1_one_colour_default_config(ctx, oracle, world):
    """Every ray one colour c at the default configuration (voxgraph's schedule, drop-off and sparsity factor
    on).  Which rays are cast and where they stop depends on the race, so the update set is bounded by the
    trace with every ray cast: an updated voxel lies on it; one whose every traced update is in the band holds
    exactly c; one with band and other updates lies between black and c; every other voxel stays 0."""
    vs, vps = 0.2, 16
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=8, n_azimuth=64, seed=1, miss_range=40.0)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    c = np.array([201, 17, 96, 254], np.uint8)
    ocfg = oracle.tsdf_config(mode=1, start_voxel_subsampling_factor=1e3, max_consecutive_ray_collisions=1 << 30)
    _, g, s, _, _ = cx.trace_rays(oracle, oracle.Layer(vs, vps), ocfg, T, pts)
    sid = next(_ids)
    ctx.submap_create(sid, vs, vps, 4096)
    try:
        st = ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(mode=1), rgba=np.tile(c, (len(pts), 1)))
        idx, d, w = ctx.submap_download(sid)
        words = ctx.submap_download_colour(sid)
    finally:
        ctx.submap_free(sid)
    assert 0 < st.voxel_updates < len(s)                   # the collision cut-off stops rays
    k_all, _, w_all = tx.layer_voxels(idx, d, w, vps)
    c_all = cx.layer_colours(idx, words, vps)[1]
    keys = tx.voxel_keys(g)
    in_band = np.abs(s) < F32(ocfg.default_truncation_distance)
    band = np.unique(keys[in_band])
    pure = np.setdiff1d(band, np.unique(keys[~in_band]))
    upd = w_all > 0
    assert np.isin(k_all[upd], keys).all()
    at_pure = np.isin(k_all, pure) & upd
    assert np.count_nonzero(at_pure) > 200
    assert (c_all[at_pure] == cx.pack(c[None])[0]).all()
    mixed = np.isin(k_all, band) & ~np.isin(k_all, pure)
    assert np.count_nonzero(mixed & upd) > 20 and (cx.unpack(c_all[mixed]) <= c).all()
    assert not c_all[~np.isin(k_all, band) | ~upd].any()


# ---------------------------------------------------------------------- projection
RES3 = [(0.1, 16), (0.05, 32), (0.2, 8)]


@pytest.fixture(scope="module")
def layers3(oracle, world):
    """Per resolution, five submaps integrated by the oracle from small scans around the room, each with random
    colour words on every voxel (the third one without a channel), and their poses: yaw 0 or pi/2 and
    translations of whole voxels or whole blocks.  -> {(vs, vps): [(idx, d, w, words or None, T)]}"""
    out = {}
    rs = np.random.RandomState(12)
    for vs, vps in RES3:
        bs = float(F32(vs)) * vps
        poses = [yaw_T(0.0), yaw_T(np.pi / 2, (3 * vs, -2 * vs, vs)), yaw_T(0.0, (bs, -bs, 0.0)),
                 yaw_T(np.pi / 2, (-bs, 2 * bs, 0.0)), yaw_T(0.0, (-5 * vs, 7 * vs, -vs))]
        subs = []
        for k, (px, py, yaw) in enumerate([(15.0, 15.0, 0.0), (16.0, 14.5, 0.5), (14.2, 15.8, -0.8),
                                           (15.5, 16.2, 1.3), (13.8, 14.1, 2.4)]):
            layer = oracle.Layer(vs, vps)
            pts = synth.lidar_scan(world, np.array([px, py, 1.2, yaw]), n_beams=8, n_azimuth=128, seed=20 + k)
            oracle.tsdf_integrate(layer, oracle.tsdf_config(max_ray_length_m=4.0), synth.pose_to_T([0, 0, 0, 0]), pts)
            idx, d, w = layer.export()
            words = rs.randint(0, 2 ** 32, w.shape, dtype=np.uint64).astype(np.uint32) if k != 2 else None
            subs.append((idx, d, w, words, poses[k]))
        out[(vs, vps)] = subs
    return out


@pytest.mark.parametrize("pick", [(0, 1), (0, 1, 2, 3, 4)], ids=["two", "five"])
@pytest.mark.parametrize("vs,vps", RES3)
def test_projection_colour_matrix(ctx, oracle, layers3, vs, vps, pick):
    subs = layers3[(vs, vps)]
    ids = {}
    try:
        for k in pick:
            ids[k] = next(_ids)
            idx, d, w, words, _ = subs[k]
            ctx.submap_upload(ids[k], vs, vps, idx, d, w)
            if words is not None:
                ctx.submap_upload_colour(ids[k], words)
        ref = None
        for order in (list(pick), list(pick)[::-1], list(np.random.RandomState(1).permutation(pick))):
            sids = [ids[i] for i in order]
            T = np.array([subs[i][4] for i in order], F32)
            out = next(_ids)
            ctx.project_map(sids, T, out)
            try:
                idx, d, w = ctx.submap_download(out)
                assert ctx.submap_has_colour(out)
                words = ctx.submap_download_colour(out)
            finally:
                ctx.submap_free(out)
            layers = [oracle.Layer.from_blocks(vs, vps, *subs[i][:3]) for i in order]
            exp = po.project_layers(layers, T, sids).export()
            tx.assert_layers_bit_equal(exp, (idx, d, w))
            ec, ew = pco.project(vs, vps, [subs[i][:4] for i in order], T, sids, idx)
            assert np.array_equal(ew.view(np.uint32), w.view(np.uint32))
            bad = np.nonzero(words != ec)
            assert bad[0].size == 0, (order, len(bad[0]), hex(int(words[bad][0])), hex(int(ec[bad][0])))
            assert np.count_nonzero(words) > 1000
            if ref is None:
                ref = (idx, words)
            else:
                assert np.array_equal(ref[0], idx) and np.array_equal(ref[1], words)
    finally:
        for sid in ids.values():
            ctx.submap_free(sid)


# ---------------------------------------------------------------------- mesh
def _crafted(vs, vps, kind, rs):
    """A crafted layer (idx, d, w, words).  Blocks around the origin with negative indices and gaps, so some
    block faces have no neighbour.  'x' / 'y' / 'z': distance +h or -h by bands of 1-3 voxels along one axis,
    every sign change across a voxel face (block faces included) with d0 = -d1, so its vertex sits on the face
    (t = 1/2); 'sphere': a generic surface.  Weight 5 except 3% of the voxels at 0; random colour words."""
    blocks = [(bx, by, bz) for bx in (-2, -1, 0, 1) for by in (-1, 0, 1) for bz in (-1, 0)
              if (bx + 2 * by + 3 * bz) % 5 != 1]
    idx = np.array(blocks, np.int32)
    lin = np.arange(vps ** 3)
    loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], -1)
    g = idx[:, None, :].astype(np.int64) * vps + loc[None]
    h = F32(0.37 * vs)
    if kind == "sphere":
        c = (g + 0.5) * float(F32(vs))
        d = (np.linalg.norm(c - np.array([0.13, -0.07, 0.02]), axis=-1) - 0.61 * vps * vs).astype(F32)
    else:
        a = "xyz".index(kind)
        cuts = np.cumsum(rs.randint(1, 4, 200)) - 100 * 2          # band edges every 1-3 voxels
        cuts = np.union1d(cuts, np.arange(-3, 4) * vps)             # and on every block face
        sign = np.searchsorted(cuts, g[..., a], side="right") % 2
        d = np.where(sign == 1, h, -h).astype(F32)
    w = np.where(rs.rand(*d.shape) < 0.03, 0.0, 5.0).astype(F32)
    words = rs.randint(0, 2 ** 32, d.shape, dtype=np.uint64).astype(np.uint32)
    return idx, d, w, words


@pytest.mark.parametrize("vs", [0.1, 0.05])
@pytest.mark.parametrize("vps", [8, 16, 32])
def test_mesh_vertex_colours_on_faces(ctx, vs, vps):
    """Vertex colours of four crafted submaps (submap frames) equal the containing-voxel rule, including the
    vertices whose position times voxel_size_inv rounds to just below a face index (the rule's 1e-6 decides
    them); the PLY carries the same positions and colour bytes."""
    rs = np.random.RandomState(vps + int(vs * 100))
    subs = [_crafted(vs, vps, kind, rs) for kind in ("x", "y", "z", "sphere")]
    sids = []
    try:
        for idx, d, w, words in subs:
            sids.append(next(_ids))
            ctx.submap_upload(sids[-1], vs, vps, idx, d, w)
            ctx.submap_upload_colour(sids[-1], words)
        vo, _ = ctx.mesh_build(sids, None, ctx.mesh_config(min_weight=2.0))
        xyz, tri = ctx.mesh_download()
        col = ctx.mesh_colours()
        pal = np.array([[9, 8, 7, 6]] * len(sids), np.uint8)
        pxyz, prgba, ptri = me.read_ply(ctx.mesh_ply(pal, voxel_colours=True))
    finally:
        for sid in sids:
            ctx.submap_free(sid)
    assert np.array_equal(pxyz.view(np.uint32), xyz.view(np.uint32)) and np.array_equal(ptri, tri)
    inv = F32(1.0 / float(F32(vs)))
    tight = 0
    for k, (idx, _, _, words) in enumerate(subs):
        a, b = vo[k], vo[k + 1]
        assert b - a > 200
        exp = cx.vertex_colours(xyz[a:b], vs, vps, idx, words)
        bad = np.nonzero(col[a:b] != exp)[0]
        assert bad.size == 0, (k, len(bad), xyz[a + bad[0]], hex(int(col[a + bad[0]])), hex(int(exp[bad[0]])))
        assert np.array_equal(prgba[a:b], cx.unpack(exp))
        assert np.count_nonzero(exp) == b - a                   # every containing voxel exists
        p = xyz[a:b] * inv
        tight += int(np.count_nonzero(np.floor(p) != np.floor((p + F32(1e-6)).astype(F32))))
    assert tight > 0
