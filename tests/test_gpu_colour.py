"""Voxel colour on the device, against the exact models of tests/colour_exact.py.

Mode 1: the stated contract (exact where a voxel has one update in the call, channel-wise range elsewhere, exact
for a one-colour scene; weights, statistics and the block set independent of colours), one run each.  Host and
device colour uploads and downloads.  Collection files carry the channel; submaps that never saw a colour have no
channel and save as before.  Ray-ordered (mode 0) colour is pinned in test_gpu_tsdf_exact.py."""
import itertools

import numpy as np
import pytest

import collection_stream as cs
import colour_exact as cx
import tsdf_exact as tx
from support import ctx, world  # noqa: F401
from voxgraph_b200 import _lib, api, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
_ids = itertools.count(7000)


def _fast_pair(ctx, vs, vps, cap, calls):
    """The calls [(T, pts, rgba)] in mode 1 into one coloured and one colourless submap -> per call the coloured
    submap's (idx, d, w, colour words) after it; checks contract (c) along the way."""
    cfg = ctx.tsdf_config(**tx.FAST_ALL)
    plain, col = next(_ids), next(_ids)
    out = []
    try:
        for sid in (plain, col):
            ctx.submap_create(sid, vs, vps, cap)
        for (T, pts, rgba) in calls:
            res = {}
            for sid in (plain, col):
                before = ctx.launch_count
                sg = ctx.tsdf_integrate(sid, T, pts, cfg, rgba=rgba if sid == col else None)
                res[sid] = (sg.rays_valid, sg.rays_cast, sg.voxel_updates, sg.blocks_allocated,
                            ctx.launch_count - before)
            assert res[col] == res[plain]
            ip, dp, wp = ctx.submap_download(plain)
            ic, dc, wc = ctx.submap_download(col)
            kp, dps, wps = tx.layer_voxels(ip, dp, wp, vps)
            kc, dcs, wcs = tx.layer_voxels(ic, dc, wc, vps)
            assert np.array_equal(kp, kc)                                        # the block set
            assert np.array_equal(wps.view(np.uint32), wcs.view(np.uint32))      # integer weights: order free
            out.append((ic, dc, wc, ctx.submap_download_colour(col), (kp, dps)))
        assert not ctx.submap_has_colour(plain) and ctx.submap_has_colour(col)
    finally:
        for sid in (plain, col):
            ctx.submap_free(sid)
    return out


def test_mode1_contract(ctx, oracle):
    """Two calls from different poses.  Every voxel with one update in a call must hold the exact rule; the others
    stay channel-wise between the previous colour and the band rays' colours; no band update, no change."""
    vs, vps = 0.2, 16
    rs = np.random.RandomState(3)
    calls = []
    for k, (t, n) in enumerate([((0.1, 0.1, 0.1), 150), ((1.3, -0.8, 0.2), 140)]):
        pts = tx.ring(n, np.linspace(-0.8, 0.9, 7), [3.0, 4.2, 5.5, 2.4], az0=0.1 + 0.37 * k)
        palette = rs.randint(0, 256, (2, 4)).astype(np.uint8)          # two colours per call
        calls.append((synth.pose_to_T([*t, 0.3 * k]), pts, palette[rs.randint(0, 2, n)]))
    ocfg = oracle.tsdf_config(**tx.FAST_ALL)
    layer = oracle.Layer(vs, vps)
    traces = [cx.trace_rays(oracle, layer, ocfg, T, pts)[1:] for (T, pts, _) in calls]
    res = _fast_pair(ctx, vs, vps, layer.num_blocks, calls)
    trunc = F32(ocfg.default_truncation_distance)
    n_single = n_multi = 0
    pk = np.zeros(0, np.int64); pw = np.zeros(0, F32); pc = np.zeros(0, np.uint32)   # state before the call
    for (T, pts, rgba), (g, s, u, r), (idx, d, w, words, (kplain, dplain)) in zip(calls, traces, res):
        keys = tx.voxel_keys(g)
        ray = cx.pack(rgba)[r]
        k_all, d_all, w_all = tx.layer_voxels(idx, d, w, vps)
        c_all = cx.layer_colours(idx, words, vps)[1]
        prev_w = np.zeros(len(k_all), F32); prev_c = np.zeros(len(k_all), np.uint32)
        if len(pk):
            pos = np.searchsorted(k_all, pk)
            prev_w[pos] = pw; prev_c[pos] = pc
        o = np.argsort(keys, kind="stable")
        ks, ss, us, rws = keys[o], s[o], u[o], ray[o]
        uniq, start, cnt = np.unique(ks, return_index=True, return_counts=True)
        at = np.searchsorted(k_all, uniq)
        assert np.array_equal(k_all[at], uniq)
        # untouched voxels keep their colour
        untouched = np.ones(len(k_all), bool); untouched[at] = False
        assert np.array_equal(c_all[untouched], prev_c[untouched])
        # (a) one update in the call: the exact rule; where the voxel was new, also the colourless run's distance
        one = cnt == 1
        j = start[one]
        exp = cx.colour_step(trunc, ss[j], us[j], prev_w[at[one]], rws[j], prev_c[at[one]])
        assert np.array_equal(c_all[at[one]], exp)
        new = at[one & (prev_w[at] == 0)]
        assert np.array_equal(d_all[new].view(np.uint32), dplain[np.searchsorted(kplain, k_all[new])].view(np.uint32))
        n_single += int(np.count_nonzero(one & (np.abs(ss[start]) < trunc)))
        # (b) several updates: channel-wise within the previous colour and the band rays' colours
        band = np.abs(ss) < trunc
        lo = cx.unpack(prev_c[at]).astype(np.int64); hi = lo.copy()
        ch = cx.unpack(rws).astype(np.int64)
        seg = np.repeat(np.arange(len(uniq)), cnt)
        for c4 in range(4):
            np.minimum.at(lo[:, c4], seg[band], ch[band, c4])
            np.maximum.at(hi[:, c4], seg[band], ch[band, c4])
        got = cx.unpack(c_all[at]).astype(np.int64)
        assert ((got >= lo) & (got <= hi)).all()
        has_band = np.zeros(len(uniq), bool); has_band[seg[band]] = True
        assert np.array_equal(c_all[at[~has_band]], prev_c[at[~has_band]])
        n_multi += int(np.count_nonzero(has_band & ~one))
        pk, pw, pc = k_all, w_all, c_all
    assert n_single > 50 and n_multi > 50


def test_mode1_one_colour_is_exact(ctx, oracle, world):
    """Every ray one colour c into an empty submap.  A voxel all of whose updates lie in the band holds exactly c
    in any order (the first sets c, equal colours blend to c).  One that also collects updates outside the band
    (rays passing in front of it raise its weight while it is still black) lies between black and c, as it would
    after a sequential run; a voxel without a band update stays 0."""
    vs, vps = 0.2, 16
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=8, n_azimuth=64, seed=1, miss_range=40.0)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    c = np.array([201, 17, 96, 254], np.uint8)
    ocfg = oracle.tsdf_config(**tx.FAST_ALL)
    layer = oracle.Layer(vs, vps)
    _, g, s, u, r = cx.trace_rays(oracle, layer, ocfg, T, pts)
    (idx, d, w, words, _), = _fast_pair(ctx, vs, vps, layer.num_blocks, [(T, pts, np.tile(c, (len(pts), 1)))])
    k_all, c_all = cx.layer_colours(idx, words, vps)
    keys = tx.voxel_keys(g)
    in_band = np.abs(s) < F32(ocfg.default_truncation_distance)
    band = np.unique(keys[in_band])
    pure = np.setdiff1d(band, np.unique(keys[~in_band]))
    mixed = np.setdiff1d(band, pure)
    assert len(pure) > 200 and len(mixed) > 20
    assert (c_all[np.searchsorted(k_all, pure)] == cx.pack(c[None])[0]).all()
    assert (cx.unpack(c_all[np.searchsorted(k_all, mixed)]) <= c).all()
    rest = np.ones(len(k_all), bool); rest[np.searchsorted(k_all, band)] = False
    assert not c_all[rest].any()


def test_colour_upload_download_and_device_pair(ctx):
    """Host and device-to-device attachment of a channel to an uploaded submap; a submap without one downloads
    zeros, peeks NULL and saves exactly as its colour-free twin."""
    vs, vps, n = 0.2, 8, 3
    rs = np.random.RandomState(5)
    idx = np.array([[0, 0, 0], [-1, 2, 0], [3, -2, 1]], np.int32)
    d = rs.uniform(-0.6, 0.6, (n, vps ** 3)).astype(F32); w = rs.uniform(0, 9, (n, vps ** 3)).astype(F32)
    words = rs.randint(0, 2 ** 32, (n, vps ** 3), dtype=np.uint64).astype(np.uint32)
    a, b, twin = next(_ids), next(_ids), next(_ids)
    try:
        for sid in (a, b, twin):
            ctx.submap_upload(sid, vs, vps, idx, d, w)
        assert not ctx.submap_has_colour(a) and ctx.submap_peek_device_colour(a) is None
        assert not ctx.submap_download_colour(a).any()
        ctx.submap_upload_colour(a, words)
        assert ctx.submap_has_colour(a) and np.array_equal(ctx.submap_download_colour(a), words)
        with pytest.raises(api.VgxError) as e:
            ctx.submap_upload_colour(a, words[:2])
        assert e.value.code == _lib.VGX_ERR_INVALID and np.array_equal(ctx.submap_download_colour(a), words)
        ctx.submap_upload_device_colour(b, n, ctx.submap_peek_device_colour(a))
        assert np.array_equal(ctx.submap_download_colour(b), words)
        tx.assert_layers_bit_equal(ctx.submap_download(a), ctx.submap_download(b))
        # the colourless twin: the bytes a save always produced; the coloured one differs only in colour words
        T = np.array([[1, 0, 0, 0, 0, 0, 0]], F32)
        plain = ctx.collection_save([twin], T)
        assert not ctx.submap_has_colour(twin)
        ctx.submap_upload_colour(twin, np.zeros_like(words))      # an all-zero channel writes the same file
        assert ctx.collection_save([twin], T) == plain
        assert len(ctx.collection_save([a], T)) > len(plain)
        with pytest.raises(api.VgxError):
            ctx.submap_has_colour(next(_ids))
    finally:
        for sid in (a, b, twin):
            ctx.submap_free(sid)


def test_collection_fixture_keeps_colour():
    """The coloured fixture: with keep_colour it saves back byte for byte (it is written unpacked, as the
    library writes); without, it is the colour-free stream as before.  A stream without colours gets no channel
    under the flag either."""
    data = cs.read("colour")
    entries = api.Context.collection_scan(data)
    ids = [e["id"] for e in entries]
    T = np.array([e["T_M_S"] for e in entries])
    c = api.Context(0)
    try:
        before = c.launch_count
        assert c.collection_load(data, keep_colour=True) == len(ids)
        kept_launches = c.launch_count - before
        assert all(c.submap_has_colour(i) for i in ids)
        assert bytes(c.collection_save(ids, T)) == data
        for i in ids:
            c.submap_free(i)
        before = c.launch_count
        assert c.collection_load(data) == len(ids)
        assert c.launch_count - before == kept_launches
        assert not any(c.submap_has_colour(i) for i in ids)
        assert bytes(c.collection_save(ids, T)) == cs.read("unpacked")
        for i in ids:
            c.submap_free(i)
        assert c.collection_load(cs.read("packed"), keep_colour=True) == len(ids)
        assert not any(c.submap_has_colour(i) for i in ids)
        assert bytes(c.collection_save(ids, T)) == cs.read("unpacked")
        assert c._L.vgx_collection_load_ex(c._h, data, len(data), 2, None) == _lib.VGX_ERR_INVALID
    finally:
        c.close()


def test_coloured_map_survives_save_and_load(world, tmp_path):
    """A mapper fed a coloured stream (Fast integration, three submaps, the last one active): saveToFile, then
    load_submap_collection(keep_colour=True) in a fresh context reproduces every brick and every colour word."""
    from voxgraph_b200.mapper import MapperConfig, VoxgraphMapper
    c = api.Context(0)
    c2 = api.Context(0)
    try:
        m = VoxgraphMapper(c, MapperConfig(voxel_size=0.2, capacity_blocks=4096, submap_creation_interval=2.0,
                                           registration_constraints_enabled=False))
        rs = np.random.RandomState(9)
        for k in range(6):
            pose = np.array([12.0 + 1.5 * k, 15.0, 1.2, 0.2 * k])
            pts = synth.lidar_scan(world, pose, n_beams=8, n_azimuth=128, seed=k)
            col = rs.randint(0, 256, (len(pts), 4)).astype(np.uint8)
            m.pointcloudCallback(float(k), pose, pts, colours=col if k != 3 else None)
        assert len(m.submap_ids) == 3 and all(c.submap_has_colour(i) for i in m.submap_ids)
        path = str(tmp_path / "coloured.bin")
        m.saveToFile(path)
        ids, _ = api.load_submap_collection(c2, path, keep_colour=True)
        assert ids.tolist() == m.submap_ids
        for i in m.submap_ids:
            want = c.submap_download(i)
            tx.assert_layers_bit_equal(want, c2.submap_download(i))
            assert np.array_equal(want[0], c2.submap_download(i)[0])        # block order is the file's order
            words = c.submap_download_colour(i)
            assert words.any() and np.array_equal(words, c2.submap_download_colour(i))
    finally:
        c.close()
        c2.close()
