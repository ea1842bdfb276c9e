"""Point-cloud messages on the device against the exact model tests/cloud_exact.py: the decoder over the layout
matrix, vgx_tsdf_integrate_cloud and vgx_tsdf_integrate_device against vgx_tsdf_integrate fed with the model's
points and colours (mode 0 bit for bit, mode 1 under the contract of two Fast runs of one scan), launch counts,
the validation rules and the mapper's message callback.  Every property is checked once per case."""
import ctypes as C
import itertools

import numpy as np
import pytest

import cloud_exact as ce
import colour_exact as cx
import tsdf_exact as tx
from support import IDENTITY, ctx, world  # noqa: F401
from voxgraph_b200 import _lib, api, mapper as vm, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
F = api.POINTFIELD_FLOAT32
_ids = itertools.count(9000)
LAYOUTS = ["xyz16", "xyzi32", "xyzi16", "xyzrgb32", "odd19", "organised"]


def _records(n, step, parts):
    """n records of `step` bytes filled with 0xA5, then parts [(offset, (n, k) uint8)] -> (n, step) uint8."""
    rec = np.full((n, step), 0xA5, np.uint8)
    for off, b in parts:
        rec[:, off:off + b.shape[1]] = b
    return rec


def _f32_bytes(a):
    return np.ascontiguousarray(a, F32).reshape(-1, 1).view(np.uint8)


def make_cloud(layout, pts, rgba, inten):
    """The points as a message in one of the layouts of the matrix."""
    n = len(pts)
    if layout == "xyz16":
        return synth.pack_pointcloud2(pts)
    if layout == "xyzi32":
        return synth.pack_pointcloud2(pts, intensity=inten)
    if layout == "xyzrgb32":
        return synth.pack_pointcloud2(pts, rgba=rgba)
    if layout == "organised":                 # 48 rows of 64 XYZRGB records, 24 bytes of padding after each row
        return synth.pack_pointcloud2(pts, rgba=rgba, organised=(n // 64, 64), pad_rows=24)
    if layout == "xyzi16":                    # x y z intensity packed into 16 bytes
        rec = _records(n, 16, [(0, pts.view(np.uint8).reshape(n, 12)), (12, _f32_bytes(inten))])
        fields = [("x", 0, F, 1), ("y", 4, F, 1), ("z", 8, F, 1), ("intensity", 12, F, 1)]
    else:                                     # 19 bytes, nothing 4-byte aligned: z at 1, rgb at 5, x at 9, y at 14
        assert layout == "odd19"
        rec = _records(n, 19, [(1, _f32_bytes(pts[:, 2])), (5, rgba[:, [2, 1, 0, 3]]), (9, _f32_bytes(pts[:, 0])),
                               (14, _f32_bytes(pts[:, 1]))])
        fields = [("z", 1, F, 1), ("rgb", 5, api.POINTFIELD_UINT32, 1), ("x", 9, F, 1), ("y", 14, F, 1)]
    step = rec.shape[1]
    return api.PointCloud2(fields=fields, width=n, height=1, point_step=step, row_step=n * step, data=rec.tobytes())


def spoil(pts, share, seed):
    """A copy with `share` of the records given a NaN, +Inf or -Inf in a random coordinate."""
    rs = np.random.RandomState(seed)
    out = np.array(pts, F32)
    bad = np.nonzero(rs.uniform(size=len(out)) < share)[0]
    out[bad, rs.randint(0, 3, len(bad))] = np.array([np.nan, np.inf, -np.inf], F32)[rs.randint(0, 3, len(bad))]
    return out


def attributes(n, seed):
    """Colours whose four channels differ, and intensities that cover the clamp's ends and NaN."""
    rs = np.random.RandomState(seed)
    rgba = rs.randint(0, 256, (n, 4)).astype(np.uint8)
    inten = rs.uniform(-500.0, 12000.0, n).astype(F32)
    inten[rs.uniform(size=n) < 0.02] = np.nan
    return rgba, inten


# ------------------------------------------------------------------ 1. the decoder
@pytest.mark.parametrize("bad", ["none", "scattered", "all", "empty"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_decode_bit_exact(ctx, layout, bad):
    n = 0 if bad == "empty" else (48 * 64 if layout == "organised" else 3001)
    pts = np.random.RandomState(1).normal(0, 5, (n, 3)).astype(F32)
    pts = {"none": pts, "empty": pts, "scattered": spoil(pts, 0.07, 2), "all": spoil(pts, 2.0, 3)}[bad]
    rgba, inten = attributes(n, 4)
    msg = make_cloud(layout, pts, rgba, inten)
    exp_p, exp_c = ce.convert_msg(msg, api.cloud_layout(msg))
    assert len(exp_p) == {"none": n, "empty": 0, "all": 0}.get(bad, len(exp_p))
    if bad == "scattered":
        assert 0.88 * n < len(exp_p) < 0.97 * n
    got_p, got_c = ctx.cloud_decode(msg)
    assert got_p.shape == exp_p.shape and np.array_equal(got_p.view(np.uint32), exp_p.view(np.uint32))
    assert np.array_equal(got_c, exp_c)


# ------------------------------------------------------------------ 2, 3. decode + integrate
def _stats(s):
    return (s.rays_valid, s.rays_cast, s.voxel_updates, s.blocks_allocated, s.saturated_batches)


def _message_scans(world, layout):
    """Three overlapping scans (two with clearing rays) with 7 % of the records spoiled -> [(T, message)]."""
    out = []
    for k, (T, pts) in enumerate(tx.scans(world, 16, 256)):
        rgba, inten = attributes(len(pts), 10 + k)
        out.append((T, make_cloud(layout, spoil(pts, 0.07, 20 + k), rgba, inten)))
    return out


def _feed_pair(ctx, scans, cfg, colours, capacity=4096):
    """The messages into one submap through tsdf_integrate_cloud and, as the model's points and colours, into a
    second one through tsdf_integrate -> the two downloads (layer, colour words, has_colour) after checking the
    statistics and the point counts call by call."""
    a, b = next(_ids), next(_ids)
    try:
        for sid in (a, b):
            ctx.submap_create(sid, 0.2, 16, capacity)
        for (T, msg) in scans:
            p, c = ce.convert_msg(msg, api.cloud_layout(msg))
            sa, n_points = ctx.tsdf_integrate_cloud(a, T, msg, cfg, colours=colours)
            sb = ctx.tsdf_integrate(b, T, p, cfg, rgba=c if colours else None)
            assert n_points == len(p) < msg.width * msg.height
            assert _stats(sa)[:4] == _stats(sb)[:4] and sa.voxel_updates > 10000
            if cfg.mode == 0:
                assert sa.saturated_batches == sb.saturated_batches
        return [(ctx.submap_download(sid), ctx.submap_download_colour(sid), ctx.submap_has_colour(sid)) for sid in (a, b)]
    finally:
        for sid in (a, b):
            ctx.submap_free(sid)


@pytest.mark.parametrize("colours", [True, False], ids=["colours", "plain"])
@pytest.mark.parametrize("layout", ["xyz16", "xyzi32", "xyzrgb32"])
def test_integrate_cloud_mode0_bit_exact(ctx, world, layout, colours):
    (la, ca, ha), (lb, cb, hb) = _feed_pair(ctx, _message_scans(world, layout), ctx.tsdf_config(mode=0), colours)
    tx.assert_layers_bit_equal(lb, la)
    assert ha == hb == colours
    ka, wa = cx.layer_colours(la[0], ca, 16)
    kb, wb = cx.layer_colours(lb[0], cb, 16)
    assert np.array_equal(ka, kb) and np.array_equal(wa, wb)
    assert (np.count_nonzero(wa) > 1000) == colours


@pytest.mark.parametrize("layout", ["xyz16", "xyzi32", "xyzrgb32"])
def test_integrate_cloud_mode1_contract(ctx, world, layout):
    """What two Fast runs of one scan share: statistics, the block set, the (integer, order-free) weights, and the
    distance of every voxel with a single update (the others depend on the order of the updates)."""
    scans = _message_scans(world, layout)[:1]
    (la, ca, ha), (lb, cb, hb) = _feed_pair(ctx, scans, ctx.tsdf_config(**tx.FAST_ALL), True)
    ka, da, wa = tx.layer_voxels(*la, 16)
    kb, db, wb = tx.layer_voxels(*lb, 16)
    assert np.array_equal(ka, kb) and np.array_equal(wa.view(np.uint32), wb.view(np.uint32))
    single = wa == 1.0                       # constant weight 1, no drop-off: one update outside the band
    assert np.count_nonzero(single) > 1000
    assert np.array_equal(da[single].view(np.uint32), db[single].view(np.uint32))
    assert ha and hb
    # colours: a voxel no ray updated keeps 0; an XYZ cloud's opaque black can only raise the alpha byte
    ga, gb = cx.layer_colours(la[0], ca, 16)[1], cx.layer_colours(lb[0], cb, 16)[1]
    assert not ga[wa == 0].any() and not gb[wb == 0].any() and ga.any() and gb.any()
    if layout == "xyz16":
        assert not ((ga | gb) & 0xffffff00).any()


# ------------------------------------------------------------------ 4. points already on the device
def test_integrate_device_matches_host(ctx, world):
    import torch
    cfg = ctx.tsdf_config(mode=0)
    dev = torch.device("cuda", ctx.device)
    a, b = next(_ids), next(_ids)
    try:
        for sid in (a, b):
            ctx.submap_create(sid, 0.2, 16, 4096)
        for k, (T, pts) in enumerate(tx.scans(world, 16, 256)):
            pts = spoil(pts, 0.03, k)
            rgba = attributes(len(pts), k)[0]
            d_pts = torch.from_numpy(pts).to(dev)
            d_col = torch.from_numpy(rgba).to(dev)
            torch.cuda.synchronize()
            # the colours as (n, 4) bytes, or as the (n,) words of those bytes
            sa = ctx.tsdf_integrate_device(a, T, d_pts, cfg, d_rgba=d_col if k != 1 else d_col.view(torch.uint32).view(-1))
            sb = ctx.tsdf_integrate(b, T, pts, cfg, rgba=rgba)
            assert _stats(sa) == _stats(sb)
        tx.assert_layers_bit_equal(ctx.submap_download(b), ctx.submap_download(a))
        assert np.array_equal(cx.layer_colours(ctx.submap_download(a)[0], ctx.submap_download_colour(a), 16)[1],
                              cx.layer_colours(ctx.submap_download(b)[0], ctx.submap_download_colour(b), 16)[1])
        before = ctx.submap_download(a)
        good = torch.zeros((8, 3), dtype=torch.float32, device=dev)
        with pytest.raises(TypeError):
            ctx.tsdf_integrate_device(a, IDENTITY, good.cpu(), cfg)                      # host memory
        with pytest.raises(TypeError):
            ctx.tsdf_integrate_device(a, IDENTITY, good.double(), cfg)                   # dtype
        with pytest.raises(ValueError):
            ctx.tsdf_integrate_device(a, IDENTITY, torch.zeros((8, 6), device=dev)[:, ::2], cfg)   # strided
        with pytest.raises(ValueError):
            ctx.tsdf_integrate_device(a, IDENTITY, torch.zeros((8, 4), device=dev), cfg)            # shape
        with pytest.raises(ValueError):
            ctx.tsdf_integrate_device(a, IDENTITY, good, cfg, d_rgba=torch.zeros((7, 4), dtype=torch.uint8, device=dev))
        wrong = api.Context.__new__(api.Context)          # the device check needs no second GPU: a context object
        wrong.device = ctx.device + 1                     # that claims another device
        with pytest.raises(ValueError):
            api.Context.tsdf_integrate_device(wrong, a, IDENTITY, good, cfg)
        tx.assert_layers_bit_equal(before, ctx.submap_download(a))
        # the C-ABI itself refuses host memory
        host = np.zeros((8, 3), F32)
        rc = ctx._L.vgx_tsdf_integrate_device(ctx._h, a, IDENTITY.ctypes.data_as(C.POINTER(C.c_float)), 8,
                                              C.c_void_p(host.ctypes.data), None, C.byref(cfg), None)
        assert rc == _lib.VGX_ERR_INVALID
    finally:
        for sid in (a, b):
            ctx.submap_free(sid)


# ------------------------------------------------------------------ 5. launches
@pytest.mark.parametrize("mode", [0, 1])
def test_one_extra_launch_whatever_the_size(ctx, world, mode):
    cfg = ctx.tsdf_config(mode=mode)
    extra = []
    for (beams, azimuth) in [(8, 256), (300, 1024)]:
        pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=beams, n_azimuth=azimuth, seed=1,
                               miss_range=40.0)
        assert len(pts) == beams * azimuth
        rgba = attributes(len(pts), 1)[0]
        msg = synth.pack_pointcloud2(pts, rgba=rgba)
        a, b = next(_ids), next(_ids)
        try:
            for sid in (a, b):
                ctx.submap_create(sid, 0.2, 16, 8192)
            l0 = ctx.launch_count
            ctx.tsdf_integrate_cloud(a, IDENTITY, msg, cfg)
            l1 = ctx.launch_count
            ctx.tsdf_integrate(b, IDENTITY, pts, cfg, rgba=rgba)
            l2 = ctx.launch_count
            extra.append((l1 - l0) - (l2 - l1))
        finally:
            for sid in (a, b):
                ctx.submap_free(sid)
    assert extra == [1, 1]


# ------------------------------------------------------------------ 6. validation
def _bad_messages():
    pts = np.random.RandomState(0).normal(0, 3, (64, 3)).astype(F32)
    rgba, inten = attributes(64, 0)
    base = lambda: synth.pack_pointcloud2(pts, rgba=rgba)
    out = {}
    for name, field, off in [("x-beyond", 0, 29), ("z-beyond", 2, 30), ("rgb-beyond", 3, 31)]:
        m = base(); f = list(m.fields[field]); f[1] = off; m.fields[field] = tuple(f); out[name] = m
    m = base(); m.point_step = 0; out["point-step-0"] = m
    m = base(); m.row_step = 64 * 32 - 1; out["row-step-short"] = m
    m = base(); m.data = m.data[:-1]; out["data-short"] = m
    m = base(); m.height = 2; out["data-short-rows"] = m
    m = base(); m.width = 1 << 20; m.height = 1 << 12; m.row_step = 32 << 20; out["too-many-records"] = m
    m = synth.pack_pointcloud2(pts, intensity=inten); f = list(m.fields[3]); f[1] = 30; m.fields[3] = tuple(f)
    out["intensity-beyond"] = m
    return out


BAD = _bad_messages()


@pytest.mark.parametrize("name", sorted(BAD))
def test_validation_leaves_the_submap_alone(ctx, world, name):
    cfg = ctx.tsdf_config(mode=0)
    sid = next(_ids)
    T, pts = tx.scans(world, 8, 128)[0]
    try:
        ctx.submap_create(sid, 0.2, 16, 4096)
        ctx.tsdf_integrate(sid, T, pts, cfg)
        before = ctx.submap_download(sid)
        with pytest.raises(api.VgxError) as e:
            ctx.tsdf_integrate_cloud(sid, T, BAD[name], cfg)
        assert e.value.code == _lib.VGX_ERR_INVALID
        with pytest.raises(api.VgxError) as e:
            ctx.cloud_decode(BAD[name])
        assert e.value.code == _lib.VGX_ERR_INVALID
        tx.assert_layers_bit_equal(before, ctx.submap_download(sid))
        assert not ctx.submap_has_colour(sid)
    finally:
        ctx.submap_free(sid)


def test_submap_errors_and_empty_cloud(ctx):
    msg = synth.pack_pointcloud2(np.ones((4, 3), F32))
    with pytest.raises(api.VgxError) as e:
        ctx.tsdf_integrate_cloud(next(_ids), IDENTITY, msg)
    assert e.value.code == _lib.VGX_ERR_NOT_FOUND
    sid = next(_ids)
    try:
        ctx.submap_create(sid, 0.2, 16, 64)
        with pytest.raises(api.VgxError) as e:
            ctx.tsdf_integrate_cloud(sid, IDENTITY, msg, colour_map_max=0.0)
        assert e.value.code == _lib.VGX_ERR_INVALID
        st, n = ctx.tsdf_integrate_cloud(sid, IDENTITY, synth.pack_pointcloud2(np.zeros((0, 3), F32)))
        assert _stats(st) == (0, 0, 0, 0, 0) and n == 0 and not ctx.submap_has_colour(sid)
        ctx.submap_finish(sid)
        with pytest.raises(api.VgxError) as e:
            ctx.tsdf_integrate_cloud(sid, IDENTITY, msg)
        assert e.value.code == _lib.VGX_ERR_INVALID
    finally:
        ctx.submap_free(sid)


# ------------------------------------------------------------------ 7. the mapper's message callback
def test_mapper_message_callback_matches_array_callback(world):
    n = 12
    s_arc = np.linspace(0.0, 9.0, n)
    gt = np.stack([8.0 + s_arc, 12.0 + 0.5 * np.sin(s_arc / 3.0), np.full(n, 1.2), 0.05 * s_arc], -1)
    odo = gt + np.cumsum(np.random.default_rng(0).normal(0, 1.0, (n, 4)) * np.array([0.02, 0.02, 0.001, 0.002]), 0)
    big = synth.make_world(7, size_xy=(40.0, 30.0), n_clutter=60, n_walls=5)
    msgs = []
    for k in range(n):
        pts = synth.lidar_scan(big, gt[k], n_beams=24, n_azimuth=360, seed=k, max_range=12.0)
        rgba = synth.surface_colours(pts, gt[k])
        msgs.append(synth.pack_pointcloud2(spoil(pts, 0.05, 40 + k), rgba=rgba))
    cfg = vm.MapperConfig(voxel_size=0.2, submap_creation_interval=4 / 10.0, capacity_blocks=4096,
                          tsdf=dict(max_ray_length_m=12.0, mode=0))
    runs = []
    for use_message in (True, False):
        c = api.Context(0)
        m = vm.VoxgraphMapper(c, cfg)
        for k, msg in enumerate(msgs):
            if use_message:
                m.pointcloudMessageCallback(k / 10.0, odo[k], msg)
            else:
                p, col = ce.convert_msg(msg, api.cloud_layout(msg))
                m.pointcloudCallback(k / 10.0, odo[k], p, col)
        layers = [(c.submap_download(i), c.submap_download_colour(i)) for i in m.submap_ids]
        runs.append((m, layers))
        c.close()
    (ma, la), (mb, lb) = runs
    assert ma.submap_ids == mb.submap_ids and len(ma.submap_ids) == 3
    assert ma.scan_points == [len(ce.convert_msg(g, api.cloud_layout(g))[0]) for g in msgs]
    assert [_stats(s)[:4] for s in ma.scan_stats] == [_stats(s)[:4] for s in mb.scan_stats]
    assert ma.overlapping_submap_list == mb.overlapping_submap_list and len(ma.overlapping_submap_list) >= 1
    for (xa, ca), (xb, cb) in zip(la, lb):
        tx.assert_layers_bit_equal(xb, xa)
        assert np.array_equal(cx.layer_colours(xa[0], ca, 16)[1], cx.layer_colours(xb[0], cb, 16)[1]) and ca.any()
    # The solves start from bit-identical submaps, pairs and odometry, but their end poses are not reproducible to
    # the bit: blocks are allocated by atomics, so the order of the registration points and of their sums differs
    # from run to run, and Levenberg-Marquardt stops at a parameter tolerance of 3e-3.  Between the two runs of this
    # test the poses were seen to differ by up to 1.3e-2 m; the bound says they describe the same map.
    for i in ma.submap_ids:
        assert np.allclose(ma.submap_pose[i], mb.submap_pose[i], rtol=0, atol=5e-2)
