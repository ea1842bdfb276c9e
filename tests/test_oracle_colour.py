"""Voxel colour on the CPU: known answers of the restated voxblox rules (tests/colour_exact.py, the models
the GPU tests compare the kernels with), and the new C-ABI exports."""
import ctypes as C

import numpy as np

import colour_exact as cx
import tsdf_exact as tx
from voxgraph_b200 import synth

F32 = np.float32


def _w(r, g, b, a):
    return cx.pack([[r, g, b, a]])[0]


def test_word_layout():
    """Four distinct channels: the stored word is a | b << 8 | g << 16 | r << 24, and unpack inverts pack."""
    assert _w(0x11, 0x22, 0x33, 0x44) == 0x11223344
    rgba = np.array([[1, 2, 3, 4], [255, 0, 128, 7]], np.uint8)
    assert np.array_equal(cx.unpack(cx.pack(rgba)), rgba)


def test_blend_known_answers():
    c1, c2 = _w(10, 200, 33, 255), _w(250, 0, 34, 0)
    # w1 = 0 gives c2 exactly, whatever w2
    for w2 in (1.0, 20.0, 1e-3, 0.3):
        assert cx.blend(c1, F32(0), c2, F32(w2)) == c2
    # equal colours stay, for weights whose normalised sum is not exactly 1
    for w1, w2 in ((1.0, 20.0), (3.0, 7.0), (0.1, 0.7), (1e4, 1.0)):
        assert cx.blend(c1, F32(w1), c1, F32(w2)) == c1
    # halves round away from zero on every channel, alpha included: (1 + 2) / 2 = 1.5 -> 2, (2 + 5) / 2 = 3.5 -> 4
    assert cx.blend(_w(1, 2, 0, 255), F32(1), _w(2, 5, 1, 0), F32(1)) == _w(2, 4, 1, 128)
    # just below and just above a half: 0.25 * 1 + 0.75 * 3 = 2.5 -> 3; 0.75 * 1 + 0.25 * 2 = 1.25 -> 1
    assert cx.blend(_w(1, 1, 0, 0), F32(1), _w(3, 3, 0, 0), F32(3)) == _w(3, 3, 0, 0)
    assert cx.blend(_w(1, 1, 0, 0), F32(3), _w(2, 2, 0, 0), F32(1)) == _w(1, 1, 0, 0)
    # four distinct channels, each blended on its own: weights 1 : 3
    assert cx.blend(_w(0, 100, 200, 40), F32(1), _w(100, 0, 100, 240), F32(3)) == _w(75, 25, 125, 190)
    # every channel stays inside the range of its two inputs over random weights
    rs = np.random.RandomState(0)
    a = rs.randint(0, 256, (2000, 4)).astype(np.uint8); b = rs.randint(0, 256, (2000, 4)).astype(np.uint8)
    w1 = rs.uniform(0, 1e4, 2000).astype(F32); w2 = rs.uniform(1e-3, 20, 2000).astype(F32)
    out = cx.unpack(cx.blend(cx.pack(a), w1, cx.pack(b), w2))
    assert (out >= np.minimum(a, b)).all() and (out <= np.maximum(a, b)).all()


def test_colour_rule_band_and_early_out():
    trunc = F32(0.6)
    old, ray = _w(10, 20, 30, 40), _w(200, 100, 50, 255)
    one = lambda sdf, uw, vw: cx.colour_step(trunc, np.array([sdf], F32), np.array([uw], F32), np.array([vw], F32),
                                             np.array([ray], np.uint32), np.array([old], np.uint32))[0]
    assert one(0.0, 1.0, 0.0) == ray                          # first update in the band: the ray's colour
    assert one(0.3, 1.0, 1.0) == _w(105, 60, 40, 148)         # equal weights: the rounded mean
    assert one(-0.3, 1.0, 3.0) == cx.blend(old, F32(3), ray, F32(1))
    assert one(0.6, 1.0, 1.0) == old                          # |sdf| = trunc is outside the band
    assert one(-0.6, 1.0, 1.0) == old
    assert one(np.nextafter(F32(0.6), F32(0)), 1.0, 1.0) != old
    assert one(2.0, 1.0, 1.0) == old                          # free space in front of the surface
    assert one(np.nan, 1.0, 1.0) == old                       # a point at the sensor origin
    assert one(0.1, 0.0, 0.0) == old                          # new_weight < 1e-6: the voxel is left untouched
    assert one(0.1, 5e-7, 4e-7) == old
    assert one(0.1, 6e-7, 5e-7) != old


def test_replay_matches_oracle_distance_and_weight(oracle):
    """The coloured sequential replay built on the per-ray trace reproduces the oracle's (distance, weight) bit
    for bit, and colours exactly the voxels that received a band update.  The clearing rays here (points at
    40 m, cut at max_ray_length_m = 16 m) end far in front of anything and colour nothing; a clearing point
    within a truncation distance of the limit does reach the band (test_clearing_rays_reach_the_band)."""
    world = synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=8, n_azimuth=64, seed=1, miss_range=40.0)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    cfg = oracle.tsdf_config()
    rs = np.random.RandomState(1)
    rgba = rs.randint(1, 256, (len(pts), 4)).astype(np.uint8)
    ref = oracle.Layer(0.2, 16)
    oracle.tsdf_integrate(ref, cfg, T, pts)
    layer = oracle.Layer(0.2, 16)
    st = cx.State()
    for _ in range(2):
        _, g, s, u, r = cx.trace_rays(oracle, layer, cfg, T, pts)
        k, d, w, c = cx.replay(tx.voxel_keys(g), s, u, cx.pack(rgba)[r], cfg.default_truncation_distance,
                               cfg.max_weight, st)
    oracle.tsdf_integrate(ref, cfg, T, pts)
    tx.assert_layers_bit_equal(ref.export(), layer.export())
    ek, ed, ew = tx.layer_voxels(*ref.export(), 16)
    pos = np.searchsorted(ek, st.keys)
    assert np.array_equal(ed[pos].view(np.uint32), st.d.view(np.uint32))
    assert np.array_equal(ew[pos].view(np.uint32), st.w.view(np.uint32))
    keys = tx.voxel_keys(g)
    band = np.unique(keys[np.abs(s) < F32(cfg.default_truncation_distance)])
    assert len(band) > 100 and np.array_equal(st.keys[st.c != 0], band)
    clearing = np.linalg.norm(pts, axis=1) > cfg.max_ray_length_m
    assert clearing.any() and not np.isin(keys[clearing[r]], band).any()


def test_clearing_rays_reach_the_band(oracle):
    """A clearing ray (norm > max_ray_length_m) ends at norm - trunc, so its last voxel's centre can lie
    further along the ray, less than trunc in front of the point: an update inside the band, which the colour
    rule blends.  400 points at 8 m + U(0.001, trunc + one voxel) with max_ray_length_m = 8: every one is a
    clearing ray, and a hundred or more of them reach the band, with sdf > 0 (in front of the point)."""
    T = synth.pose_to_T([0.1, 0.1, 0.1, 0.3])
    cfg = oracle.tsdf_config(max_ray_length_m=8.0)
    trunc = F32(cfg.default_truncation_distance)
    for vs in (0.2, 0.1, 0.05):
        rs = np.random.RandomState(0)
        d = rs.normal(size=(400, 3))
        d /= np.linalg.norm(d, axis=1)[:, None]
        pts = (d * (8.0 + rs.uniform(0.001, float(trunc) + vs, 400))[:, None]).astype(F32)
        assert (np.linalg.norm(pts.astype(np.float64), axis=1) > 8.0).all()
        _, g, s, u, r = cx.trace_rays(oracle, oracle.Layer(vs, 8), cfg, T, pts)
        band = np.abs(s) < trunc
        assert len(np.unique(r[band])) > 100, vs
        assert (s[band] > 0).all() and (u[band] > 0).all()
        # and the replay colours those voxels with the clearing rays' colours
        st = cx.State()
        words = cx.pack(np.full((400, 4), [10, 20, 30, 40], np.uint8))
        cx.replay(tx.voxel_keys(g), s, u, words[r], trunc, cfg.max_weight, st)
        assert np.array_equal(st.keys[st.c != 0], np.unique(tx.voxel_keys(g[band])))


def test_merge_known_answers():
    cA, cB = _w(200, 100, 50, 255), _w(10, 20, 30, 40)
    c, w = cx.merge(cA, F32(1), cB, F32(1))
    assert c == _w(105, 60, 40, 148) and w == 2                      # colourA first, as mergeVoxelAIntoVoxelB calls it
    c, w = cx.merge(cA, F32(0), cB, F32(3))
    assert c == cB and w == 3                                         # a (0, 0) voxel merges to nothing
    c, w = cx.merge(cA, F32(0), cB, F32(0))
    assert c == cB and w == 0                                         # w = 0: untouched
    c, w = cx.merge(0, F32(2), cB, F32(2))
    assert c == _w(5, 10, 15, 20) and w == 4                          # a colourless input counts as black


def test_interpolation_truncates():
    words = [_w(10, 0, 255, 7)] * 8
    assert cx.interp_channels(words, [0.3, 0.6, 0.9]) == _w(10, 0, 255, 7)
    # along x only (neighbour 4 = +x): 10 + 0.75 * (13 - 10) = 12.25 -> 12; 0.25 -> 10.75 -> 10, not 11
    words = [_w(10, 0, 0, 0)] * 4 + [_w(13, 0, 0, 0)] * 4
    assert cx.interp_channels(words, [0.75, 0.0, 0.0]) == _w(12, 0, 0, 0)
    assert cx.interp_channels(words, [0.25, 0.0, 0.0]) == _w(10, 0, 0, 0)
    # 0.999 of the way from 0 to 255 is 254.745: truncation gives 254 where round would give 255
    words = [_w(0, 0, 0, 0)] * 4 + [_w(255, 255, 255, 255)] * 4
    assert cx.interp_channels(words, [0.999, 0.0, 0.0]) == _w(254, 254, 254, 254)
    # per channel, each on its own axis
    words = [_w(0, 0, 0, 0)] * 8
    words[4] = _w(100, 0, 0, 0); words[2] = _w(0, 100, 0, 0); words[1] = _w(0, 0, 100, 0)
    assert cx.interp_channels(words, [0.5, 0.0, 0.0]) == _w(50, 0, 0, 0)
    assert cx.interp_channels(words, [0.0, 0.5, 0.0]) == _w(0, 50, 0, 0)
    assert cx.interp_channels(words, [0.0, 0.0, 0.5]) == _w(0, 0, 50, 0)


def test_containing_voxel_rule():
    vs, vps = 0.25, 8
    # a vertex on the x edge between the centres of voxels 3 and 4: below the face the low voxel, at t = 0.5 (on
    # the face, 1.0 exactly) the high voxel, since floor(4 + 1e-6) = 4
    lo = (3 + 0.5) * vs
    p = np.array([[lo + 0.4 * vs, 0.125, 0.125], [lo + 0.5 * vs, 0.125, 0.125], [lo + 0.6 * vs, 0.125, 0.125]], F32)
    assert cx.containing_voxel(p, vs)[:, 0].tolist() == [3, 4, 4]
    # across a block face: voxel 7 of block 0 and voxel 0 of block 1 (x = 2.0), and the same at negative indices
    p = np.array([[1.99, 0.1, 0.1], [2.0, 0.1, 0.1], [-0.01, 0.1, 0.1], [0.0, 0.1, 0.1]], F32)
    assert cx.containing_voxel(p, vs)[:, 0].tolist() == [7, 8, -1, 0]
    idx = np.array([[0, 0, 0], [1, 0, 0]], np.int32)
    words = np.zeros((2, vps ** 3), np.uint32); words[0, 7] = 0x11223344; words[1, 0] = 0x55667788
    got = cx.vertex_colours(p, vs, vps, idx, words)
    assert got.tolist() == [0x11223344, 0x55667788, 0, 0x0]          # block (-1, 0, 0) is missing -> 0


def test_surface_colours_are_pose_independent():
    world = np.array([[3.2, 4.1, 0.7], [3.3, 4.2, 0.6], [9.1, 1.3, 2.2]])
    cols = []
    for pose in ([0.0, 0.0, 0.0, 0.0], [1.0, -2.0, 0.5, 0.9]):
        pts = (world - np.array(pose[:3])) @ synth.rot_z(pose[3])
        cols.append(synth.surface_colours(pts, np.array(pose)))
    assert np.array_equal(cols[0], cols[1]) and np.array_equal(cols[0][0], cols[0][1])
    assert not np.array_equal(cols[0][0], cols[0][2]) and len(set(cols[0][0].tolist())) == 4


def test_project_colour_restatement_single_submap(oracle):
    """One coloured submap at the identity: the restated projection returns every observed voxel's own colour
    where all 8 neighbours are observed (offset 0 interpolates to neighbour 0), and its weight."""
    import project_colour_oracle as pco
    vs, vps = 0.2, 8
    rs = np.random.RandomState(2)
    idx = np.array([[0, 0, 0], [1, 0, 0]], np.int32)
    d = rs.uniform(-0.5, 0.5, (2, vps ** 3)).astype(F32); w = rs.uniform(1, 9, (2, vps ** 3)).astype(F32)
    words = rs.randint(0, 2 ** 32, (2, vps ** 3), dtype=np.uint64).astype(np.uint32)
    T = np.array([[1, 0, 0, 0, 0, 0, 0]], F32)
    c, ow = pco.project(vs, vps, [(idx, d, w, words)], T, [5], idx)
    lin = np.arange(vps ** 3)
    inner = ((lin % vps) < vps - 1) & (((lin // vps) % vps) < vps - 1) & ((lin // vps // vps) < vps - 1)
    assert np.array_equal(c[0][inner], words[0][inner]) and np.array_equal(ow[0][inner], w[0][inner])
    c0, _ = pco.project(vs, vps, [(idx, d, w, None)], T, [5], idx)
    assert not c0.any()


def test_grayscale_colours():
    from voxgraph_b200 import api
    got = api.grayscale_colours([-5.0, 0.0, 19.6, 19.7, 5000.0, 10000.0, 2e4])
    assert got.dtype == np.uint8 and got[:, 3].tolist() == [255] * 7
    assert got[:, 0].tolist() == [0, 0, 0, 1, 128, 255, 255]       # 19.6 / 1e4 * 255 = 0.4998, 19.7 -> 0.5024
    assert np.array_equal(got[:, 0], got[:, 1]) and np.array_equal(got[:, 0], got[:, 2])


def test_colour_exports_load():
    from voxgraph_b200 import _lib, build
    build.build()
    L = _lib.load()
    for name in ("vgx_submap_has_colour", "vgx_submap_download_colour", "vgx_submap_upload_colour",
                 "vgx_submap_peek_device_colour", "vgx_submap_upload_device_colour", "vgx_collection_load_ex",
                 "vgx_mesh_download_colours", "vgx_mesh_ply_ex"):
        assert name in _lib.EXPORTS and hasattr(L, name), name
    assert _lib.VGX_COLLECTION_KEEP_COLOUR == 1
    # without a context every one of them refuses instead of touching a device
    n = C.c_int(0)
    assert L.vgx_submap_has_colour(None, 0, C.byref(n)) == _lib.VGX_ERR_INVALID
    assert L.vgx_submap_download_colour(None, 0, 0, None, C.byref(n)) == _lib.VGX_ERR_INVALID
    assert L.vgx_submap_upload_colour(None, 0, 0, None) == _lib.VGX_ERR_INVALID
    assert L.vgx_submap_upload_device_colour(None, 0, 0, None) == _lib.VGX_ERR_INVALID
    assert L.vgx_collection_load_ex(None, None, 0, 1, C.byref(n)) == _lib.VGX_ERR_INVALID
