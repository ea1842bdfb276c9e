"""finishSubmap on the device pinned to the harness (tests/finish_exact.py) and the oracle, bit for bit
and in the same order: ESDF (and its sweep bound), relevant voxels, surface OBB and isosurface vertices
over resolutions, block layouts, fields, filters and ESDF configurations; device-integrated submaps;
re-entrance; overlap pairs; and the upload input rules."""
import ctypes as C
import itertools

import numpy as np
import pytest

import finish_exact as fx
from finish_exact import ESDF_CASES, FILTERS, MATRIX
from support import ctx  # noqa: F401
from voxgraph_b200 import _lib, synth

pytestmark = pytest.mark.gpu
_ids = itertools.count(5000)


def _esdf_kw(cfg):
    return {k[:-2] if k.endswith("_m") else k: v for k, v in cfg.items()}


def check_device(ctx, oracle, sid, vs, vps, idx, d, w, min_w=1.0, max_d=0.3, esdf_cfg=None, upload=True):
    """Device == harness == oracle for ESDF, both point sets (TSDF and ESDF distance) and the OBB."""
    from voxgraph_b200 import api
    cfg = esdf_cfg or {}
    if upload:
        ctx.submap_upload(sid, vs, vps, idx, d, w)
    g = fx.Grid(vs, vps, idx, d, w)
    L = oracle.Layer.from_blocks(vs, vps, idx, d, w)
    sweeps = ctx.submap_generate_esdf(sid, ctx.esdf_config(**cfg) if cfg else None)
    e, ob, _ = fx.esdf(g, **_esdf_kw(cfg))
    eo, obo, _ = oracle.generate_esdf(L, oracle.esdf_config(**cfg) if cfg else None)
    fx.assert_bits(eo, e, "harness esdf")
    eg, obg = ctx.submap_download_esdf(sid)
    fx.assert_bits(e, eg, "device esdf")
    fx.assert_bits(ob, obg, "device observed")
    if len(idx):
        assert 2 <= sweeps <= fx.sweep_bound(cfg.get("max_distance_m", 2.0), vs)[0]
    for use_esdf in (0, 1):
        ctx.submap_extract_points(sid, ctx.registration_filter(min_voxel_weight=min_w, max_voxel_distance=max_d,
                                                               use_esdf_distance=use_esdf))
        xyz, dd, ww, (ok, mn, mx) = fx.relevant(g, min_w, max_d, e if use_esdf else None)
        if not use_esdf:
            fx.assert_points(oracle.find_relevant_voxels(L, min_w, max_d), (xyz, dd, ww), "oracle relevant")
        fx.assert_points((xyz, dd, ww), ctx.submap_download_points(sid, api.K_VOXELS), "device relevant")
        ok_g, mn_g, mx_g = ctx.submap_surface_obb(sid)
        assert ok_g == ok
        if ok:
            fx.assert_bits(mn, mn_g, "obb min"); fx.assert_bits(mx, mx_g, "obb max")
        iso = fx.isosurface(g, min_w)
        exp = (iso["xyz"], iso["distance"], iso["weight"])
        if not use_esdf:
            xo, do_, wo, _ = oracle.find_isosurface_vertices(L, min_w)
            fx.assert_points((xo, do_, wo), exp, "oracle isosurface")
        fx.assert_points(exp, ctx.submap_download_points(sid, api.K_ISOSURFACE_POINTS), "device isosurface")
    return sweeps, iso, e


@pytest.mark.parametrize("case", range(len(MATRIX)), ids=[m[0] for m in MATRIX])
def test_matrix(ctx, oracle, case):
    sid = next(_ids)
    check_device(ctx, oracle, sid, *MATRIX[case][1])
    ctx.submap_free(sid)


@pytest.mark.parametrize("case", range(len(FILTERS)), ids=[f[0] for f in FILTERS])
def test_filters(ctx, oracle, case):
    vs, vps, idx, d, w, mw, md = FILTERS[case][1]
    sid = next(_ids)
    check_device(ctx, oracle, sid, vs, vps, idx, d, w, min_w=mw, max_d=md)
    if md == 0.0:
        assert ctx.submap_surface_obb(sid)[0] is False
    ctx.submap_free(sid)


@pytest.mark.parametrize("case", range(len(ESDF_CASES)), ids=[c[0] for c in ESDF_CASES])
def test_esdf_configs(ctx, oracle, case):
    name, lay, cfg = ESDF_CASES[case]
    sid = next(_ids)
    sweeps, _, _ = check_device(ctx, oracle, sid, *lay, esdf_cfg=cfg)
    if name == "5m-at-0.05":
        assert sweeps >= 100
    ctx.submap_free(sid)


def test_large_noise_layer_multi_chunk_scans(ctx, oracle):
    """540 blocks of noise at vps 16 (2,211,840 voxels): both voxel scans and the candidate scan run
    the multi-chunk path of scan_sums_kernel (more than 1024 tiles of 2048), with millions of
    candidates under maximal bucket contention."""
    vs, vps, idx, d, w = fx.noise_layer(0.1, 16, (9, 10, 6), seed=11, origin=(-4, -5, -3))
    assert len(idx) * vps ** 3 > 2 * 1024 * 1024
    g = fx.Grid(vs, vps, idx, d, w)
    assert len(fx.candidates(g, 1.0)[0]) > 2 * 1024 * 1024
    sid = next(_ids)
    check_device(ctx, oracle, sid, vs, vps, idx, d, w, min_w=1.0, max_d=0.3)
    ctx.submap_free(sid)


@pytest.mark.parametrize("mode", [0, 1])
def test_device_integrated_submap(ctx, oracle, mode):
    """The path the mapper runs: bricks integrated on the device (capacity-sized, slots in allocation
    order, the view built by vgx_submap_finish), then finish_ex and generate_esdf.  The result equals the
    harness and oracle on the downloaded bricks in slot order, and a host upload of those bricks."""
    from voxgraph_b200 import api
    world = synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=16, n_azimuth=256, seed=1)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    sid, sid_h = next(_ids), next(_ids)
    ctx.submap_create(sid, 0.2, 16, 4096)
    ctx.tsdf_integrate(sid, T, pts, ctx.tsdf_config(mode=mode))
    filt = ctx.registration_filter(min_voxel_weight=1e-6)
    ctx.submap_finish_ex(sid, filt)
    idx, d, w = ctx.submap_download(sid)
    assert len(idx) > 50
    got = [ctx.submap_download_points(sid, t) for t in (api.K_VOXELS, api.K_ISOSURFACE_POINTS)]
    obb = ctx.submap_surface_obb(sid)
    ctx.submap_generate_esdf(sid)
    eg = ctx.submap_download_esdf(sid)
    _, iso, e = check_device(ctx, oracle, sid_h, 0.2, 16, idx, d, w, min_w=1e-6, max_d=0.3)
    assert len(iso["xyz"]) > 100
    fx.assert_bits(e, eg[0], "integrated esdf")
    ctx.submap_extract_points(sid_h, filt)
    for t, pg in zip((api.K_VOXELS, api.K_ISOSURFACE_POINTS), got):
        fx.assert_points(ctx.submap_download_points(sid_h, t), pg, "integrated vs uploaded")
    oh = ctx.submap_surface_obb(sid_h)
    assert obb[0] == oh[0] and np.array_equal(obb[1], oh[1]) and np.array_equal(obb[2], oh[2])
    ctx.submap_free(sid); ctx.submap_free(sid_h)


def test_reentrance(ctx, oracle):
    from voxgraph_b200 import api
    vs, vps, idx, d, w = fx.layer((0.2, 16), "box", "sphere")
    a, b = next(_ids), next(_ids)
    ctx.submap_upload(a, vs, vps, idx, d, w)
    ctx.submap_upload(b, vs, vps, idx, d, w)
    # find_overlapping_pairs refuses a submap that has not been extracted
    with pytest.raises(api.VgxError):
        ctx.find_overlapping_pairs([a, b], np.tile(np.float32([1, 0, 0, 0, 0, 0, 0]), (2, 1)))
    # extracting twice with different filters equals a fresh extraction
    ctx.submap_extract_points(a, ctx.registration_filter(min_voxel_weight=0.0, max_voxel_distance=0.6))
    ctx.submap_extract_points(a, ctx.registration_filter(min_voxel_weight=1.0, max_voxel_distance=0.3))
    ctx.submap_extract_points(b, ctx.registration_filter(min_voxel_weight=1.0, max_voxel_distance=0.3))
    for t in (api.K_VOXELS, api.K_ISOSURFACE_POINTS):
        fx.assert_points(ctx.submap_download_points(b, t), ctx.submap_download_points(a, t), "re-extraction")
    assert [np.array_equal(x, y) for x, y in zip(ctx.submap_surface_obb(a)[1:], ctx.submap_surface_obb(b)[1:])] == [True, True]
    # a regenerated ESDF replaces the first everywhere: download, use_esdf_distance extraction, emit branch
    ctx.submap_generate_esdf(a, ctx.esdf_config(max_distance_m=0.5, default_distance_m=0.5))
    ctx.submap_generate_esdf(a)
    ctx.submap_generate_esdf(b)
    fx.assert_bits(ctx.submap_download_esdf(b)[0], ctx.submap_download_esdf(a)[0], "regenerated esdf")
    f1 = ctx.registration_filter(use_esdf_distance=1)
    ctx.submap_extract_points(a, f1); ctx.submap_extract_points(b, f1)
    fx.assert_points(ctx.submap_download_points(b, api.K_VOXELS), ctx.submap_download_points(a, api.K_VOXELS),
                     "esdf-distance extraction")
    ref = np.array([0.0, 0.0, 0.0, 0.0]); read = np.array([0.05, -0.03, 0.02, 0.01])
    ra = ctx.reg_eval_emit(b, a, ref, read, ctx.reg_config(use_esdf_distance=1))    # reads a's ESDF
    rb = ctx.reg_eval_emit(a, b, ref, read, ctx.reg_config(use_esdf_distance=1))
    assert ra[0] and rb[0] and all(np.array_equal(x, y) for x, y in zip(ra[1:], rb[1:]))
    # re-uploading under the same id clears the extraction state
    ctx.submap_upload(a, vs, vps, idx, d, w)
    assert ctx.submap_num_points(a, api.K_VOXELS) == 0 and ctx.submap_num_points(a, api.K_ISOSURFACE_POINTS) == 0
    with pytest.raises(api.VgxError):
        ctx.find_overlapping_pairs([a, b], np.tile(np.float32([1, 0, 0, 0, 0, 0, 0]), (2, 1)))
    ctx.submap_free(a); ctx.submap_free(b)


# --------------------------------------------------------------------------- overlap
def _overlap_expect(oracle, subs, T):
    """updateOverlappingSubmapList over the oracle's overlapsWith; subs = [(vs, vps, idx, d, w)]."""
    layers = [oracle.Layer.from_blocks(*s) for s in subs]
    obbs = [oracle.surface_obb(L, 1.0, 0.3) for L in layers]
    isos = [oracle.find_isosurface_vertices(L, 1.0)[3] for L in layers]
    aabbs = [oracle.aabb_from_obb_and_pose(o[1], o[2], T[k]) for k, o in enumerate(obbs)]
    for k, (ok, mn, mx) in enumerate(obbs):          # each AABB holds its transformed OBB corners (float64)
        if not ok:
            continue
        q = T[k, :4].astype(np.float64); t = T[k, 4:].astype(np.float64)
        R = _quat_R(q)
        for c in range(8):
            p = np.array([mn[a] if (c >> a) & 1 else mx[a] for a in range(3)], np.float64)
            m = R @ p + t
            tol = 1e-5 * (1 + np.abs(m))
            assert np.all(m >= aabbs[k][0] - tol) and np.all(m <= aabbs[k][1] + tol)
    want = []
    for i in range(len(subs)):
        for j in range(i + 1, len(subs)):
            bs = np.float32(np.float32(subs[i][0]) * np.float32(subs[i][1]))
            if oracle.submaps_overlap(aabbs[i], aabbs[j], T[i], T[j], isos[i], bs, layers[j]):
                want.append((i, j))
    return want, isos


def _quat_R(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _run_overlap(ctx, oracle, subs, T, max_pairs=None):
    ids = [next(_ids) for _ in subs]
    for sid, s in zip(ids, subs):
        ctx.submap_upload(sid, *s)
        ctx.submap_extract_points(sid, None)
    want, isos = _overlap_expect(oracle, subs, T)
    got = ctx.find_overlapping_pairs(ids, T)
    assert got == [(ids[i], ids[j]) for i, j in want]
    if want:      # the capacity error at max_pairs one short, and success at exactly enough
        idv = np.ascontiguousarray(ids, np.uint32); Tv = np.ascontiguousarray(T, np.float32)
        out = np.zeros((len(want), 2), np.uint32); n = C.c_int(0)
        p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
        rc = ctx._L.vgx_find_overlapping_pairs(ctx._h, len(ids), p(idv, C.c_uint32), p(Tv, C.c_float),
                                               len(want) - 1, p(out, C.c_uint32), C.byref(n))
        assert rc == _lib.VGX_ERR_CAPACITY and n.value == len(want)
        rc = ctx._L.vgx_find_overlapping_pairs(ctx._h, len(ids), p(idv, C.c_uint32), p(Tv, C.c_float),
                                               len(want), p(out, C.c_uint32), C.byref(n))
        assert rc == 0 and [tuple(int(v) for v in r) for r in out] == [(ids[i], ids[j]) for i, j in want]
    for sid in ids:
        ctx.submap_free(sid)
    return want, isos


def _T(x, y, z, yaw=0.0):
    return synth.pose_to_T([x, y, z, yaw]).astype(np.float32)


def test_overlap_mixed_resolutions(ctx, oracle):
    """0.1/16 with 0.2/16 and with 0.05/32 (other_block_size_inv of the other submap), rotated poses."""
    subs = [fx.layer((0.1, 16), "box", "tilted"), fx.layer((0.2, 16), "box", "sphere"),
            fx.layer((0.05, 32), "box", "plane"), fx.layer((0.1, 16), "straddle", "sphere")]
    rs = np.random.RandomState(4)
    hits = 0
    for trial in range(6):
        T = np.stack([_T(*rs.uniform(-1.0, 1.0, 3), rs.uniform(-3, 3)) for _ in subs])
        want, _ = _run_overlap(ctx, oracle, subs, T)
        hits += len(want)
    assert hits > 5


def test_overlap_exact_binary_block_centres(ctx, oracle):
    """Block sizes 2 m (0.25/8) and 1 m (0.125/8 at vps 8): the 2 m block centres land exactly on the
    1 m grid's block boundaries (the +1e-6 floor decides), at translations of whole metres."""
    a = fx.layer((0.25, 8), "box", "crafted")
    b = fx.layer((0.125, 8), "straddle", "tilted")
    c = fx.layer((0.125, 8), "negative", "tilted")
    for t in ([0, 0, 0], [1, 0, 0], [-1, 1, 0], [0, -2, 1], [3, 0, 0], [-4, -3, -2]):
        _run_overlap(ctx, oracle, [a, b, c], np.stack([_T(0, 0, 0), _T(*t), _T(*t)]))


def test_overlap_touching_aabbs_invalid_obb_and_no_isosurface(ctx, oracle):
    """Two unrotated box submaps whose surface AABBs touch exactly (the separation test is strict),
    then one submap without relevant voxels (invalid OBB) and one without isosurface vertices."""
    from voxgraph_b200 import api
    vs, vps = 0.25, 8
    # block 0 holds every relevant voxel (surface OBB = block 0, [0, 2] m in x); block 1 holds
    # crossings of +-0.5 only (isosurface vertices, none of them relevant)
    idx = np.array([(0, 0, 0), (1, 0, 0)], np.int32)
    d = np.full((2, vps ** 3), 0.1, np.float32); w = np.full_like(d, 2.0)
    d[1] = np.where(np.arange(vps ** 3) % 2 == 0, 0.5, -0.5)
    s = (vs, vps, idx, d, w)
    # translating by exactly 2 m makes the AABBs touch at x = 2, and block 1's centre lands in block 0
    want, isos = _run_overlap(ctx, oracle, [s, s], np.stack([_T(0, 0, 0), _T(2.0, 0, 0)]))
    assert want == [(0, 1)]
    empty_obb = (vs, vps, idx, np.full_like(d, 0.5), w)          # no |d| < 0.3, no crossing
    no_iso = (vs, vps, idx, np.full_like(d, 0.1), w)             # relevant voxels, no crossing
    want, isos = _run_overlap(ctx, oracle, [s, empty_obb, no_iso, s],
                              np.stack([_T(0, 0, 0), _T(0.5, 0, 0), _T(0.2, 0.1, 0), _T(0.3, 0, 0)]))
    assert len(isos[2]) == 0 and (0, 3) in want and not any(1 in p for p in want)
    sid = next(_ids)
    ctx.submap_upload(sid, *empty_obb)
    ctx.submap_extract_points(sid, None)
    assert ctx.submap_surface_obb(sid)[0] is False
    assert ctx.submap_num_points(sid, api.K_VOXELS) == 0
    ctx.submap_free(sid)


def test_overlap_many_isosurface_blocks_pair_order_and_small_n(ctx, oracle):
    """A submap with more than 128 isosurface blocks (more than one pass of the 128-thread CTA), pairs
    reported in (i, j > i) order, and n = 0 and n = 1."""
    vs, vps = 0.1, 4
    idx = np.array([(i, j, k) for k in range(2) for j in range(12) for i in range(12)], np.int32)
    d, w = fx.field("tilted", vs, vps, idx)
    big = (vs, vps, idx, d, w)
    subs = [big, fx.layer((0.2, 16), "box", "sphere"), big, fx.layer((0.1, 4), "one", "plane")]
    T = np.stack([_T(0, 0, 0), _T(0.2, 0.1, 0.0, 0.3), _T(0.05, 0, 0, 0.1), _T(0.3, 0.3, 0)])
    want, isos = _run_overlap(ctx, oracle, subs, T)
    assert len(isos[0]) > 128 and len(want) >= 3
    assert ctx.find_overlapping_pairs([], np.zeros((0, 7), np.float32)) == []
    sid = next(_ids)
    ctx.submap_upload(sid, *big)
    ctx.submap_extract_points(sid, None)
    assert ctx.find_overlapping_pairs([sid], T[:1]) == []
    ctx.submap_free(sid)


# --------------------------------------------------------------------------- input rules
def _upload_device(ctx, sid, vs, vps, idx, d, w):
    import torch
    bi = torch.tensor(np.asarray(idx, np.int32), device="cuda")
    dw = torch.tensor(np.stack([np.asarray(d, np.float32), np.asarray(w, np.float32)], -1), device="cuda")
    torch.cuda.synchronize()
    ctx.submap_upload_device(sid, vs, vps, len(idx), bi.data_ptr(), dw.data_ptr())


@pytest.mark.parametrize("path", ["host", "device"])
def test_upload_rejects_repeated_and_out_of_range_indices(ctx, oracle, path):
    """Repeated block indices, and indices whose +-1 neighbours would alias in the 21-bit hash key
    (one index on each side of both edges of the accepted range), fail with VGX_ERR_INVALID and leave
    no submap under the id; the indices at the edges themselves are accepted and extract as the
    oracle does."""
    from voxgraph_b200 import api
    up = ctx.submap_upload if path == "host" else (lambda *a: _upload_device(ctx, *a))
    vs, vps = 0.25, 8
    lo, hi = fx.INDEX_MIN, fx.INDEX_MAX
    base = [(0, 0, 0), (1, 0, 0), (0, 1, 0)]
    bad_sets = [base + [(1, 0, 0)]]
    for v in (lo - 1, hi + 1):
        for a in range(3):
            q = [0, 0, 0]; q[a] = v
            bad_sets.append(base + [tuple(q)])
    for bad in bad_sets:
        idx = np.array(bad, np.int32)
        d, w = fx.field("tilted", vs, vps, idx)
        sid = next(_ids)
        with pytest.raises(api.VgxError) as e:
            up(sid, vs, vps, idx, d, w)
        assert e.value.code == _lib.VGX_ERR_INVALID
        with pytest.raises(api.VgxError):
            ctx.submap_info(sid)
    for v in (lo, hi):
        idx = np.array([(v, 0, 0), (0, v, 0), (0, 0, v), (v, v, v)], np.int32)
        d, w = fx.field("tilted", vs, vps, idx)
        sid = next(_ids)
        up(sid, vs, vps, idx, d, w)
        check_device(ctx, oracle, sid, vs, vps, idx, d, w, upload=False)
        ctx.submap_free(sid)
