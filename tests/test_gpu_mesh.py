"""vgx_mesh_build / vgx_mesh_download / vgx_mesh_ply on the device against the restatement in
tests/mesh_exact.py, bit for bit and in the same order: the finishSubmap layer matrix, all 256 cube
configurations, special values, device-integrated submaps (an active one mid-stream included),
separated meshes with poses and mixed voxel sizes, the error and capacity paths, non-interference with
the rest of the device state, and the mapper end to end."""
import ctypes as C
import itertools

import numpy as np
import pytest

import finish_exact as fx
import mesh_exact as me
from finish_exact import MATRIX
from support import ctx, same_bits  # noqa: F401
from voxgraph_b200 import _lib, synth

pytestmark = pytest.mark.gpu
_ids = itertools.count(9000)


def _check(ctx, layers, poses=None, min_weight=1.0, upload=True, ids=None):
    """Separated mesh of layers [(vs, vps, idx, d, w)] on the device == restatement."""
    ids = ids or [next(_ids) for _ in layers]
    if upload:
        for sid, lay in zip(ids, layers):
            ctx.submap_upload(sid, *lay)
    from voxgraph_b200 import api
    xyz, tri, vo, to = api.separated_mesh(ctx, ids, poses, min_weight)
    ex, et, evo, eto = me.separated([fx.Grid(*lay) for lay in layers], poses, min_weight)
    assert vo.tolist() == evo.tolist() and to.tolist() == eto.tolist()
    same_bits(ex, xyz, "vertices")
    same_bits(et, tri, "triangles")
    return ids, xyz, tri


@pytest.mark.parametrize("case", range(len(MATRIX)), ids=[m[0] for m in MATRIX])
def test_matrix(ctx, case):
    ids, _, _ = _check(ctx, [MATRIX[case][1]])
    ctx.submap_free(ids[0])


def test_matrix_in_one_build(ctx):
    """Every layer of the matrix in one build (one launch per pass over all of them), each at a pose."""
    layers = [m[1] for m in MATRIX]
    rs = np.random.RandomState(3)
    T = np.stack([synth.pose_to_T([*rs.uniform(-5, 5, 3), rs.uniform(-3, 3)]) for _ in layers]).astype(np.float32)
    ctx.profile_reset()
    ids, xyz, tri = _check(ctx, layers, T)
    ms, launches = ctx.profile_get(_lib.VGX_SLOT_MESH)
    assert launches == 11      # count, scan (3), popcount, scan (3), offsets, vertices, triangles
    assert len(tri) > 10000
    for sid in ids:
        ctx.submap_free(sid)


def _all_configurations(vs=0.1, vps=16):
    """256 isolated 2x2x2 cubes (stride 3 voxels, invalid voxels between them), cube c with configuration c."""
    starts = [3 * k for k in range(vps) if 3 * k + 1 < vps]
    per_block = len(starts) ** 3
    n_blocks = -(-256 // per_block)
    idx = np.array([(b, 0, 0) for b in range(n_blocks)], np.int32)
    d = np.full((n_blocks, vps ** 3), 0.3, np.float32)
    w = np.zeros((n_blocks, vps ** 3), np.float32)
    rs = np.random.RandomState(5)
    cfg = 0
    for b in range(n_blocks):
        for z in starts:
            for y in starts:
                for x in starts:
                    if cfg >= 256:
                        continue
                    for k, (ox, oy, oz) in enumerate(me.CUBE_OFF):
                        lin = (x + ox) + vps * ((y + oy) + vps * (z + oz))
                        mag = np.float32(rs.uniform(0.01, 0.1))
                        d[b, lin] = -mag if (cfg >> k) & 1 else mag
                        w[b, lin] = 3.0
                    cfg += 1
    return vs, vps, idx, d, w


def test_all_256_configurations(ctx):
    lay = _all_configurations()
    ids, xyz, tri = _check(ctx, [lay], min_weight=2.0)
    assert len(tri) == sum(len(me.triangles(c)) for c in range(256))
    ctx.submap_free(ids[0])


def test_special_values(ctx):
    """+-0.0, sdf exactly 0 at corners, |d| < 1e-6 edges (the midpoint branch), weights equal to
    min_weight (invalid), NaN and Inf distances."""
    vs, vps = 0.25, 8
    idx = fx.layout("straddle")
    d, w = fx.field("crafted", vs, vps, idx)
    rs = np.random.RandomState(1)
    d = d.copy(); w = w.copy()
    flat = d.reshape(-1)
    pick = rs.choice(flat.size, 400, replace=False)
    flat[pick[:100]] = np.float32(-0.0)
    flat[pick[100:150]] = np.float32(0.0)
    flat[pick[150:200]] = np.float32(np.nan)
    flat[pick[200:250]] = np.float32(np.inf)
    flat[pick[250:300]] = np.float32(-np.inf)
    flat[pick[300:350]] = np.float32(-4e-7)
    w = np.full_like(w, 2.5)
    w.reshape(-1)[pick[350:]] = np.float32(2.0)        # == min_weight: invalid
    w.reshape(-1)[rs.choice(flat.size, 200, replace=False)] = np.float32(2.0000002)   # just above: valid
    ids, xyz, tri = _check(ctx, [(vs, vps, idx, d, w)], min_weight=2.0)
    assert np.isnan(xyz).any() and len(tri) > 0
    # every weight at or below min_weight: nothing is meshed
    _, xyz, tri = _check(ctx, [(vs, vps, idx, d, w)], min_weight=2.5, upload=False, ids=ids)
    assert len(xyz) == 0 and len(tri) == 0
    ctx.submap_free(ids[0])


@pytest.mark.parametrize("mode", [0, 1])
def test_device_integrated_and_active_submaps(ctx, mode):
    """Bricks integrated on the device (capacity-sized, allocation order), meshed while the submap is
    still active, after another scan, and after finishing; each equals the restatement on the
    downloaded bricks."""
    world = synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)
    sid = next(_ids)
    ctx.submap_create(sid, 0.2, 16, 4096)
    cfg = ctx.tsdf_config(mode=mode)
    for k, pose in enumerate(([15.0, 15.0, 1.2, 0.4], [16.0, 14.5, 1.2, 0.6])):
        pts = synth.lidar_scan(world, np.array(pose), n_beams=16, n_azimuth=256, seed=k)
        ctx.tsdf_integrate(sid, synth.pose_to_T([0.3 * k, -0.2, 0.1, 0.4]), pts, cfg)
        idx, d, w = ctx.submap_download(sid)
        _, _, tri = _check(ctx, [(0.2, 16, idx, d, w)], min_weight=0.5, upload=False, ids=[sid])
        assert len(tri) > 100
    ctx.submap_finish_ex(sid, ctx.registration_filter(min_voxel_weight=1e-6))
    idx, d, w = ctx.submap_download(sid)
    _check(ctx, [(0.2, 16, idx, d, w)], min_weight=2.0, upload=False, ids=[sid])
    ctx.submap_free(sid)


def test_separated_mesh_poses_and_mixed_resolutions(ctx):
    layers = [fx.layer((0.1, 16), "box", "tilted"), fx.layer((0.2, 16), "box", "sphere"),
              fx.layer((0.05, 32), "box", "plane"), fx.layer((0.1, 4), "zero", "plane"),
              fx.layer((0.125, 16), "negative", "crafted")]
    T = np.stack([synth.pose_to_T(p) for p in ([0, 0, 0, 0], [1.5, -2.0, 0.3, 0.7], [-3.0, 4.0, 1.0, -2.5],
                                              [0, 0, 0, 1.0], [10.0, 0.25, -1.0, 3.0])]).astype(np.float32)
    ids, xyz, tri = _check(ctx, layers, T)
    # without poses: the submap frames
    from voxgraph_b200 import api
    xyz0, tri0, _, _ = api.separated_mesh(ctx, ids, None, 1.0)
    ex, et, _, _ = me.separated([fx.Grid(*lay) for lay in layers], None, 1.0)
    same_bits(ex, xyz0, "submap frame"); same_bits(et, tri0, "submap frame triangles")
    for sid in ids:
        ctx.submap_free(sid)


def test_errors_release_and_ply_paths(ctx):
    from voxgraph_b200 import api
    lay = fx.layer((0.1, 8), "box", "sphere")
    a, b = next(_ids), next(_ids)
    ctx.submap_upload(a, *lay)
    ctx.submap_upload(b, *lay)
    cfg = ctx.mesh_config(min_weight=1.0)     # the layer's weights are 2.0, the default min_weight
    vo, to = ctx.mesh_build([a, b], None, cfg)
    xyz, tri = ctx.mesh_download()
    assert len(tri) > 0 and vo[-1] == len(xyz) and to[-1] == len(tri)
    # PLY: the default palette is rainbowColorMap((id mod 20) / 20), and the file parses back to the mesh
    data = ctx.mesh_ply()
    assert bytes(data) == bytes(ctx.mesh_ply(np.array([me.rainbow((a % 20) / 20.0), me.rainbow((b % 20) / 20.0)],
                                                      np.uint8)))
    px, prgba, ptri = me.read_ply(data)
    same_bits(xyz, px, "ply vertices")
    assert np.array_equal(ptri, tri.astype(np.int64))
    for k, sid in enumerate((a, b)):
        assert (prgba[vo[k]:vo[k + 1]] == me.rainbow((sid % 20) / 20.0)).all()
    # size query, capacity error, exact capacity
    L, h = ctx._L, ctx._h
    size = C.c_uint64(0)
    assert L.vgx_mesh_ply(h, None, None, 0, C.byref(size)) == 0 and size.value == len(data)
    buf = (C.c_char * len(data))()
    assert L.vgx_mesh_ply(h, None, buf, len(data) - 1, C.byref(size)) == _lib.VGX_ERR_CAPACITY
    assert size.value == len(data)
    assert L.vgx_mesh_ply(h, None, buf, len(data), C.byref(size)) == 0 and bytes(buf) == bytes(data)
    # download capacity and NULL outputs
    nv, nt = C.c_int64(0), C.c_int64(0)
    small = np.zeros((len(xyz) - 1, 3), np.float32)
    assert L.vgx_mesh_download(h, len(xyz) - 1, small.ctypes.data_as(C.POINTER(C.c_float)), 0, None,
                               C.byref(nv), C.byref(nt)) == _lib.VGX_ERR_CAPACITY
    assert nv.value == len(xyz) and nt.value == len(tri)
    # unknown id: VGX_ERR_NOT_FOUND and an empty mesh
    with pytest.raises(api.VgxError) as e:
        ctx.mesh_build([a, 4242424242], None, cfg)
    assert e.value.code == _lib.VGX_ERR_NOT_FOUND
    x2, t2 = ctx.mesh_download()
    assert len(x2) == 0 and len(t2) == 0
    # n = 0 releases the buffer; the PLY of nothing is a header
    ctx.mesh_build([a], None, cfg)
    assert len(ctx.mesh_download()[1]) > 0
    vo, to = ctx.mesh_build([])
    assert vo.tolist() == [0] and to.tolist() == [0] and len(ctx.mesh_download()[0]) == 0
    px, _, ptri = me.read_ply(ctx.mesh_ply())
    assert len(px) == 0 and len(ptri) == 0
    ctx.submap_free(a); ctx.submap_free(b)


def test_default_palette_is_rainbow_of_id_mod_20(ctx):
    """vgx_mesh_ply without colours gives submap id k rainbowColorMap((k mod 20) / 20): one full cycle, its wrap
    and the largest id."""
    lay = fx.layer((0.1, 8), "box", "sphere")
    ids = list(range(21)) + [2 ** 32 - 1]
    for sid in ids:
        ctx.submap_upload(sid, *lay)
    vo, _ = ctx.mesh_build(ids, None, ctx.mesh_config(min_weight=1.0))
    _, rgba, _ = me.read_ply(ctx.mesh_ply())
    for k, sid in enumerate(ids):
        assert vo[k + 1] > vo[k] and (rgba[vo[k]:vo[k + 1]] == me.rainbow((sid % 20) / 20.0)).all(), sid
    for sid in ids:
        ctx.submap_free(sid)


def test_non_interference_and_repeatability(ctx, pair_scene):
    """Bricks, registration points and the fused evaluation are bit-identical before and after mesh
    builds, and two builds are bit-identical."""
    from voxgraph_b200 import api
    c = api.Context(0)
    for s in pair_scene.submaps:
        c.upload_synth_submap(s)
        c.submap_extract_points(s.submap_id, None)
    pg = api.PoseGraph(c)
    for i in range(2):
        pg.addSubmapNode(api.SubmapNodeConfig(i, pair_scene.poses_init[i], set_constant=(i == 0)))
    pg.addRegistrationConstraint(api.RegistrationConstraintConfig(0, 1))
    ids = [s.submap_id for s in pair_scene.submaps]

    def state():
        out = [c.submap_download(i) for i in ids]
        out += [c.submap_download_points(i, t) for i in ids for t in (0, 1)]
        ok, cost, g, H = pg.evaluate()
        return out, (ok, cost, g.tobytes(), H.tobytes())

    before = state()
    T = np.stack([synth.pose_to_T(p) for p in pair_scene.poses_init]).astype(np.float32)
    m1 = api.separated_mesh(c, ids, T, 1.0)
    m2 = api.separated_mesh(c, ids, T, 1.0)
    after = state()
    assert len(m1[1]) > 0
    for x, y in zip(m1, m2):
        assert x.tobytes() == y.tobytes()
    for x, y in zip(before[0], after[0]):
        for p, q in zip(x, y):
            assert p.tobytes() == q.tobytes()
    assert before[1] == after[1]
    c.close()


def test_mapper_save_separated_mesh(tmp_path):
    from voxgraph_b200 import api, mapper as vm
    c = api.Context(0)
    world = synth.make_world(7, size_xy=(40.0, 30.0), n_clutter=60, n_walls=5)
    n = 10
    s_arc = np.arange(n) * 0.6
    gt = np.stack([8.0 + s_arc, 12.0 + 0.5 * np.sin(s_arc / 3.0), np.full(n, 1.2), 0.05 * s_arc], -1)
    cfg = vm.MapperConfig(voxel_size=0.2, submap_creation_interval=4 / 10.0, capacity_blocks=4096,
                          tsdf=dict(max_ray_length_m=12.0))
    m = vm.VoxgraphMapper(c, cfg)
    for k in range(n):
        m.pointcloudCallback(k / 10.0, gt[k], synth.lidar_scan(world, gt[k], n_beams=24, n_azimuth=360,
                                                               seed=k, max_range=12.0))
    assert len(m.submap_ids) == 3
    path = tmp_path / "mesh.ply"
    size = m.saveSeparatedMesh(str(path))
    data = path.read_bytes()
    assert size == len(data)
    xyz, rgba, tri = me.read_ply(data)
    per = [len(api.separated_mesh(c, [i], None, 2.0)[1]) for i in m.submap_ids]
    assert all(p > 0 for p in per) and len(tri) == sum(per)
    ax, at = m.activeSubmapMesh()
    idx, d, w = c.submap_download(m.active_id)
    ex, et = me.mesh(fx.Grid(0.2, 16, idx, d, w), 2.0)
    same_bits(ex, ax, "active submap"); same_bits(et.astype(np.uint32), at, "active submap triangles")
    c.close()
