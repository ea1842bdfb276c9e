"""Voxel colour past integration: the projected map against its CPU restatements (tests/project_oracle.c for
distance and weight, tests/project_colour_oracle.c for colour) bit for bit in any order of the ids, mesh vertex
colours against the containing-voxel rule, the coloured PLY, the end-to-end mapper on a coloured RGB-D stream, and
the invariance of projection and meshing for submaps without a colour channel."""
import itertools

import numpy as np
import pytest

import colour_exact as cx
import mesh_exact as me
import project_colour_oracle as pco
import project_oracle as po
import tsdf_exact as tx
from support import ctx, world, yaw_T  # noqa: F401
from voxgraph_b200 import api, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
_ids = itertools.count(9000)
VS, VPS = 0.2, 8


@pytest.fixture(scope="module")
def submaps(ctx, world):
    """Five submaps integrated (ray ordered) from coloured scans around the room, the third one without colours:
    [(id, T_M_S, (idx, d, w), colour words or None)], yawed and overlapping."""
    out = []
    for k, (px, py, yaw) in enumerate([(15.0, 15.0, 0.0), (16.0, 14.5, 0.5), (14.2, 15.8, -0.8), (15.5, 16.2, 1.3),
                                       (13.8, 14.1, 2.4)]):
        sid = next(_ids)
        pose = np.array([px, py, 1.2, yaw])
        ctx.submap_create(sid, VS, VPS, 4096)
        for j in range(3):     # a few scans, so the weights pass the mesher's min_weight
            pts = synth.lidar_scan(world, pose, n_beams=16, n_azimuth=256, seed=10 * k + j)
            col = synth.surface_colours(pts, pose, cell=0.7) if k != 2 else None
            ctx.tsdf_integrate(sid, synth.pose_to_T([0, 0, 0, 0]), pts, ctx.tsdf_config(max_ray_length_m=8.0), rgba=col)
        T = yaw_T(yaw, (px - 15.0, py - 15.0, 0.05 * k))
        words = ctx.submap_download_colour(sid) if k != 2 else None
        assert ctx.submap_has_colour(sid) == (k != 2)
        out.append((sid, T, ctx.submap_download(sid), words))
    yield out
    for s in out:
        ctx.submap_free(s[0])


def _project_and_check(ctx, oracle, subs, order):
    ids = [subs[i][0] for i in order]
    T = np.array([subs[i][1] for i in order], F32)
    out = next(_ids)
    before = ctx.launch_count
    ctx.project_map(ids, T, out)
    launches = ctx.launch_count - before
    try:
        idx, d, w = ctx.submap_download(out)
        has = ctx.submap_has_colour(out)
        words = ctx.submap_download_colour(out)
    finally:
        ctx.submap_free(out)
    layers = [oracle.Layer.from_blocks(VS, VPS, *subs[i][2]) for i in order]
    exp = po.project_layers(layers, T, ids).export()
    assert np.array_equal(exp[0], idx)
    tx.assert_layers_bit_equal(exp, (idx, d, w))
    ec, ew = pco.project(VS, VPS, [(*subs[i][2], subs[i][3]) for i in order], T, ids, idx)
    # the restated colour pass follows the same weights
    assert np.array_equal(ew.view(np.uint32), w.view(np.uint32))
    return idx, d, w, has, words, ec, launches


@pytest.mark.parametrize("pick", [(0, 1), (0, 1, 2, 3, 4)], ids=["two", "five"])
def test_projection_colour_bit_exact_in_any_order(ctx, oracle, submaps, pick):
    ref = None
    for order in (list(pick), list(pick)[::-1], list(np.random.RandomState(1).permutation(pick))):
        idx, d, w, has, words, ec, _ = _project_and_check(ctx, oracle, submaps, order)
        assert has
        bad = np.nonzero(words != ec)
        assert bad[0].size == 0, (len(bad[0]), hex(int(words[bad][0])), hex(int(ec[bad][0])))
        assert np.count_nonzero(words) > 1000
        if ref is None:
            ref = (idx, d, w, words)
        else:
            assert all(np.array_equal(a.view(np.uint32) if a.dtype == F32 else a, b.view(np.uint32) if b.dtype == F32 else b)
                       for a, b in zip(ref, (idx, d, w, words)))


def test_colourless_projection_and_mesh_are_unchanged(ctx, oracle, submaps):
    """Twins of two coloured submaps uploaded without colour: the projection has no channel and the same distance,
    weight and launch count as the coloured one; the mesh has the same vertices and triangles, the same launch
    count, all-zero vertex colours, and the coloured-PLY call writes the plain PLY."""
    twins = []
    for (sid, T, bricks, _) in submaps[:2]:
        t = next(_ids)
        ctx.submap_upload(t, VS, VPS, *bricks)
        twins.append((t, T, bricks, None))
    try:
        idx, d, w, has, words, ec, launches = _project_and_check(ctx, oracle, twins, [0, 1])
        cidx, cd, cw, chas, _, _, claunches = _project_and_check(ctx, oracle, submaps, [0, 1])
        assert not has and chas and not words.any() and not ec.any() and launches == claunches
        tx.assert_layers_bit_equal((idx, d, w), (cidx, cd, cw))
        res = {}
        for name, subs in (("plain", twins), ("colour", submaps[:2])):
            ids = [s[0] for s in subs]
            T = np.array([s[1] for s in subs], F32)
            before = ctx.launch_count
            vo, to = ctx.mesh_build(ids, T, ctx.mesh_config(min_weight=2.0))
            n_launch = ctx.launch_count - before
            pal = np.array([[1, 2, 3, 4], [5, 6, 7, 8]], np.uint8)
            res[name] = (ctx.mesh_download(), vo, to, n_launch, ctx.mesh_colours(), bytes(ctx.mesh_ply(pal)),
                         bytes(ctx.mesh_ply(pal, voxel_colours=True)))
        (pxyz, ptri), pvo, pto, pl, pcol, pply, pply_ex = res["plain"]
        (cxyz, ctri), cvo, cto, cl, ccol, cply, cply_ex = res["colour"]
        assert len(pxyz) > 1000 and np.array_equal(pxyz.view(np.uint32), cxyz.view(np.uint32))
        assert np.array_equal(ptri, ctri) and np.array_equal(pvo, cvo) and pl == cl
        assert not pcol.any() and ccol.any()
        assert pply == cply == pply_ex and cply_ex != cply      # vgx_mesh_ply itself keeps one colour per submap
    finally:
        for t in twins:
            ctx.submap_free(t[0])


def test_mesh_vertex_colours_follow_the_containing_voxel(ctx, submaps):
    """Submap frames (no pose), so the vertex positions are the layer-frame points of the rule; the colourless
    submap's vertices get 0 and, in the coloured PLY, the colour given for it."""
    ids = [s[0] for s in submaps[1:4]]            # coloured, colourless, coloured
    vo, to = ctx.mesh_build(ids, None, ctx.mesh_config(min_weight=2.0))
    xyz, tri = ctx.mesh_download()
    col = ctx.mesh_colours()
    assert len(col) == len(xyz) == vo[-1]
    pal = np.array([[9, 8, 7, 6], [50, 60, 70, 80], [1, 1, 1, 1]], np.uint8)
    pxyz, prgba, ptri = me.read_ply(ctx.mesh_ply(pal, voxel_colours=True))
    assert np.array_equal(pxyz.view(np.uint32), xyz.view(np.uint32)) and np.array_equal(ptri, tri)
    for k, s in enumerate(submaps[1:4]):
        a, b = vo[k], vo[k + 1]
        assert b - a > 500
        if s[3] is None:
            assert not col[a:b].any() and (prgba[a:b] == pal[k]).all()
            continue
        exp = cx.vertex_colours(xyz[a:b], VS, VPS, s[2][0], s[3])
        assert np.array_equal(col[a:b], exp)
        assert np.count_nonzero(exp) > 0.9 * len(exp) and len(np.unique(exp)) > 20
        assert np.array_equal(prgba[a:b], cx.unpack(exp))
    _, plain, _ = me.read_ply(ctx.mesh_ply(pal))
    for k in range(3):
        assert (plain[vo[k]:vo[k + 1]] == pal[k]).all()
    # with poses the colours are the same: the rule uses the position before T_M_S
    ctx.mesh_build(ids, np.array([s[1] for s in submaps[1:4]], F32), ctx.mesh_config(min_weight=2.0))
    assert np.array_equal(ctx.mesh_colours(), col)


def test_mapper_coloured_rgbd_stream_end_to_end(world, tmp_path):
    """A coloured RGB-D stream over four submaps: the combined mesh PLY carries the projected map's voxel colours
    (equal to mesh_colours(), not all white), the separated mesh stays one colour per submap, and the saved
    collection reloads with every colour channel."""
    from voxgraph_b200.mapper import MapperConfig, VoxgraphMapper
    c, c2 = api.Context(0), api.Context(0)
    try:
        m = VoxgraphMapper(c, MapperConfig(voxel_size=0.1, capacity_blocks=4096, submap_creation_interval=2.0,
                                           registration_constraints_enabled=False, mesh_min_weight=1.5,
                                           tsdf=dict(max_ray_length_m=5.0, default_truncation_distance=0.3)))
        for k in range(8):
            pose = np.array([14.0 + 0.25 * k, 15.0, 1.2, 0.15 * k])
            pts = synth.depth_scan(world, pose, width=160, height=120, fx=131.0, fy=131.0, seed=k)
            m.pointcloudCallback(float(k), pose, pts, colours=synth.surface_colours(pts, pose))
        assert len(m.submap_ids) == 4 and all(c.submap_has_colour(i) for i in m.submap_ids)
        m.saveCombinedMesh(str(tmp_path / "combined.ply"))
        words = c.mesh_colours()
        xyz, rgba, tri = me.read_ply((tmp_path / "combined.ply").read_bytes())
        assert len(xyz) > 1000 and len(tri) > 1000
        assert np.array_equal(rgba, cx.unpack(words)) and not (rgba == 255).all(1).all()
        assert len(np.unique(words)) > 50
        m.saveSeparatedMesh(str(tmp_path / "separated.ply"))
        vo = c.mesh_build(m.submap_ids, None, c.mesh_config(min_weight=1.5))[0]
        _, srgba, _ = me.read_ply((tmp_path / "separated.ply").read_bytes())
        for k, sid in enumerate(m.submap_ids):
            assert (srgba[vo[k]:vo[k + 1]] == me.rainbow((sid % 20) / 20.0)).all()
        m.saveToFile(str(tmp_path / "map.bin"))
        ids, _ = api.load_submap_collection(c2, str(tmp_path / "map.bin"), keep_colour=True)
        for i in ids:
            assert np.array_equal(c.submap_download_colour(int(i)), c2.submap_download_colour(int(i)))
    finally:
        c.close()
        c2.close()
