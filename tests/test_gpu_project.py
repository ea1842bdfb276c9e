"""vgx_project_map (cblox SubmapCollection::getProjectedMap) on the device against its CPU restatement
tests/project_oracle.c, bit for bit and in the same block order: the finishSubmap layer matrix at identity,
translations, yaw and random poses; 1, 2 and 20 overlapping submaps at two resolutions with NaN and
unobserved voxels; device-integrated submaps, active and finished.  Also: every error path (nothing left
behind, other submaps untouched), the launch count of profiling slot 13, determinism, the combined mesh
against tests/mesh_exact.py on the restatement's projected layer, the collection save / load round trip of a
projected map, and the mapper's combined-mesh PLY."""
import itertools

import numpy as np
import pytest

import finish_exact as fx
import mesh_exact as me
import project_oracle as po
from finish_exact import MATRIX
from support import IDENTITY, ctx, exists, poses_for, same_bits, yaw_T  # noqa: F401
from voxgraph_b200 import _lib, synth

pytestmark = pytest.mark.gpu
_ids = itertools.count(20000)
F32 = np.float32
LAUNCHES = 15    # candidates, sort, flags, 2 scans (3 each), scatter, occupancy, scan (3), fold
SCRATCH_ID = 0xFFFFFFFE   # vgx_mesh_build_combined's scratch submap while the context holds no id above 20000


def _oracle(oracle, layers, poses, ids):
    L = [oracle.Layer.from_blocks(vs, vps, idx, d, w) for (vs, vps, idx, d, w) in layers]
    return po.project_layers(L, np.asarray(poses, F32).reshape(-1, 7), ids).export()


def _check(ctx, oracle, layers, poses, ids=None, upload=True):
    """Project layers [(vs, vps, idx, d, w)] at poses on the device == oracle -> (idx, d, w) or None when
    both refuse (VGX_ERR_INVALID, no output submap)."""
    from voxgraph_b200 import api
    ids = ids or [next(_ids) for _ in layers]
    if upload:
        for sid, lay in zip(ids, layers):
            ctx.submap_upload(sid, *lay)
    out = next(_ids)
    try:
        exp = _oracle(oracle, layers, poses, ids)
    except ValueError:
        exp = None
    if exp is None:
        with pytest.raises(api.VgxError) as e:
            ctx.project_map(ids, poses, out)
        assert e.value.code == _lib.VGX_ERR_INVALID and not exists(ctx, out)
        return ids, None
    n = ctx.project_map(ids, poses, out)
    vs, vps, nb, fin = ctx.submap_info(out)
    assert fin and nb == n == len(exp[0]) and vps == layers[0][1] and vs == F32(layers[0][0])
    got = ctx.submap_download(out)
    ctx.submap_free(out)
    same_bits(exp[0], got[0], "block indices")
    same_bits(exp[1], got[1], "distance")
    same_bits(exp[2], got[2], "weight")
    return ids, got


@pytest.mark.parametrize("case", range(len(MATRIX)), ids=[m[0] for m in MATRIX])
def test_matrix(ctx, oracle, case):
    lay = MATRIX[case][1]
    ids = None
    for name, T in poses_for(lay[0], lay[1]).items():
        ids, _ = _check(ctx, oracle, [lay], T[None], ids=ids, upload=ids is None)
    ctx.submap_free(ids[0])


def _overlapping(vs, vps, n, seed):
    """n submaps over one region: noisy planes and spheres, some voxels unobserved, a few NaN distances,
    at poses within a block of each other."""
    rs = np.random.RandomState(seed)
    layers, poses = [], []
    bs = float(F32(vs) * vps)
    for k in range(n):
        lay = fx.layer((vs, vps), "box", ["tilted", "sphere", "plane", "noise"][k % 4], seed=seed + k)
        d = lay[3].copy(); w = lay[4].copy()
        w *= rs.uniform(0.5, 3.0, w.shape).astype(F32)
        w[rs.uniform(size=w.shape) < 0.05] = 0
        d[rs.uniform(size=d.shape) < 0.002] = np.nan
        layers.append((vs, vps, lay[2], d, w))
        poses.append(yaw_T(rs.uniform(-0.5, 0.5), rs.uniform(-0.5 * bs, 0.5 * bs, 3)))
    return layers, np.stack(poses)


@pytest.mark.parametrize("res", [(0.1, 8), (0.2, 16)], ids=["0.1-8", "0.2-16"])
@pytest.mark.parametrize("n", [1, 2, 20])
def test_overlapping_submaps(ctx, oracle, res, n):
    layers, poses = _overlapping(res[0], res[1], n, seed=7 * n + res[1])
    ids, got = _check(ctx, oracle, layers, poses)
    assert got is not None and len(got[0]) > 0
    if n > 1:   # the ids in any order give the same map
        perm = np.random.RandomState(n).permutation(n)
        out = next(_ids)
        ctx.project_map([ids[p] for p in perm], poses[perm], out)
        again = ctx.submap_download(out)
        ctx.submap_free(out)
        for x, y in zip(got, again):
            assert x.tobytes() == y.tobytes()
    for sid in ids:
        ctx.submap_free(sid)


@pytest.mark.parametrize("mode", [0, 1])
def test_device_integrated_active_and_finished(ctx, oracle, mode):
    world = synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)
    a, b = next(_ids), next(_ids)
    cfg = ctx.tsdf_config(mode=mode)
    for k, sid in enumerate((a, b)):
        ctx.submap_create(sid, 0.2, 16, 4096)
        pose = np.array([15.0 + k, 15.0 - 0.5 * k, 1.2, 0.4 + 0.2 * k])
        pts = synth.lidar_scan(world, pose, n_beams=16, n_azimuth=256, seed=k)
        ctx.tsdf_integrate(sid, synth.pose_to_T([0.3 * k, -0.2, 0.1, 0.4]), pts, cfg)
    ctx.submap_finish_ex(a, ctx.registration_filter(min_voxel_weight=1e-6))   # b stays active
    assert ctx.submap_info(a)[3] and not ctx.submap_info(b)[3]
    layers = [(0.2, 16, *ctx.submap_download(s)) for s in (a, b)]
    T = np.stack([yaw_T(0.0), yaw_T(0.3, (0.4, -0.2, 0.0))])
    _, got = _check(ctx, oracle, layers, T, ids=[a, b], upload=False)
    assert len(got[0]) > 20 and (got[2] > 0).sum() > 1000
    ctx.submap_free(a); ctx.submap_free(b)


def test_errors_leave_nothing(ctx):
    from voxgraph_b200 import api
    a, b, c8, far, out = (next(_ids) for _ in range(5))
    ctx.submap_upload(a, *fx.layer((0.1, 16), "box", "sphere"))
    ctx.submap_upload(b, *fx.layer((0.2, 16), "box", "plane"))
    ctx.submap_upload(c8, *fx.layer((0.1, 8), "box", "plane"))
    ctx.submap_upload(far, *fx.layer((0.1, 16), "range_edges", "plane"))
    keep = [a, b, c8, far]

    def state():
        return [tuple(x.tobytes() for x in ctx.submap_download(s)) for s in keep]

    before = state()
    shift = IDENTITY.copy(); shift[4] = 2 * 1.6     # two blocks of 1.6 along x
    cases = [([a, 4242424242], _lib.VGX_ERR_NOT_FOUND, out),  # unknown id
             ([a], _lib.VGX_ERR_INVALID, a),                  # out_id is an input
             ([a], _lib.VGX_ERR_INVALID, b),                  # out_id exists
             ([a, b], _lib.VGX_ERR_INVALID, out),             # voxel size differs
             ([a, c8], _lib.VGX_ERR_INVALID, out),            # voxels per side differ
             ([a, a], _lib.VGX_ERR_INVALID, out),             # repeated id
             ([], _lib.VGX_ERR_INVALID, out),                 # n < 1
             ([far], _lib.VGX_ERR_INVALID, out)]              # candidates beyond VGX_BLOCK_INDEX_MAX
    for ids, code, oid in cases:
        T = np.tile(shift if ids == [far] else IDENTITY, (len(ids), 1))
        with pytest.raises(api.VgxError) as e:
            ctx.project_map(ids, T, oid)
        assert e.value.code == code, (ids, oid, e.value)
        if oid == out:
            assert not exists(ctx, out)
    assert state() == before
    # an empty submap projects to an empty map
    e = next(_ids)
    ctx.submap_create(e, 0.1, 16, 8)
    assert ctx.project_map([e], IDENTITY[None], out) == 0
    assert ctx.submap_info(out)[2:] == (0, True)
    ctx.submap_free(out)
    for s in keep + [e]:
        ctx.submap_free(s)


def test_launch_count_and_determinism(ctx, oracle):
    layers, poses = _overlapping(0.2, 16, 4, seed=3)
    ids, got = _check(ctx, oracle, layers, poses)
    ctx.profile_reset()
    ctx.profile_enable(True)
    out = next(_ids)
    ctx.project_map(ids, poses, out)
    ms, launches = ctx.profile_get(_lib.VGX_SLOT_PROJECT)
    ctx.profile_enable(False)
    assert launches == LAUNCHES and ms > 0
    again = ctx.submap_download(out)
    for x, y in zip(got, again):
        assert x.tobytes() == y.tobytes()
    ctx.submap_free(out)
    for sid in ids:
        ctx.submap_free(sid)


def test_combined_mesh_equals_restatement(ctx, oracle):
    from voxgraph_b200 import api
    layers = [fx.layer((0.1, 16), "box", "sphere"), fx.layer((0.1, 16), "box", "tilted"),
              fx.layer((0.1, 16), "checker", "plane")]
    T = np.stack([yaw_T(0.0), yaw_T(0.4, (0.3, -0.2, 0.05)), yaw_T(-0.2, (-0.5, 0.4, 0.0))])
    ids = [next(_ids) for _ in layers]
    for sid, lay in zip(ids, layers):
        ctx.submap_upload(sid, *lay)
    idx, d, w = _oracle(oracle, layers, T, ids)
    for min_weight in (1.0, 2.0):
        xyz, tri = api.combined_mesh(ctx, ids, T, min_weight)
        ex, et = me.mesh(fx.Grid(0.1, 16, idx, d, w), min_weight)
        same_bits(ex, xyz, "combined vertices")
        same_bits(et.astype(np.uint32), tri, "combined triangles")
        assert len(tri) > 0
        assert not exists(ctx, SCRATCH_ID)   # the projection's scratch submap is freed again
    # the projected map it meshes is the restatement's layer
    out = next(_ids)
    ctx.project_map(ids, T, out)
    got = ctx.submap_download(out)
    ctx.submap_free(out)
    for x, y in zip((idx, d, w), got):
        assert np.asarray(x).tobytes() == y.tobytes()
    for sid in ids:
        ctx.submap_free(sid)


def test_projected_map_round_trips_and_finishes(ctx, oracle):
    layers, poses = _overlapping(0.2, 16, 3, seed=11)
    ids, got = _check(ctx, oracle, layers, poses)
    out = next(_ids)
    ctx.project_map(ids, poses, out)
    # the output is an ordinary finished submap: finishSubmap, the ESDF and the collection writer take it
    ctx.submap_finish_ex(out, ctx.registration_filter(min_voxel_weight=1e-6))
    assert ctx.submap_num_points(out, 1) > 0
    ctx.submap_generate_esdf(out)
    data = ctx.collection_save([out], IDENTITY[None])
    ctx.submap_free(out)
    assert ctx.collection_load(data) == 1
    back = ctx.submap_download(out)
    for x, y in zip(got, back):
        assert x.tobytes() == y.tobytes()
    ctx.submap_free(out)
    for sid in ids:
        ctx.submap_free(sid)


def test_mapper_save_combined_mesh(tmp_path):
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
    path = tmp_path / "combined.ply"
    size = m.saveCombinedMesh(str(path))
    data = path.read_bytes()
    assert size == len(data)
    ids = list(m.submap_ids)
    T = np.array([vm._pose4_to_T(m.submap_pose[i]) for i in ids], F32).reshape(-1, 7)
    ref = tmp_path / "ref.ply"
    api.save_combined_mesh(c, str(ref), ids, T, min_weight=cfg.mesh_min_weight)
    assert ref.read_bytes() == data
    xyz, rgba, tri = me.read_ply(data)
    assert len(tri) > 0 and (rgba == 255).all()
    ax, at = m.combinedMesh()
    same_bits(xyz, ax, "mapper combined mesh")
    c.close()
