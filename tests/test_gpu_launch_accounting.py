"""Launch accounting per entry point: on one context, every entry point that launches a kernel runs in the order
a user would call them, and after each call the total launch count (vgx_launch_count) and the launch count of
every profile slot (vgx_profile_get) must equal the table.  A slot counts the launches inside its profile scopes,
a cub sort counting as one; a launch outside every scope counts in the total only."""
import numpy as np
import pytest

from support import ctx, layer_stream  # noqa: F401
from voxgraph_b200 import _lib, api, synth

pytestmark = pytest.mark.gpu

# step -> (launches, {slot: launches} for the slots that counted any); slots: VgxProfileSlotId (voxgraph_b200.h)
EXPECTED = {
    'submap_upload': (4, {}),
    'submap_upload_points': (0, {}),
    'upload_synth_submap': (4, {}),
    'submap_create': (1, {}),
    'tsdf_mode0': (9, {2: 8, 3: 1}),
    'tsdf_mode0_colour': (9, {2: 8, 3: 1}),
    'submap_create_fast': (1, {}),
    'tsdf_mode1': (1, {2: 1}),
    'tsdf_mode1_colour': (1, {2: 1}),
    'tsdf_integrate_cloud': (10, {2: 8, 3: 1, 15: 1}),
    'cloud_decode': (10, {15: 10}),
    'submap_finish': (1, {}),
    'generate_esdf': (15, {}),
    'extract_points': (18, {}),
    'download_points': (1, {}),
    'submap_download': (1, {}),
    'graph_eval': (5, {0: 1, 6: 1, 7: 1, 8: 1}),
    'graph_solve': (56, {0: 6, 4: 31, 5: 1, 6: 6, 7: 6, 8: 6}),
    'edge_covariances': (8, {0: 1, 4: 4, 6: 1, 7: 1, 8: 1}),
    'mesh_build': (11, {12: 11}),
    'mesh_ply': (1, {12: 1}),
    'project_map': (18, {13: 15}),
    'submap_transform': (18, {13: 14, 14: 1}),
    'evaluate_layers_rmse': (2, {14: 2}),
    'layer_load': (4, {9: 1, 11: 2}),
    'map_evaluate': (110, {0: 1, 4: 1, 6: 1, 7: 1, 8: 1, 13: 29, 14: 3}),
    'submap_finish_ex': (19, {}),
    'find_overlapping_pairs': (1, {}),
    'collection_save': (6, {9: 6}),
    'collection_load': (8, {9: 2, 11: 4}),
}


def _steps(ctx):
    sc = synth.make_pair_scene(seed=1, n_points=1000)
    a, b = sc.submaps
    ids = [a.submap_id, b.submap_id]
    poses = np.stack([synth.pose_to_T(p) for p in sc.poses_init])
    world = synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)
    pts = synth.lidar_scan(world, np.array([15.0, 15.0, 1.2, 0.4]), n_beams=16, n_azimuth=256, seed=1)
    rgba = np.random.RandomState(0).randint(0, 256, (len(pts), 4)).astype(np.uint8)
    T = synth.pose_to_T([0.3, -0.2, 0.1, 0.4])
    T2 = synth.pose_to_T([0.5, 0.2, 0.1, 0.7])
    msg = synth.pack_pointcloud2(pts, rgba=rgba)
    mode0, mode1 = ctx.tsdf_config(mode=0), ctx.tsdf_config(mode=1)
    ACTIVE, FAST, PROJ, GT = 10, 11, 20, 30
    pg = api.PoseGraph(ctx)
    for i in range(2):
        pg.addSubmapNode(api.SubmapNodeConfig(ids[i], sc.poses_init[i], set_constant=(i == 0)))
    for (i, j, t, y) in sc.odometry:
        pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(i, j, np.array([*t, y]), sc.odom_information))
    pg.addRegistrationConstraint(api.RegistrationConstraintConfig(ids[0], ids[1]))
    store = {}

    def collection_load():
        for i in ids:
            ctx.submap_free(i)
        ctx.collection_load(store["collection"])

    return [
        ("submap_upload", lambda: ctx.submap_upload(a.submap_id, a.voxel_size, a.vps, a.block_idx, a.distance,
                                                    a.weight)),
        ("submap_upload_points", lambda: ctx.submap_upload_points(a.submap_id, api.K_ISOSURFACE_POINTS, a.points_xyz,
                                                                  a.points_distance, a.points_weight)),
        ("upload_synth_submap", lambda: ctx.upload_synth_submap(b)),
        ("submap_create", lambda: ctx.submap_create(ACTIVE, 0.2, 16, 4096)),
        ("tsdf_mode0", lambda: ctx.tsdf_integrate(ACTIVE, T, pts, mode0)),
        ("tsdf_mode0_colour", lambda: ctx.tsdf_integrate(ACTIVE, T2, pts, mode0, rgba)),
        ("submap_create_fast", lambda: ctx.submap_create(FAST, 0.2, 16, 4096)),
        ("tsdf_mode1", lambda: ctx.tsdf_integrate(FAST, T, pts, mode1)),
        ("tsdf_mode1_colour", lambda: ctx.tsdf_integrate(FAST, T2, pts, mode1, rgba)),
        ("tsdf_integrate_cloud", lambda: ctx.tsdf_integrate_cloud(ACTIVE, T, msg, mode0)),
        ("cloud_decode", lambda: ctx.cloud_decode(msg)),
        ("submap_finish", lambda: ctx.submap_finish(ACTIVE)),
        ("generate_esdf", lambda: ctx.submap_generate_esdf(ACTIVE)),
        ("extract_points", lambda: ctx.submap_extract_points(ACTIVE)),
        ("download_points", lambda: ctx.submap_download_points(ACTIVE, api.K_ISOSURFACE_POINTS)),
        ("submap_download", lambda: ctx.submap_download(ACTIVE)),
        ("graph_eval", lambda: pg.evaluate()),
        ("graph_solve", lambda: pg.optimize()),
        ("edge_covariances", lambda: pg.getEdgeCovarianceMap([tuple(ids)])),
        ("mesh_build", lambda: ctx.mesh_build([ACTIVE])),
        ("mesh_ply", lambda: ctx.mesh_ply()),
        ("project_map", lambda: ctx.project_map(ids, poses, PROJ)),
        ("submap_transform", lambda: ctx.submap_transform(PROJ, T)),
        ("evaluate_layers_rmse", lambda: ctx.evaluate_layers_rmse(ids[0], PROJ, _lib.VGX_LAYER_TSDF,
                                                                  _lib.VGX_LAYER_TSDF)),
        ("layer_load", lambda: ctx.layer_load(GT, layer_stream(a.voxel_size, a.vps, a.block_idx, a.distance,
                                                                 a.weight))),
        ("map_evaluate", lambda: ctx.map_evaluate(GT, ids, poses)),
        ("submap_finish_ex", lambda: ctx.submap_finish_ex(FAST)),
        ("find_overlapping_pairs", lambda: ctx.find_overlapping_pairs([ACTIVE, FAST], poses)),
        ("collection_save", lambda: store.update(collection=ctx.collection_save(ids, poses))),
        ("collection_load", collection_load),
    ]


def test_launch_accounting(ctx):
    got = {}
    for name, call in _steps(ctx):
        ctx.profile_reset()
        call()
        slots = {k: ctx.profile_get(k)[1] for k in range(_lib.VGX_PROFILE_SLOTS)}
        got[name] = (ctx.launch_count, {k: n for k, n in slots.items() if n})
    print("MEASURED = {\n" + "".join("    %r: %r,\n" % row for row in got.items()) + "}")
    assert list(got) == list(EXPECTED)
    bad = {name: (EXPECTED[name], row) for name, row in got.items() if row != EXPECTED[name]}
    assert not bad, bad
