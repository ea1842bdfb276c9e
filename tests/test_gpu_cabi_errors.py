"""Every C-ABI entry point that takes a context reports its own failure: one call per entry point (an unknown
submap id where the function takes one, otherwise one invalid argument) returns the status it has always
returned, and vgx_last_error names that function, never the failure planted on the context just before.  A
successful call leaves the message empty.  With two GPUs, a context on device 1 computes the same results
whichever device the calling thread has current."""
import ctypes as C

import numpy as np
import pytest

from voxgraph_b200 import _lib
from support import ctx  # noqa: F401

pytestmark = pytest.mark.gpu

U = 123456789   # a submap id no row creates
OK, INVALID, NOT_FOUND = _lib.VGX_OK, _lib.VGX_ERR_INVALID, _lib.VGX_ERR_NOT_FOUND


def _ids(*v):
    return (C.c_uint32 * len(v))(*v)


def _pose():
    return (C.c_float * 7)(1, 0, 0, 0, 0, 0, 0)


def _layout():
    """A valid empty point-cloud layout (no records)."""
    from voxgraph_b200 import api
    return api.CloudLayout(width=0, height=0, point_step=16, row_step=0, x_offset=0, y_offset=4, z_offset=8,
                           rgb_offset=-1, intensity_offset=-1)


# (entry point, arguments after the context, status at the parent of the guard)
ROWS = [
    ("vgx_ctx_synchronize", lambda: (), OK),
    ("vgx_profile_enable", lambda: (0,), OK),
    ("vgx_profile_reset", lambda: (), OK),
    ("vgx_profile_get", lambda: (-1, None, None), INVALID),
    ("vgx_submap_upload", lambda: (U, 0.1, 16, -1, None, None, None), INVALID),
    ("vgx_submap_create", lambda: (U, 0.1, 16, 0), INVALID),
    ("vgx_submap_finish", lambda: (U,), NOT_FOUND),
    ("vgx_submap_free", lambda: (U,), NOT_FOUND),
    ("vgx_submap_block_count", lambda: (U, C.byref(C.c_int())), NOT_FOUND),
    ("vgx_submap_download", lambda: (U, 0, None, None, None, None), NOT_FOUND),
    ("vgx_submap_upload_points", lambda: (U, 0, 0, None, None, None), NOT_FOUND),
    ("vgx_tsdf_integrate", lambda: (U, _pose(), 0, None, None, None, None), NOT_FOUND),
    ("vgx_tsdf_integrate_device", lambda: (U, _pose(), 0, None, None, None, None), NOT_FOUND),
    ("vgx_cloud_decode", lambda: (None, None, 0, 1.0, 0, None, None, None), INVALID),
    ("vgx_tsdf_integrate_cloud", lambda: (U, _pose(), C.byref(_layout()), None, 0, 0, 1.0, None, None, None),
     NOT_FOUND),
    ("vgx_reg_num_residuals", lambda: (U, C.byref(_lib.RegConfig(1, 0.0, -1.0, 0)), C.byref(C.c_int())), NOT_FOUND),
    ("vgx_reg_eval_emit", lambda: (U, U + 1, C.byref(_lib.RegConfig(1, 0.0, -1.0, 0)), (C.c_double * 4)(),
                                   (C.c_double * 4)(), (C.c_double * 4)(), None, None), NOT_FOUND),
    ("vgx_graph_set_nodes", lambda: (-1, None, None, None), INVALID),
    ("vgx_graph_set_poses", lambda: (None,), INVALID),
    ("vgx_graph_get_poses", lambda: (None,), INVALID),
    ("vgx_graph_set_relative_edges", lambda: (-1, None, None, None, None), INVALID),
    ("vgx_graph_set_registration_constraints", lambda: (-1, None, None, None), INVALID),
    ("vgx_graph_set_registration_constraints_v", lambda: (-1, None, None, None), INVALID),
    ("vgx_graph_num_registration_residuals", lambda: (None, None), INVALID),   # the graph has no nodes
    ("vgx_graph_eval", lambda: (0, None, None, None), INVALID),
    ("vgx_graph_eval_async", lambda: (0,), INVALID),
    ("vgx_graph_registration_costs", lambda: (None,), INVALID),
    ("vgx_graph_solve", lambda: (None, None, None), INVALID),
    ("vgx_graph_get_sample_indices", lambda: (0, 0, None, None), INVALID),
    ("vgx_graph_set_sample_indices", lambda: (-1, 0, None), INVALID),
    ("vgx_graph_edge_covariances", lambda: (-1, None, None, None), INVALID),
    ("vgx_comm_init", lambda: (0, 0, (C.c_uint8 * 128)()), INVALID),
    ("vgx_comm_destroy", lambda: (), OK),
    ("vgx_comm_p2p_export", lambda: (0, (C.c_uint8 * 64)()), INVALID),
    ("vgx_comm_p2p_import", lambda: (0, 0, (C.c_uint8 * 64)()), INVALID),
    ("vgx_comm_suspend", lambda: (0,), OK),
    ("vgx_submap_info", lambda: (U, None, None, None, None), NOT_FOUND),
    ("vgx_submap_draw_samples", lambda: (U, 0, 0, None), NOT_FOUND),
    ("vgx_submap_extract_points", lambda: (U, None), NOT_FOUND),
    ("vgx_submap_finish_ex", lambda: (U, None), NOT_FOUND),
    ("vgx_submap_num_points", lambda: (U, 0, C.byref(C.c_int())), NOT_FOUND),
    ("vgx_submap_download_points", lambda: (U, 0, 0, None, None, None, None), NOT_FOUND),
    ("vgx_submap_surface_obb", lambda: (U, (C.c_float * 3)(), (C.c_float * 3)()), NOT_FOUND),
    ("vgx_find_overlapping_pairs", lambda: (1, _ids(U), _pose(), 0, None, C.byref(C.c_int())), NOT_FOUND),
    ("vgx_submap_generate_esdf", lambda: (U, None, None), NOT_FOUND),
    ("vgx_submap_download_esdf", lambda: (U, 0, None, None, None), NOT_FOUND),
    ("vgx_submap_peek_device", lambda: (U, None, None, None), NOT_FOUND),
    ("vgx_submap_upload_device", lambda: (U, 0.1, 16, -1, None, None), INVALID),
    ("vgx_collection_load", lambda: (None, 5, C.byref(C.c_int())), INVALID),
    ("vgx_collection_load_ex", lambda: (None, 0, 2, C.byref(C.c_int())), INVALID),
    ("vgx_collection_save", lambda: (1, _ids(U), _pose(), None, 0, C.byref(C.c_uint64())), NOT_FOUND),
    ("vgx_mesh_build", lambda: (1, _ids(U), None, None, None, None), NOT_FOUND),
    ("vgx_mesh_download", lambda: (0, None, 0, None, None, None), OK),   # no mesh: nothing can be too small
    ("vgx_mesh_download_colours", lambda: (0, None, None), OK),
    ("vgx_mesh_ply", lambda: (None, None, 0, None), INVALID),
    ("vgx_mesh_ply_ex", lambda: (None, 0, None, 0, None), INVALID),
    ("vgx_project_map", lambda: (1, _ids(U), _pose(), U + 1, None), NOT_FOUND),
    ("vgx_mesh_build_combined", lambda: (1, _ids(U), _pose(), None), NOT_FOUND),
    ("vgx_layer_load", lambda: (U, None, 5, None), INVALID),
    ("vgx_submap_transform", lambda: (U, _pose()), NOT_FOUND),
    ("vgx_evaluate_layers_rmse", lambda: (U, 0, U + 1, 0, C.byref(_lib.VoxelEvaluationDetails())), NOT_FOUND),
    ("vgx_map_evaluate", lambda: (U, 1, _ids(U + 1), _pose(), C.byref(_lib.MapEvaluationResult())), NOT_FOUND),
    ("vgx_submap_has_colour", lambda: (U, C.byref(C.c_int())), NOT_FOUND),
    ("vgx_submap_download_colour", lambda: (U, 0, None, None), NOT_FOUND),
    ("vgx_submap_upload_colour", lambda: (U, 0, None), NOT_FOUND),
    ("vgx_submap_peek_device_colour", lambda: (U, C.byref(C.c_void_p())), NOT_FOUND),
    ("vgx_submap_upload_device_colour", lambda: (U, 0, None), NOT_FOUND),
]

CONTEXT_FREE = {"vgx_device_count", "vgx_ctx_create", "vgx_ctx_destroy", "vgx_collection_scan",
                "vgx_shard_constraints", "vgx_sqrt_information", "vgx_comm_unique_id"}
ACCESSORS = {"vgx_last_error", "vgx_ctx_stream", "vgx_launch_count"}


def test_every_context_entry_point_has_a_row():
    rows = [r[0] for r in ROWS]
    assert len(rows) == len(set(rows))
    expected = {n for n in _lib.EXPORTS if not n.endswith("_default")} - CONTEXT_FREE - ACCESSORS
    assert set(rows) == expected


@pytest.mark.parametrize("k", range(len(ROWS)), ids=[r[0] for r in ROWS])
def test_entry_point_reports_its_own_failure(ctx, k):  # noqa: F811
    L, h = _lib.load(), ctx._h
    name, args, status = ROWS[k]
    planted = 900000 + k   # a different failure before every row: an unknown submap of vgx_submap_info
    assert L.vgx_submap_info(h, planted, None, None, None, None) == NOT_FOUND
    before = L.vgx_last_error(h).decode()
    assert before.startswith("vgx_submap_info: ") and str(planted) in before
    rc = getattr(L, name)(h, *args())
    msg = L.vgx_last_error(h).decode()
    assert rc == status, (name, rc, msg)
    if status == OK:
        assert msg == "", (name, msg)
    else:
        assert msg.startswith(name + ": ") and msg != before and str(planted) not in msg, (name, msg)
    assert L.vgx_ctx_synchronize(h) == OK and L.vgx_last_error(h).decode() == ""


def _sequence(device):
    """create -> integrate -> finish -> extract -> eval -> solve -> mesh -> project on a context of `device`."""
    from voxgraph_b200 import api, synth
    c = api.Context(device)
    try:
        sc = synth.make_pair_scene(seed=3, n_points=1000)
        for s in sc.submaps:
            c.upload_synth_submap(s)
        s0 = sc.submaps[0]
        c.submap_create(7, s0.voxel_size, s0.vps, 4096)
        rng = np.random.default_rng(5)
        pts = rng.uniform(-4, 4, (20000, 3)).astype(np.float32)
        pts[:, 2] = np.float32(1.5)
        c.tsdf_integrate(7, [1, 0, 0, 0, 0, 0, 0], pts)
        c.submap_finish_ex(7)
        idx, d, w = c.submap_download(7)
        order = np.lexsort(idx.T[::-1])   # block slots follow the allocation order: compare by block index
        out = [idx[order], d[order], w[order], c.submap_num_points(7, 0), c.submap_num_points(7, 1)]
        ids = [s.submap_id for s in sc.submaps]
        c.graph_set_nodes(ids, np.array(sc.poses_init), [1, 0])
        c.graph_set_registration_constraints([ids[0], ids[1]], [ids[1], ids[0]])
        ok, cost, g, H = c.graph_eval(2)
        x, summary = c.graph_solve(2)
        out += [ok, cost, g, H, x, summary.iterations, summary.final_cost]
        vo, to = c.mesh_build(ids)
        out += [vo, to, *c.mesh_download()]
        T = np.array([[1, 0, 0, 0, 0, 0, 0]] * 2, np.float32)
        c.project_map(ids, T, 99)
        out += list(c.submap_download(99))
        return out
    finally:
        c.close()


def test_context_on_another_device_ignores_the_current_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    torch.cuda.set_device(1)
    ref = _sequence(1)
    torch.cuda.set_device(0)
    got = _sequence(1)
    assert len(ref) == len(got)
    for a, b in zip(ref, got):
        assert np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)
