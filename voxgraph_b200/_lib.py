"""ctypes binding of libvoxgraph_b200.so (the C-ABI in include/voxgraph_b200.h).

The product path has no CPU fallback: loading fails loudly when the CUDA extension has not
been built, and every compute entry point returns VGX_ERR_CUDA without a GPU.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libvoxgraph_b200.so")

VGX_OK = 0
VGX_ZERO_WEIGHT = 1
VGX_ERR_INVALID = -1
VGX_ERR_CUDA = -2
VGX_ERR_NOT_FOUND = -3
VGX_ERR_NOMEM = -4
VGX_ERR_NCCL = -5
VGX_ERR_CAPACITY = -6

# vgx_profile_get's `which` (enum VgxProfileSlotId)
VGX_SLOT_REG_REDUCE = 0
VGX_SLOT_REG_EMIT = 1
VGX_SLOT_TSDF_INTEGRATE = 2
VGX_SLOT_TSDF_ALLOCATE = 3
VGX_SLOT_SOLVE = 4
VGX_SLOT_OTHER = 5
VGX_SLOT_REG_POSE_SETUP = 6
VGX_SLOT_REG_SUMS = 7
VGX_SLOT_ASSEMBLY = 8
VGX_SLOT_COLL_CODEC = 9
VGX_SLOT_COLL_COPY = 10
VGX_SLOT_COLL_UPLOAD = 11
VGX_SLOT_MESH = 12
VGX_SLOT_PROJECT = 13
VGX_SLOT_EVAL = 14
VGX_SLOT_CLOUD_DECODE = 15
VGX_PROFILE_SLOTS = 16


class TsdfConfig(C.Structure):
    _fields_ = [("default_truncation_distance", C.c_float),
                ("max_weight", C.c_float),
                ("voxel_carving_enabled", C.c_int),
                ("min_ray_length_m", C.c_float),
                ("max_ray_length_m", C.c_float),
                ("use_const_weight", C.c_int),
                ("allow_clear", C.c_int),
                ("use_weight_dropoff", C.c_int),
                ("use_sparsity_compensation_factor", C.c_int),
                ("sparsity_compensation_factor", C.c_float),
                ("start_voxel_subsampling_factor", C.c_float),
                ("max_consecutive_ray_collisions", C.c_int),
                ("mode", C.c_int),
                ("deterministic", C.c_int)]


class TsdfStats(C.Structure):
    _fields_ = [("rays_valid", C.c_int64), ("rays_cast", C.c_int64),
                ("voxel_updates", C.c_int64), ("blocks_allocated", C.c_int64),
                ("saturated_batches", C.c_int64)]


class RegistrationFilter(C.Structure):
    _fields_ = [("min_voxel_weight", C.c_double), ("max_voxel_distance", C.c_double),
                ("use_esdf_distance", C.c_int)]


class RegConfig(C.Structure):
    _fields_ = [("registration_point_type", C.c_int),
                ("no_correspondence_cost", C.c_double),
                ("sampling_ratio", C.c_float),
                ("use_esdf_distance", C.c_int)]


class EsdfConfig(C.Structure):
    _fields_ = [("max_distance_m", C.c_float), ("default_distance_m", C.c_float),
                ("min_distance_m", C.c_float), ("min_weight", C.c_float)]


class SolverOptions(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int),
                ("parameter_tolerance", C.c_double),
                ("function_tolerance", C.c_double),
                ("gradient_tolerance", C.c_double),
                ("initial_trust_region_radius", C.c_double),
                ("max_trust_region_radius", C.c_double),
                ("min_trust_region_radius", C.c_double),
                ("min_relative_decrease", C.c_double),
                ("min_lm_diagonal", C.c_double),
                ("max_lm_diagonal", C.c_double),
                ("max_solver_time_s", C.c_double),
                ("jacobi_scaling", C.c_int),
                ("exclude_registration", C.c_int)]


class SolverSummary(C.Structure):
    _fields_ = [("iterations", C.c_int),
                ("num_successful_steps", C.c_int),
                ("num_residual_evals", C.c_int),
                ("termination", C.c_int),
                ("initial_cost", C.c_double),
                ("final_cost", C.c_double),
                ("total_time_s", C.c_double)]


class CollectionEntry(C.Structure):
    _fields_ = [("id", C.c_uint32), ("num_blocks", C.c_uint32), ("voxel_size", C.c_float),
                ("voxels_per_side", C.c_int32), ("T_M_S", C.c_float * 7)]


class MeshConfig(C.Structure):
    _fields_ = [("min_weight", C.c_float)]


VGX_COLLECTION_KEEP_COLOUR = 1   # vgx_collection_load_ex flag

VGX_LAYER_TSDF = 0
VGX_LAYER_ESDF = 1


class VoxelEvaluationDetails(C.Structure):
    _fields_ = [("rmse", C.c_float), ("max_error", C.c_float), ("min_error", C.c_float), ("pad", C.c_float),
                ("num_evaluated_voxels", C.c_uint64), ("num_ignored_voxels", C.c_uint64),
                ("num_overlapping_voxels", C.c_uint64), ("num_non_overlapping_voxels", C.c_uint64)]


class MapEvaluationResult(C.Structure):
    _fields_ = [("details", VoxelEvaluationDetails),
                ("aligned_pose", C.c_double * 4),
                ("T_projected_map__ground_truth", C.c_float * 7),
                ("T_ground_truth__reading", C.c_float * 7),
                ("summary", SolverSummary)]


class CloudLayout(C.Structure):
    """vgx_cloud_layout: the part of a PointCloud2 that pcl::fromROSMsg reads."""
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("point_step", C.c_uint32),
                ("row_step", C.c_uint32), ("x_offset", C.c_int32), ("y_offset", C.c_int32),
                ("z_offset", C.c_int32), ("rgb_offset", C.c_int32), ("intensity_offset", C.c_int32)]


_P = C.POINTER
_vp, _i32, _u32, _i64, _u64, _f32 = C.c_void_p, C.c_int, C.c_uint32, C.c_int64, C.c_uint64, C.c_float
_pi32, _pu32, _pi64, _pu64, _pu8 = _P(C.c_int32), _P(C.c_uint32), _P(C.c_int64), _P(C.c_uint64), _P(C.c_uint8)
_pf, _pd = _P(C.c_float), _P(C.c_double)

# (restype, argtypes) of every function include/voxgraph_b200.h declares, in the header's order.  c_void_p stands
# only for the opaque vgx_ctx*, a byte stream passed as bytes or a c_char array, or a device address;
# tests/test_host_binding_signatures.py compares every entry with the header's prototype.
SIGNATURES = {
    # context
    "vgx_device_count": (_i32, []),
    "vgx_ctx_create": (_i32, [_i32, _P(_vp)]),
    "vgx_ctx_destroy": (None, [_vp]),
    "vgx_last_error": (C.c_char_p, [_vp]),
    "vgx_ctx_stream": (_vp, [_vp]),
    "vgx_ctx_synchronize": (_i32, [_vp]),
    "vgx_profile_enable": (_i32, [_vp, _i32]),
    "vgx_profile_reset": (_i32, [_vp]),
    "vgx_profile_get": (_i32, [_vp, _i32, _pd, _pi64]),
    "vgx_launch_count": (_i64, [_vp]),
    # submaps
    "vgx_submap_upload": (_i32, [_vp, _u32, _f32, _i32, _i32, _pi32, _pf, _pf]),
    "vgx_submap_create": (_i32, [_vp, _u32, _f32, _i32, _i32]),
    "vgx_submap_finish": (_i32, [_vp, _u32]),
    "vgx_registration_filter_default": (None, [_P(RegistrationFilter)]),
    "vgx_submap_extract_points": (_i32, [_vp, _u32, _P(RegistrationFilter)]),
    "vgx_submap_finish_ex": (_i32, [_vp, _u32, _P(RegistrationFilter)]),
    "vgx_submap_num_points": (_i32, [_vp, _u32, _i32, _pi32]),
    "vgx_submap_download_points": (_i32, [_vp, _u32, _i32, _i32, _pf, _pf, _pf, _pi32]),
    "vgx_submap_surface_obb": (_i32, [_vp, _u32, _pf, _pf]),
    "vgx_esdf_config_default": (None, [_P(EsdfConfig)]),
    "vgx_submap_generate_esdf": (_i32, [_vp, _u32, _P(EsdfConfig), _pi32]),
    "vgx_submap_download_esdf": (_i32, [_vp, _u32, _i32, _pf, _pf, _pi32]),
    "vgx_find_overlapping_pairs": (_i32, [_vp, _i32, _pu32, _pf, _i32, _pu32, _pi32]),
    "vgx_submap_free": (_i32, [_vp, _u32]),
    "vgx_submap_block_count": (_i32, [_vp, _u32, _pi32]),
    "vgx_submap_info": (_i32, [_vp, _u32, _pf, _pi32, _pi32, _pi32]),
    "vgx_submap_download": (_i32, [_vp, _u32, _i32, _pi32, _pf, _pf, _pi32]),
    "vgx_submap_peek_device": (_i32, [_vp, _u32, _P(_vp), _P(_vp), _pi32]),
    "vgx_submap_upload_device": (_i32, [_vp, _u32, _f32, _i32, _i32, _vp, _vp]),
    "vgx_submap_has_colour": (_i32, [_vp, _u32, _pi32]),
    "vgx_submap_download_colour": (_i32, [_vp, _u32, _i32, _pu32, _pi32]),
    "vgx_submap_upload_colour": (_i32, [_vp, _u32, _i32, _pu32]),
    "vgx_submap_peek_device_colour": (_i32, [_vp, _u32, _P(_vp)]),
    "vgx_submap_upload_device_colour": (_i32, [_vp, _u32, _i32, _vp]),
    # submap collection files
    "vgx_collection_scan": (_i32, [_vp, _u64, _i32, _P(CollectionEntry), _pi32]),
    "vgx_collection_load": (_i32, [_vp, _vp, _u64, _pi32]),
    "vgx_collection_load_ex": (_i32, [_vp, _vp, _u64, _i32, _pi32]),
    "vgx_collection_save": (_i32, [_vp, _i32, _pu32, _pf, _vp, _u64, _pu64]),
    # submap meshes
    "vgx_mesh_config_default": (None, [_P(MeshConfig)]),
    "vgx_mesh_build": (_i32, [_vp, _i32, _pu32, _pf, _P(MeshConfig), _pi64, _pi64]),
    "vgx_mesh_download": (_i32, [_vp, _i64, _pf, _i64, _pu32, _pi64, _pi64]),
    "vgx_mesh_ply": (_i32, [_vp, _pu8, _vp, _u64, _pu64]),
    "vgx_mesh_download_colours": (_i32, [_vp, _i64, _pu32, _pi64]),
    "vgx_mesh_ply_ex": (_i32, [_vp, _pu8, _i32, _vp, _u64, _pu64]),
    # projected global map, registration points
    "vgx_project_map": (_i32, [_vp, _i32, _pu32, _pf, _u32, _pi32]),
    "vgx_mesh_build_combined": (_i32, [_vp, _i32, _pu32, _pf, _P(MeshConfig)]),
    "vgx_submap_upload_points": (_i32, [_vp, _u32, _i32, _i32, _pf, _pf, _pf]),
    # b3: TSDF integration, point-cloud messages
    "vgx_tsdf_config_default": (None, [_P(TsdfConfig)]),
    "vgx_tsdf_integrate": (_i32, [_vp, _u32, _pf, _i32, _pf, _pu8, _P(TsdfConfig), _P(TsdfStats)]),
    "vgx_tsdf_integrate_device": (_i32, [_vp, _u32, _pf, _i32, _vp, _vp, _P(TsdfConfig), _P(TsdfStats)]),
    "vgx_cloud_decode": (_i32, [_vp, _P(CloudLayout), _vp, _u64, _f32, _i32, _pf, _pu8, _pi32]),
    "vgx_tsdf_integrate_cloud": (_i32, [_vp, _u32, _pf, _P(CloudLayout), _vp, _u64, _i32, _f32, _P(TsdfConfig),
                                        _P(TsdfStats), _pi32]),
    # b1: cost function
    "vgx_reg_config_default": (None, [_P(RegConfig)]),
    "vgx_reg_num_residuals": (_i32, [_vp, _u32, _P(RegConfig), _pi32]),
    "vgx_reg_eval_emit": (_i32, [_vp, _u32, _u32, _P(RegConfig), _pd, _pd, _pd, _pd, _pd]),
    "vgx_submap_draw_samples": (_i32, [_vp, _u32, _i32, _i32, _pi32]),
    # b2: pose graph
    "vgx_graph_set_nodes": (_i32, [_vp, _i32, _pu32, _pd, _pu8]),
    "vgx_graph_set_poses": (_i32, [_vp, _pd]),
    "vgx_graph_get_poses": (_i32, [_vp, _pd]),
    "vgx_graph_set_relative_edges": (_i32, [_vp, _i32, _pu32, _pu32, _pd, _pd]),
    "vgx_sqrt_information": (_i32, [_pd, _i32, _pd]),
    "vgx_graph_set_registration_constraints": (_i32, [_vp, _i32, _pu32, _pu32, _P(RegConfig)]),
    "vgx_graph_set_registration_constraints_v": (_i32, [_vp, _i32, _pu32, _pu32, _P(RegConfig)]),
    "vgx_graph_get_sample_indices": (_i32, [_vp, _i32, _i32, _pi32, _pi32]),
    "vgx_graph_set_sample_indices": (_i32, [_vp, _i32, _i32, _pi32]),
    "vgx_graph_num_registration_residuals": (_i32, [_vp, _pi64, _pi64]),
    "vgx_graph_eval": (_i32, [_vp, _i32, _pd, _pd, _pd]),
    "vgx_graph_eval_async": (_i32, [_vp, _i32]),
    "vgx_graph_registration_costs": (_i32, [_vp, _pd]),
    "vgx_solver_options_default": (None, [_P(SolverOptions)]),
    "vgx_graph_solve": (_i32, [_vp, _P(SolverOptions), _pd, _P(SolverSummary)]),
    "vgx_graph_edge_covariances": (_i32, [_vp, _i32, _pu32, _pu32, _pd]),
    # map evaluation
    "vgx_layer_load": (_i32, [_vp, _u32, _vp, _u64, _pi32]),
    "vgx_submap_transform": (_i32, [_vp, _u32, _pf]),
    "vgx_evaluate_layers_rmse": (_i32, [_vp, _u32, _i32, _u32, _i32, _P(VoxelEvaluationDetails)]),
    "vgx_map_evaluate": (_i32, [_vp, _u32, _i32, _pu32, _pf, _P(MapEvaluationResult)]),
    # multi-GPU
    "vgx_shard_constraints": (_i32, [_i32, _i32, _pi32, _pu32, _pi32]),
    "vgx_comm_unique_id": (_i32, [_pu8]),
    "vgx_comm_init": (_i32, [_vp, _i32, _i32, _pu8]),
    "vgx_comm_destroy": (_i32, [_vp]),
    "vgx_comm_suspend": (_i32, [_vp, _i32]),
    "vgx_comm_p2p_export": (_i32, [_vp, _u64, _pu8]),
    "vgx_comm_p2p_import": (_i32, [_vp, _i32, _i32, _pu8]),
}
EXPORTS = list(SIGNATURES)

_lib = None


def load():
    """Load the CUDA extension; raise if it has not been built (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "voxgraph_b200: CUDA extension %s is missing - run `python -m voxgraph_b200.build` "
            "(or __graft_entry__.build()); there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L
