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
VGX_PROFILE_SLOTS = 15


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


# every symbol include/voxgraph_b200.h declares
EXPORTS = [
    "vgx_device_count", "vgx_ctx_create", "vgx_ctx_destroy", "vgx_last_error", "vgx_ctx_stream",
    "vgx_ctx_synchronize", "vgx_profile_enable", "vgx_profile_reset", "vgx_profile_get",
    "vgx_launch_count", "vgx_submap_upload", "vgx_submap_create", "vgx_submap_finish",
    "vgx_submap_free", "vgx_submap_block_count", "vgx_submap_download", "vgx_submap_upload_points",
    "vgx_tsdf_config_default", "vgx_tsdf_integrate", "vgx_reg_config_default",
    "vgx_reg_num_residuals", "vgx_reg_eval_emit", "vgx_graph_set_nodes", "vgx_graph_set_poses",
    "vgx_graph_get_poses", "vgx_graph_set_relative_edges",
    "vgx_graph_set_registration_constraints", "vgx_graph_num_registration_residuals",
    "vgx_graph_eval", "vgx_graph_eval_async", "vgx_graph_registration_costs",
    "vgx_solver_options_default", "vgx_graph_solve", "vgx_shard_constraints", "vgx_comm_unique_id",
    "vgx_comm_init",
    "vgx_comm_destroy", "vgx_comm_p2p_export", "vgx_comm_p2p_import",
    "vgx_submap_info", "vgx_submap_draw_samples", "vgx_graph_set_registration_constraints_v",
    "vgx_graph_get_sample_indices", "vgx_graph_set_sample_indices", "vgx_comm_suspend",
    "vgx_registration_filter_default", "vgx_submap_extract_points", "vgx_submap_finish_ex",
    "vgx_submap_num_points", "vgx_submap_download_points", "vgx_submap_surface_obb",
    "vgx_find_overlapping_pairs", "vgx_esdf_config_default", "vgx_submap_generate_esdf",
    "vgx_submap_download_esdf", "vgx_graph_edge_covariances", "vgx_submap_peek_device",
    "vgx_submap_upload_device", "vgx_collection_scan", "vgx_collection_load", "vgx_collection_save",
    "vgx_mesh_config_default", "vgx_mesh_build", "vgx_mesh_download", "vgx_mesh_ply", "vgx_project_map",
    "vgx_layer_load", "vgx_submap_transform", "vgx_evaluate_layers_rmse", "vgx_map_evaluate",
]

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
    vp = C.c_void_p
    u32, i32 = C.c_uint32, C.c_int
    pu32, pi32 = C.POINTER(C.c_uint32), C.POINTER(C.c_int32)
    pf, pd, pu8 = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_uint8)
    L.vgx_device_count.restype = i32
    L.vgx_ctx_create.argtypes = [i32, C.POINTER(vp)]
    L.vgx_ctx_destroy.argtypes = [vp]
    L.vgx_ctx_destroy.restype = None
    L.vgx_last_error.argtypes = [vp]
    L.vgx_last_error.restype = C.c_char_p
    L.vgx_ctx_stream.argtypes = [vp]
    L.vgx_ctx_stream.restype = vp
    L.vgx_ctx_synchronize.argtypes = [vp]
    L.vgx_profile_enable.argtypes = [vp, i32]
    L.vgx_profile_reset.argtypes = [vp]
    L.vgx_profile_get.argtypes = [vp, i32, pd, C.POINTER(C.c_int64)]
    L.vgx_launch_count.argtypes = [vp]
    L.vgx_launch_count.restype = C.c_int64
    L.vgx_submap_upload.argtypes = [vp, u32, C.c_float, i32, i32, pi32, pf, pf]
    L.vgx_submap_create.argtypes = [vp, u32, C.c_float, i32, i32]
    L.vgx_submap_finish.argtypes = [vp, u32]
    L.vgx_submap_free.argtypes = [vp, u32]
    L.vgx_submap_block_count.argtypes = [vp, u32, C.POINTER(i32)]
    L.vgx_submap_download.argtypes = [vp, u32, i32, pi32, pf, pf, C.POINTER(i32)]
    L.vgx_submap_upload_points.argtypes = [vp, u32, i32, i32, pf, pf, pf]
    L.vgx_tsdf_config_default.argtypes = [C.POINTER(TsdfConfig)]
    L.vgx_tsdf_config_default.restype = None
    L.vgx_tsdf_integrate.argtypes = [vp, u32, pf, i32, pf, pu8, C.POINTER(TsdfConfig),
                                     C.POINTER(TsdfStats)]
    L.vgx_reg_config_default.argtypes = [C.POINTER(RegConfig)]
    L.vgx_reg_config_default.restype = None
    L.vgx_reg_num_residuals.argtypes = [vp, u32, C.POINTER(RegConfig), C.POINTER(i32)]
    L.vgx_reg_eval_emit.argtypes = [vp, u32, u32, C.POINTER(RegConfig), pd, pd, pd, pd, pd]
    L.vgx_graph_set_nodes.argtypes = [vp, i32, pu32, pd, pu8]
    L.vgx_graph_set_poses.argtypes = [vp, pd]
    L.vgx_graph_get_poses.argtypes = [vp, pd]
    L.vgx_graph_set_relative_edges.argtypes = [vp, i32, pu32, pu32, pd, pd]
    L.vgx_graph_set_registration_constraints.argtypes = [vp, i32, pu32, pu32, C.POINTER(RegConfig)]
    L.vgx_graph_set_registration_constraints_v.argtypes = [vp, i32, pu32, pu32, C.POINTER(RegConfig)]
    L.vgx_graph_get_sample_indices.argtypes = [vp, i32, i32, pi32, C.POINTER(i32)]
    L.vgx_graph_set_sample_indices.argtypes = [vp, i32, i32, pi32]
    L.vgx_registration_filter_default.argtypes = [C.POINTER(RegistrationFilter)]
    L.vgx_registration_filter_default.restype = None
    L.vgx_submap_extract_points.argtypes = [vp, u32, C.POINTER(RegistrationFilter)]
    L.vgx_submap_finish_ex.argtypes = [vp, u32, C.POINTER(RegistrationFilter)]
    L.vgx_submap_num_points.argtypes = [vp, u32, i32, C.POINTER(i32)]
    L.vgx_submap_download_points.argtypes = [vp, u32, i32, i32, pf, pf, pf, C.POINTER(i32)]
    L.vgx_submap_surface_obb.argtypes = [vp, u32, pf, pf]
    L.vgx_find_overlapping_pairs.argtypes = [vp, i32, pu32, pf, i32, pu32, C.POINTER(i32)]
    L.vgx_esdf_config_default.argtypes = [C.POINTER(EsdfConfig)]
    L.vgx_esdf_config_default.restype = None
    L.vgx_submap_generate_esdf.argtypes = [vp, u32, C.POINTER(EsdfConfig), C.POINTER(i32)]
    L.vgx_submap_download_esdf.argtypes = [vp, u32, i32, pf, pf, C.POINTER(i32)]
    L.vgx_graph_edge_covariances.argtypes = [vp, i32, pu32, pu32, pd]
    L.vgx_submap_peek_device.argtypes = [vp, u32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(i32)]
    L.vgx_submap_upload_device.argtypes = [vp, u32, C.c_float, i32, i32, C.c_void_p, C.c_void_p]
    L.vgx_collection_scan.argtypes = [C.c_void_p, C.c_uint64, i32, C.POINTER(CollectionEntry), C.POINTER(i32)]
    L.vgx_collection_load.argtypes = [vp, C.c_void_p, C.c_uint64, C.POINTER(i32)]
    L.vgx_collection_save.argtypes = [vp, i32, pu32, pf, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.vgx_mesh_config_default.argtypes = [C.POINTER(MeshConfig)]
    L.vgx_mesh_config_default.restype = None
    pi64 = C.POINTER(C.c_int64)
    L.vgx_mesh_build.argtypes = [vp, i32, pu32, pf, C.POINTER(MeshConfig), pi64, pi64]
    L.vgx_mesh_download.argtypes = [vp, C.c_int64, pf, C.c_int64, pu32, pi64, pi64]
    L.vgx_mesh_ply.argtypes = [vp, pu8, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.vgx_project_map.argtypes = [vp, i32, pu32, pf, u32, C.POINTER(i32)]
    L.vgx_layer_load.argtypes = [vp, u32, C.c_void_p, C.c_uint64, C.POINTER(i32)]
    L.vgx_submap_transform.argtypes = [vp, u32, pf]
    L.vgx_evaluate_layers_rmse.argtypes = [vp, u32, i32, u32, i32, C.POINTER(VoxelEvaluationDetails)]
    L.vgx_map_evaluate.argtypes = [vp, u32, i32, pu32, pf, C.POINTER(MapEvaluationResult)]
    L.vgx_submap_info.argtypes = [vp, u32, pf, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.vgx_submap_draw_samples.argtypes = [vp, u32, i32, i32, pi32]
    L.vgx_graph_num_registration_residuals.argtypes = [vp, C.POINTER(C.c_int64),
                                                       C.POINTER(C.c_int64)]
    L.vgx_graph_eval.argtypes = [vp, i32, pd, pd, pd]
    L.vgx_graph_eval_async.argtypes = [vp, i32]
    L.vgx_graph_registration_costs.argtypes = [vp, pd]
    L.vgx_solver_options_default.argtypes = [C.POINTER(SolverOptions)]
    L.vgx_solver_options_default.restype = None
    L.vgx_graph_solve.argtypes = [vp, C.POINTER(SolverOptions), pd, C.POINTER(SolverSummary)]
    L.vgx_shard_constraints.argtypes = [i32, i32, pi32, pu32, pi32]
    L.vgx_comm_unique_id.argtypes = [pu8]
    L.vgx_comm_init.argtypes = [vp, i32, i32, pu8]
    L.vgx_comm_destroy.argtypes = [vp]
    L.vgx_comm_suspend.argtypes = [vp, i32]
    L.vgx_comm_p2p_export.argtypes = [vp, C.c_uint64, pu8]
    L.vgx_comm_p2p_import.argtypes = [vp, i32, i32, pu8]
    _lib = L
    return L
