"""ctypes loader of the C-ABI library (include/b200reg.h). There is no fallback: if the CUDA library is missing
or cannot be loaded this module raises, and every compute call goes through sm_90a kernels."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(_HERE)
LIB_PATH = os.path.join(_HERE, "csrc", "libb200reg.so")

OK, ERR_ARG, ERR_NO_TARGET, ERR_NO_SOURCE, ERR_CUDA, ERR_TIMEOUT, ERR_GRID, ERR_IO, ERR_FORMAT = 0, -1, -2, -3, -4, -5, -6, -7, -8
PCD_LOAD_PIECE_BYTES = 64 << 20  # B200REG_PCD_LOAD_PIECE_BYTES
NDT, GICP = 0, 1
KDTREE, DIRECT26, DIRECT7, DIRECT1 = 0, 1, 2, 3

# every symbol include/b200reg.h declares
SYMBOLS = [
    "b200reg_create", "b200reg_destroy", "b200reg_last_error",
    "b200reg_set_transformation_epsilon", "b200reg_set_maximum_iterations",
    "b200reg_set_max_correspondence_distance", "b200reg_set_euclidean_fitness_epsilon",
    "b200reg_set_ransac_iterations",
    "b200reg_ndt_set_resolution", "b200reg_ndt_set_step_size", "b200reg_ndt_set_outlier_ratio",
    "b200reg_ndt_set_neighborhood_search_method", "b200reg_ndt_set_num_threads",
    "b200reg_ndt_get_transformation_probability", "b200reg_ndt_get_final_num_iteration",
    "b200reg_ndt_calculate_score",
    "b200reg_gicp_set_rotation_epsilon", "b200reg_gicp_set_correspondence_randomness",
    "b200reg_gicp_set_maximum_optimizer_iterations", "b200reg_gicp_set_epsilon",
    "b200reg_set_input_target", "b200reg_set_input_source",
    "b200reg_set_input_target_device", "b200reg_set_input_source_device",
    "b200reg_align", "b200reg_get_final_transformation", "b200reg_has_converged",
    "b200reg_get_fitness_score", "b200reg_get_aligned", "b200reg_align_batch",
    "b200reg_ndt_align_batch", "b200reg_ndt_align_batch_device", "b200reg_ndt_set_batch_slots", "b200reg_ndt_sweep",
    "b200reg_ndt_attach_pose_board", "b200reg_ndt_gathered_poses",
    "b200reg_voxelgrid", "b200reg_get_stats", "b200reg_ndt_derivatives", "b200reg_ndt_hessian_radius",
    "b200reg_ndt_num_voxels", "b200reg_ndt_get_voxels", "b200reg_nn1",
    "b200reg_gicp_get_covariances", "b200reg_gicp_num_correspondences", "b200reg_gicp_correspondences",
    "b200reg_gicp_objective", "b200reg_ndt_set_trace", "b200reg_ndt_get_trace", "b200reg_gicp_set_trace",
    "b200reg_gicp_get_trace", "b200reg_get_kind",
    "b200sm_create", "b200sm_destroy", "b200sm_last_error", "b200sm_set_params", "b200sm_set_initial_pose",
    "b200sm_set_scan", "b200sm_update_map", "b200sm_receive_cloud", "b200sm_num_submaps", "b200sm_get_targeted",
    "b200sm_get_submap", "b200sm_get_filtered_scan", "b200sm_get_stats", "b200sm_search_loop", "b200sm_search_loop_all", "b200sm_import_submap",
    "b200sm_imu_set_scan_period", "b200sm_imu_push", "b200sm_deskew_next_scan", "b200sm_imu_adjust_distortion",
    "b200sm_imu_get_state", "b200sm_imu_get_sample", "b200sm_imu_get_trace", "b200sm_pose_adjust", "b200sm_assemble_map",
    "b200sm_save_map_pcd_ascii", "b200reg_encode_pcd_ascii", "b200sm_set_sensor_transform", "b200sm_odom_next_scan",
    "b200reg_load_pcd", "b200reg_set_input_target_pcd",
    "b200sm_set_prior_map_pcd", "b200sm_set_prior_map", "b200sm_set_localization_params", "b200sm_localize_cloud",
    "b200sm_localize_init", "b200sm_get_localize_stats", "b200sm_get_cut", "b200reg_ndt_score_poses",
    "b200sm_localize_global", "b200sm_get_global_search",
    "b200sm_relocalize", "b200sm_get_relocalize_grid", "b200sm_relocalize_score_nodes",
    "b200sm_set_scan_context_params", "b200sm_get_scan_context", "b200sm_search_loop_place", "b200sm_get_place_scores",
    "b200sm_build_occupancy_grid", "b200sm_get_occupancy_grid", "b200sm_save_occupancy_map",
    "b200sm_build_elevation_map", "b200sm_get_elevation_map", "b200sm_save_traversability_map",
    "b200sm_build_static_map", "b200sm_get_static_map", "b200sm_get_map_voxels", "b200sm_save_static_map_pcd_ascii",
    "b200sm_build_map_consistency", "b200sm_get_map_consistency", "b200sm_get_submap_consistency",
    "b200sm_save_map_consistency_pcd_ascii",
    "b200sm_build_map_changes", "b200sm_get_map_changes", "b200sm_get_change_voxels", "b200sm_get_updated_map",
    "b200sm_save_updated_map_pcd_ascii",
    "b200sm_build_mesh", "b200sm_get_mesh", "b200sm_get_mesh_voxels", "b200sm_save_mesh_ply",
    "b200sm_build_octomap", "b200sm_get_octomap_states", "b200sm_get_octomap_bt", "b200sm_save_octomap_bt",
    "b200sm_merge_session", "b200sm_get_merge_scores", "b200sm_get_segments",
    "b200sm_save_session", "b200sm_load_session", "b200sm_get_session_graph",
    # include/b200comm.h
    "b200comm_unique_id", "b200comm_create", "b200comm_destroy", "b200comm_all_gather_rows", "b200comm_rank", "b200comm_last_error",
    "b200comm_board_create", "b200comm_board_destroy", "b200comm_board_info",
]


class SmLoopResult(C.Structure):
    _fields_ = [("is_candidate", C.c_int), ("id_min", C.c_int), ("accepted", C.c_int), ("pad", C.c_int),
                ("min_dist", C.c_double), ("fitness", C.c_double), ("final_T", C.c_float * 16),
                ("relative_pose", C.c_double * 16), ("n_source", C.c_size_t), ("n_target", C.c_size_t)]


class SmScanContextParams(C.Structure):
    _fields_ = [("num_rings", C.c_int), ("num_sectors", C.c_int), ("max_radius", C.c_double), ("lidar_height", C.c_double)]


class SmPlaceResult(C.Structure):
    _fields_ = [("loop", SmLoopResult), ("sc_distance", C.c_double), ("shift", C.c_int), ("pad", C.c_int),
                ("guess", C.c_float * 16)]


class SmOccupancyParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("z_min", C.c_double), ("z_max", C.c_double), ("max_range", C.c_double),
                ("sensor_origin", C.c_double * 3), ("occupied_thresh", C.c_double), ("free_thresh", C.c_double)]


class SmOccupancyInfo(C.Structure):
    _fields_ = [("width", C.c_uint), ("height", C.c_uint), ("origin", C.c_double * 2), ("resolution", C.c_double),
                ("n_rays", C.c_ulonglong), ("n_skipped", C.c_ulonglong), ("n_batches", C.c_int), ("n_occupied", C.c_ulonglong),
                ("n_free", C.c_ulonglong), ("n_unknown", C.c_ulonglong)]


class SmElevationParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("max_range", C.c_double), ("sensor_origin", C.c_double * 3),
                ("clearance", C.c_double), ("min_points", C.c_int), ("window_cells", C.c_int), ("min_cells", C.c_int),
                ("max_slope", C.c_double), ("max_step", C.c_double), ("max_roughness", C.c_double),
                ("occupied_thresh", C.c_double), ("free_thresh", C.c_double)]


class SmElevationInfo(C.Structure):
    _fields_ = [("width", C.c_uint), ("height", C.c_uint), ("origin", C.c_double * 2), ("resolution", C.c_double),
                ("n_points", C.c_ulonglong), ("n_skipped", C.c_ulonglong), ("n_overhang", C.c_ulonglong),
                ("n_observed", C.c_ulonglong), ("n_lethal", C.c_ulonglong), ("n_traversable", C.c_ulonglong),
                ("n_unknown", C.c_ulonglong)]


class SmStaticMapParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("max_range", C.c_double), ("sensor_origin", C.c_double * 3),
                ("ray_fraction", C.c_double), ("min_frees", C.c_uint), ("dynamic_thresh", C.c_double)]


class SmMapConsistencyParams(C.Structure):
    _fields_ = [("radius", C.c_double), ("min_neighbors", C.c_int), ("query_stride", C.c_int)]


class SmMapConsistencyInfo(C.Structure):
    _fields_ = [("box_origin", C.c_int * 3), ("box_dims", C.c_uint * 3), ("n_points", C.c_ulonglong), ("n_skipped", C.c_ulonglong),
                ("n_cells", C.c_ulonglong), ("n_queries", C.c_ulonglong), ("n_valid", C.c_ulonglong),
                ("n_neighbors", C.c_ulonglong), ("n_candidates", C.c_ulonglong), ("sum_h_q", C.c_longlong),
                ("sum_plane_q", C.c_longlong), ("mme", C.c_double), ("mpv", C.c_double)]


class SmSubmapConsistency(C.Structure):
    _fields_ = [("n_points", C.c_ulonglong), ("n_queries", C.c_ulonglong), ("n_valid", C.c_ulonglong),
                ("n_neighbors", C.c_ulonglong), ("sum_h_q", C.c_longlong), ("sum_plane_q", C.c_longlong), ("mme", C.c_double),
                ("mpv", C.c_double)]


class SmStaticMapInfo(C.Structure):
    _fields_ = [("box_origin", C.c_int * 3), ("box_dims", C.c_uint * 3), ("n_rays", C.c_ulonglong), ("n_skipped", C.c_ulonglong),
                ("n_voxels", C.c_ulonglong), ("n_dynamic_voxels", C.c_ulonglong), ("n_points", C.c_ulonglong),
                ("n_static_points", C.c_ulonglong), ("n_batches", C.c_int)]


class SmMeshParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("truncation", C.c_double), ("max_range", C.c_double),
                ("sensor_origin", C.c_double * 3), ("min_weight", C.c_uint)]


class SmMeshInfo(C.Structure):
    _fields_ = [("box_origin", C.c_int * 3), ("box_dims", C.c_uint * 3), ("n_points", C.c_ulonglong), ("n_rays", C.c_ulonglong),
                ("n_skipped", C.c_ulonglong), ("n_walked", C.c_ulonglong), ("n_band_voxels", C.c_ulonglong),
                ("n_observed_voxels", C.c_ulonglong), ("n_vertices", C.c_ulonglong), ("n_faces", C.c_ulonglong)]


class SmOctoMapInfo(C.Structure):
    _fields_ = [("box_origin", C.c_int * 3), ("box_dims", C.c_uint * 3), ("n_rays", C.c_ulonglong), ("n_skipped", C.c_ulonglong),
                ("n_occupied_voxels", C.c_ulonglong), ("n_dynamic_voxels", C.c_ulonglong), ("n_free_voxels", C.c_ulonglong),
                ("n_inner_nodes", C.c_ulonglong), ("n_occupied_leaves", C.c_ulonglong), ("n_free_leaves", C.c_ulonglong),
                ("tree_size", C.c_ulonglong), ("n_bytes", C.c_ulonglong), ("n_batches", C.c_int)]


class SmMapChangeInfo(C.Structure):
    _fields_ = [("box_origin", C.c_int * 3), ("box_dims", C.c_uint * 3), ("split_submap", C.c_longlong),
                ("n_rays", C.c_ulonglong), ("n_skipped", C.c_ulonglong), ("n_voxels", C.c_ulonglong),
                ("n_appeared_voxels", C.c_ulonglong), ("n_vanished_voxels", C.c_ulonglong), ("n_points", C.c_ulonglong),
                ("n_appeared_points", C.c_ulonglong), ("n_vanished_points", C.c_ulonglong),
                ("n_updated_points", C.c_ulonglong), ("n_batches", C.c_int)]


class SmLoopEdge(C.Structure):
    _fields_ = [("from_", C.c_int), ("to", C.c_int), ("relative_pose", C.c_double * 16)]


class SmPoseAdjustResult(C.Structure):
    _fields_ = [("chi2_initial", C.c_double), ("chi2_final", C.c_double), ("iterations", C.c_int), ("trials", C.c_int),
                ("n_vertices", C.c_int), ("n_edges", C.c_int)]


class SmMergeParams(C.Structure):
    _fields_ = [("sc_threshold", C.c_double), ("top_k", C.c_int), ("max_verifications", C.c_int), ("voxel_leaf_size", C.c_float),
                ("threshold_loop_closure_score", C.c_double), ("search_submap_num", C.c_int),
                ("consistency_translation", C.c_double), ("consistency_rotation", C.c_double),
                ("consistency_drift_translation", C.c_double), ("consistency_drift_rotation", C.c_double),
                ("min_inliers", C.c_int), ("num_adjacent_pose_cnstraints", C.c_int), ("max_iterations", C.c_int)]


MERGE_DEFAULTS = dict(sc_threshold=0.4, top_k=3, max_verifications=64, voxel_leaf_size=0.3, threshold_loop_closure_score=1.0,
                      search_submap_num=1, consistency_translation=1.5, consistency_rotation=0.1,
                      consistency_drift_translation=0.02, consistency_drift_rotation=0.003, min_inliers=2,
                      num_adjacent_pose_cnstraints=5, max_iterations=10)


class SmMergeRow(C.Structure):
    _fields_ = [("place", SmPlaceResult), ("src_id", C.c_int), ("inlier", C.c_int)]


class SmMergeResult(C.Structure):
    _fields_ = [("merged", C.c_int), ("query_tile", C.c_int), ("pairs_scored", C.c_ulonglong), ("candidates", C.c_int),
                ("verified", C.c_int), ("accepted", C.c_int), ("inliers", C.c_int), ("first_submap", C.c_int),
                ("T", C.c_double * 16), ("adjust", SmPoseAdjustResult)]


class SmSessionIoInfo(C.Structure):
    _fields_ = [("n_submaps", C.c_size_t), ("n_segments", C.c_size_t), ("n_points", C.c_size_t), ("n_loop_edges", C.c_int),
                ("num_adjacent_pose_cnstraints", C.c_int), ("adjusted", C.c_int), ("n_bytes", C.c_ulonglong)]


class SmStats(C.Structure):
    _fields_ = [("n_scan", C.c_size_t), ("n_filtered", C.c_size_t), ("n_targeted", C.c_size_t), ("n_submaps", C.c_size_t),
                ("kernel_launches", C.c_int), ("trans", C.c_double), ("latest_distance", C.c_double)]


class SmLocalizeStats(C.Structure):
    _fields_ = [("n_map", C.c_size_t), ("n_cut", C.c_size_t), ("n_target", C.c_size_t), ("cut_centre", C.c_double * 2),
                ("dist_from_centre", C.c_double), ("n_cuts", C.c_int), ("cut_pending", C.c_int)]


class BatchResult(C.Structure):
    _fields_ = [("final_T", C.c_float * 16), ("trans_probability", C.c_double), ("converged", C.c_int), ("iterations", C.c_int),
                ("evaluations", C.c_int), ("status", C.c_int), ("hits_total", C.c_longlong)]


class SmGlobalSearch(C.Structure):
    _fields_ = [("radius", C.c_double), ("step", C.c_double), ("yaw_steps", C.c_int), ("top_k", C.c_int)]


class SmGlobalResult(C.Structure):
    _fields_ = [("n_hypotheses", C.c_longlong), ("hits_total", C.c_longlong), ("n_refined", C.c_int), ("best", C.c_int),
                ("score_ms", C.c_float)]


class SmRelocalizeParams(C.Structure):
    _fields_ = [("resolution", C.c_double), ("z_min", C.c_double), ("z_max", C.c_double), ("yaw_steps", C.c_int),
                ("num_levels", C.c_int), ("min_score", C.c_double), ("top_k", C.c_int), ("accept_fitness", C.c_double)]


RELOCALIZE_DEFAULTS = dict(resolution=0.25, z_min=0.3, z_max=3.0, yaw_steps=360, num_levels=6, min_score=0.3, top_k=4,
                           accept_fitness=1.0)


class SmRelocalizeRow(C.Structure):
    _fields_ = [("yaw_index", C.c_int), ("cell_i", C.c_int), ("cell_j", C.c_int), ("score", C.c_int), ("guess", C.c_float * 16),
                ("final_T", C.c_float * 16), ("fitness", C.c_double), ("trans_probability", C.c_double), ("converged", C.c_int),
                ("iterations", C.c_int), ("status", C.c_int), ("pad", C.c_int)]


class SmRelocalizeResult(C.Structure):
    _fields_ = [("width", C.c_longlong), ("height", C.c_longlong), ("origin_cell", C.c_int * 2), ("m", C.c_longlong),
                ("t0", C.c_longlong), ("t", C.c_longlong), ("leaves", C.c_ulonglong), ("nodes", C.c_longlong * 16),
                ("n_rows", C.c_int), ("best", C.c_int), ("pyramid_builds", C.c_int), ("search_ms", C.c_float)]


class SweepResult(C.Structure):
    _fields_ = [("final_T", C.c_float * 16), ("fitness", C.c_double), ("trans_probability", C.c_double), ("converged", C.c_int),
                ("iterations", C.c_int), ("status", C.c_int), ("pad", C.c_int)]


class Stats(C.Structure):
    _fields_ = [
        ("evaluations", C.c_int), ("iterations", C.c_int),
        ("hits", C.c_longlong), ("hits_total", C.c_longlong),
        ("solve_ms", C.c_float), ("target_build_ms", C.c_float),
        ("kernel_launches", C.c_int),
        ("grid_ctas", C.c_int), ("block_threads", C.c_int), ("index_in_smem", C.c_int),
        ("n_voxels", C.c_longlong), ("n_cells", C.c_longlong), ("n_source", C.c_longlong), ("n_target", C.c_longlong),
        ("gicp_inner_ms", C.c_float), ("gicp_inner_launches", C.c_int), ("gicp_pair_evaluations", C.c_double),
    ]


def build(force: bool = False) -> str:
    """Compile the sm_90a library in-tree with nvcc (build.sh)."""
    env = dict(os.environ)
    if force:
        for f in os.listdir(os.path.join(_HERE, "csrc")):
            if f.endswith(".o"):
                os.remove(os.path.join(_HERE, "csrc", f))
    subprocess.check_call(["bash", os.path.join(REPO_ROOT, "build.sh")], env=env)
    return LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, sz, i, d, f = C.c_void_p, C.c_size_t, C.c_int, C.c_double, C.c_float
    L.b200reg_create.argtypes = [i, i, C.POINTER(vp)]
    L.b200reg_destroy.argtypes = [vp]
    L.b200reg_last_error.argtypes = [vp]
    L.b200reg_last_error.restype = C.c_char_p
    for name in ("b200reg_set_transformation_epsilon", "b200reg_set_max_correspondence_distance",
                 "b200reg_set_euclidean_fitness_epsilon", "b200reg_ndt_set_step_size", "b200reg_ndt_set_outlier_ratio",
                 "b200reg_gicp_set_rotation_epsilon", "b200reg_gicp_set_epsilon"):
        getattr(L, name).argtypes = [vp, d]
    for name in ("b200reg_set_maximum_iterations", "b200reg_set_ransac_iterations",
                 "b200reg_ndt_set_neighborhood_search_method", "b200reg_ndt_set_num_threads",
                 "b200reg_gicp_set_correspondence_randomness", "b200reg_gicp_set_maximum_optimizer_iterations"):
        getattr(L, name).argtypes = [vp, i]
    L.b200reg_ndt_set_resolution.argtypes = [vp, f]
    L.b200reg_ndt_get_transformation_probability.argtypes = [vp, C.POINTER(d)]
    L.b200reg_ndt_get_final_num_iteration.argtypes = [vp, C.POINTER(i)]
    L.b200reg_ndt_calculate_score.argtypes = [vp, vp, sz, sz, C.POINTER(d)]
    L.b200reg_set_input_target.argtypes = [vp, vp, sz, sz]
    L.b200reg_set_input_source.argtypes = [vp, vp, sz, sz]
    L.b200reg_set_input_target_device.argtypes = [vp, vp, sz]
    L.b200reg_set_input_source_device.argtypes = [vp, vp, sz]
    L.b200reg_align.argtypes = [vp, vp, vp]
    L.b200reg_get_final_transformation.argtypes = [vp, vp]
    L.b200reg_has_converged.argtypes = [vp, C.POINTER(i)]
    L.b200reg_get_fitness_score.argtypes = [vp, d, C.POINTER(d)]
    L.b200reg_get_aligned.argtypes = [vp, vp, sz]
    L.b200reg_align_batch.argtypes = [vp, i, vp, vp]
    L.b200reg_ndt_align_batch.argtypes = [vp, i, vp, vp, sz, vp, vp]
    L.b200reg_ndt_align_batch_device.argtypes = [vp, i, vp, vp, vp, vp]
    L.b200reg_ndt_set_batch_slots.argtypes = [vp, i]
    L.b200reg_ndt_attach_pose_board.argtypes = [vp, vp]
    L.b200reg_ndt_gathered_poses.argtypes = [vp, vp, vp, i]
    L.b200reg_ndt_sweep.argtypes = [vp, i, vp, vp, vp, vp, sz, vp, d, vp]
    L.b200reg_voxelgrid.argtypes = [i, vp, sz, sz, C.c_long, f, vp, sz, C.POINTER(sz)]
    L.b200reg_get_stats.argtypes = [vp, C.POINTER(Stats)]
    L.b200reg_ndt_derivatives.argtypes = [vp, vp, vp, i, C.POINTER(d), vp, vp]
    L.b200reg_ndt_hessian_radius.argtypes = [vp, vp, vp, vp]
    L.b200reg_ndt_num_voxels.argtypes = [vp, C.POINTER(sz)]
    L.b200reg_ndt_get_voxels.argtypes = [vp, vp, vp, vp, vp, vp]
    L.b200reg_nn1.argtypes = [vp, vp, sz, sz, vp, vp]
    L.b200reg_gicp_get_covariances.argtypes = [vp, i, vp, C.POINTER(sz)]
    L.b200reg_gicp_num_correspondences.argtypes = [vp, C.POINTER(i)]
    L.b200reg_gicp_correspondences.argtypes = [vp, vp, vp, vp, vp, C.POINTER(i)]
    L.b200reg_gicp_objective.argtypes = [vp, vp, i, C.POINTER(d), vp, vp]
    L.b200reg_ndt_set_trace.argtypes = [vp, i]
    L.b200reg_ndt_get_trace.argtypes = [vp, vp, i, C.POINTER(i)]
    L.b200reg_gicp_set_trace.argtypes = [vp, i]
    L.b200reg_gicp_get_trace.argtypes = [vp, vp, i, C.POINTER(i)]
    L.b200reg_get_kind.argtypes = [vp, C.POINTER(i)]
    L.b200sm_create.argtypes = [i, C.POINTER(vp)]
    L.b200sm_destroy.argtypes = [vp]
    L.b200sm_destroy.restype = None
    L.b200sm_last_error.argtypes = [vp]
    L.b200sm_last_error.restype = C.c_char_p
    L.b200sm_set_params.argtypes = [vp, f, f, i, d, i, d, d]
    L.b200sm_set_initial_pose.argtypes = [vp, vp, vp]
    L.b200sm_set_scan.argtypes = [vp, vp, vp, sz, sz, C.c_long, C.POINTER(sz)]
    L.b200sm_update_map.argtypes = [vp, vp, vp, vp, vp, i]
    L.b200sm_receive_cloud.argtypes = [vp, vp, vp, sz, sz, C.c_long, vp, vp, C.POINTER(i)]
    L.b200sm_num_submaps.argtypes = [vp, C.POINTER(sz)]
    L.b200sm_get_targeted.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.b200sm_get_submap.argtypes = [vp, sz, vp, sz, C.POINTER(sz), vp, C.POINTER(d)]
    L.b200sm_get_filtered_scan.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.b200sm_get_stats.argtypes = [vp, C.POINTER(SmStats)]
    L.b200sm_search_loop.argtypes = [vp, vp, f, d, d, d, i, C.POINTER(SmLoopResult)]
    L.b200sm_search_loop_all.argtypes = [vp, vp, f, d, d, d, i, i, i, vp, sz, C.POINTER(sz), C.POINTER(sz)]
    L.b200sm_import_submap.argtypes = [vp, vp, sz, sz, C.c_long, vp, d]
    L.b200sm_imu_set_scan_period.argtypes = [vp, d]
    L.b200sm_imu_push.argtypes = [vp, vp, vp, vp, d]
    L.b200sm_deskew_next_scan.argtypes = [vp, d]
    L.b200sm_imu_adjust_distortion.argtypes = [vp, vp, sz, sz, C.c_long, d]
    L.b200sm_imu_get_state.argtypes = [vp, C.POINTER(i), C.POINTER(i), C.POINTER(i)]
    L.b200sm_imu_get_sample.argtypes = [vp, i, C.POINTER(d), vp, vp, vp]
    L.b200sm_imu_get_trace.argtypes = [vp, sz, C.POINTER(sz), vp, vp, vp, vp, C.POINTER(i), C.POINTER(i)]
    L.b200sm_pose_adjust.argtypes = [vp, i, vp, i, i, vp, C.POINTER(SmPoseAdjustResult)]
    L.b200sm_assemble_map.argtypes = [vp, vp, vp, sz, C.POINTER(sz), vp]
    L.b200sm_save_map_pcd_ascii.argtypes = [vp, vp, C.c_char_p, C.POINTER(sz), C.POINTER(sz)]
    L.b200reg_encode_pcd_ascii.argtypes = [i, vp, sz, sz, C.c_long, vp, sz, C.POINTER(sz)]
    L.b200sm_set_sensor_transform.argtypes = [vp, vp, vp]
    L.b200reg_load_pcd.argtypes = [i, C.c_char_p, vp, sz, C.POINTER(sz)]
    L.b200reg_set_input_target_pcd.argtypes = [vp, C.c_char_p, C.POINTER(sz)]
    L.b200sm_odom_next_scan.argtypes = [vp, vp, vp]
    L.b200sm_set_prior_map_pcd.argtypes = [vp, C.c_char_p, C.POINTER(sz)]
    L.b200sm_set_prior_map.argtypes = [vp, vp, sz, sz, C.c_long]
    L.b200sm_set_localization_params.argtypes = [vp, d, d]
    L.b200sm_localize_cloud.argtypes = [vp, vp, vp, sz, sz, C.c_long, vp, vp, C.POINTER(i)]
    L.b200sm_localize_init.argtypes = [vp, vp, vp, sz, sz, C.c_long, vp, i, vp, C.POINTER(i)]
    L.b200sm_get_localize_stats.argtypes = [vp, C.POINTER(SmLocalizeStats)]
    L.b200sm_get_cut.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.b200reg_ndt_score_poses.argtypes = [vp, i, vp, vp, vp]
    L.b200sm_localize_global.argtypes = [vp, vp, vp, sz, sz, C.c_long, C.POINTER(SmGlobalSearch), vp, vp, C.POINTER(SmGlobalResult)]
    L.b200sm_get_global_search.argtypes = [vp, sz, C.POINTER(sz), vp, vp, vp]
    L.b200sm_relocalize.argtypes = [vp, vp, vp, sz, sz, C.c_long, C.POINTER(SmRelocalizeParams), C.POINTER(SmRelocalizeRow), sz,
                                    C.POINTER(SmRelocalizeResult)]
    L.b200sm_get_relocalize_grid.argtypes = [vp, i, vp, sz, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    L.b200sm_relocalize_score_nodes.argtypes = [vp, i, C.c_longlong, vp, vp]
    L.b200sm_set_scan_context_params.argtypes = [vp, C.POINTER(SmScanContextParams)]
    L.b200sm_get_scan_context.argtypes = [vp, sz, vp, sz]
    L.b200sm_search_loop_place.argtypes = [vp, vp, f, d, d, i, d, i, vp, sz, C.POINTER(sz), C.POINTER(sz)]
    L.b200sm_get_place_scores.argtypes = [vp, sz, C.POINTER(sz), vp, vp]
    L.b200sm_build_occupancy_grid.argtypes = [vp, vp, C.POINTER(SmOccupancyParams), C.POINTER(SmOccupancyInfo)]
    L.b200sm_get_occupancy_grid.argtypes = [vp, vp, vp, vp, sz]
    L.b200sm_save_occupancy_map.argtypes = [vp, C.c_char_p, C.c_char_p]
    L.b200sm_build_elevation_map.argtypes = [vp, vp, C.POINTER(SmElevationParams), C.POINTER(SmElevationInfo)]
    L.b200sm_get_elevation_map.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, sz]
    L.b200sm_save_traversability_map.argtypes = [vp, C.c_char_p, C.c_char_p]
    L.b200sm_build_static_map.argtypes = [vp, vp, C.POINTER(SmStaticMapParams), C.POINTER(SmStaticMapInfo)]
    L.b200sm_get_static_map.argtypes = [vp, vp, sz, C.POINTER(sz), vp]
    L.b200sm_get_map_voxels.argtypes = [vp, vp, vp, vp, vp, sz, C.POINTER(sz)]
    L.b200sm_save_static_map_pcd_ascii.argtypes = [vp, C.c_char_p, C.POINTER(sz), C.POINTER(sz)]
    L.b200sm_build_map_consistency.argtypes = [vp, vp, C.POINTER(SmMapConsistencyParams), C.POINTER(SmMapConsistencyInfo)]
    L.b200sm_get_map_consistency.argtypes = [vp, vp, vp, vp, sz]
    L.b200sm_get_submap_consistency.argtypes = [vp, vp, sz]
    L.b200sm_save_map_consistency_pcd_ascii.argtypes = [vp, C.c_char_p, C.POINTER(sz), C.POINTER(sz)]
    L.b200sm_build_map_changes.argtypes = [vp, vp, C.POINTER(SmStaticMapParams), C.c_longlong, C.POINTER(SmMapChangeInfo)]
    L.b200sm_get_map_changes.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.b200sm_get_change_voxels.argtypes = [vp, vp, vp, vp, vp, vp, vp, sz, C.POINTER(sz)]
    L.b200sm_get_updated_map.argtypes = [vp, vp, sz, C.POINTER(sz), vp]
    L.b200sm_save_updated_map_pcd_ascii.argtypes = [vp, C.c_char_p, C.POINTER(sz), C.POINTER(sz)]
    L.b200sm_build_mesh.argtypes = [vp, vp, C.POINTER(SmMeshParams), C.POINTER(SmMeshInfo)]
    L.b200sm_get_mesh.argtypes = [vp, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz)]
    L.b200sm_get_mesh_voxels.argtypes = [vp, vp, vp, vp, sz, C.POINTER(sz)]
    L.b200sm_save_mesh_ply.argtypes = [vp, C.c_char_p, C.POINTER(sz)]
    L.b200sm_build_octomap.argtypes = [vp, vp, C.POINTER(SmStaticMapParams), C.POINTER(SmOctoMapInfo)]
    L.b200sm_get_octomap_states.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.b200sm_get_octomap_bt.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.b200sm_save_octomap_bt.argtypes = [vp, C.c_char_p, C.POINTER(sz)]
    L.b200sm_merge_session.argtypes = [vp, vp, vp, C.POINTER(SmMergeParams), vp, i, vp, sz, C.POINTER(sz), vp,
                                        C.POINTER(SmMergeResult)]
    L.b200sm_get_merge_scores.argtypes = [vp, sz, C.POINTER(sz), C.POINTER(sz), vp, vp]
    L.b200sm_get_segments.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.b200sm_save_session.argtypes = [vp, C.c_char_p, i, vp, i, vp, C.POINTER(SmSessionIoInfo)]
    L.b200sm_load_session.argtypes = [vp, C.c_char_p, C.POINTER(SmSessionIoInfo)]
    L.b200sm_get_session_graph.argtypes = [vp, vp, sz, C.POINTER(sz), vp, C.POINTER(i)]
    L.b200comm_unique_id.argtypes = [vp]
    L.b200comm_create.argtypes = [vp, i, i, i, C.POINTER(vp)]
    L.b200comm_destroy.argtypes = [vp]
    L.b200comm_all_gather_rows.argtypes = [vp, vp, i, i, vp]
    L.b200comm_rank.argtypes = [vp, C.POINTER(i), C.POINTER(i)]
    L.b200comm_board_create.argtypes = [vp, i, C.POINTER(vp)]
    L.b200comm_board_destroy.argtypes = [vp]
    L.b200comm_board_info.argtypes = [vp, C.POINTER(i), C.POINTER(i), C.POINTER(i)]
    L.b200comm_last_error.argtypes = []
    L.b200comm_last_error.restype = C.c_char_p
    for name in SYMBOLS:
        fn = getattr(L, name)
        if name not in ("b200reg_last_error", "b200sm_last_error", "b200sm_destroy", "b200comm_last_error"):
            fn.restype = i
    _lib = L
    return L
