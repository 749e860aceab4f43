"""ctypes binding of libloamlivox_b200.so (include/loamlivox_b200.h).

The CUDA library is the product: importing this module without the shared object, or creating a context without a
Hopper (sm_90a) GPU, fails loudly — there is no CPU or PyTorch fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libloamlivox_b200.so")

LL_FMT_XYZI16, LL_FMT_PCL32, LL_FMT_STRIDED = 0, 1, 2
LL_I_NONE, LL_I_UINT8, LL_I_UINT16, LL_I_FLOAT32 = 0, 2, 4, 7   # sensor_msgs/PointField datatype codes
LL_HOST, LL_DEVICE = 0, 1
LL_OK, LL_ERR_INVALID, LL_ERR_CUDA, LL_ERR_CAPACITY, LL_ERR_NO_BLOCKS, LL_ERR_CAP_BINDS = 0, -1, -2, -3, -4, -5
LL_IPC_HANDLE_BYTES = 64
LL_MAX_PIECES_PER_FRAME = 16
LL_MAX_BATCH = 16
LL_RELOC_MAX_SCORE_POINTS = 8192
LL_RECOVERY_LOG = 1024
LL_TRACKING, LL_SUSPECT, LL_LOST = 0, 1, 2
LL_BAD_NONE, LL_BAD_REJECTED, LL_BAD_INLIER = 0, 1, 2
LL_PG_MAX_BORDER = 64
LL_MAX_LOOPS = LL_PG_MAX_BORDER // 2
LL_LOOP_LOG = 1024
LL_LOOP_KEYFRAME, LL_LOOP_ALIGNMENT, LL_LOOP_CLOSED, LL_LOOP_ERROR = 0, 1, 2, 3
LL_LOOP_SKIP10, LL_LOOP_SKIP5, LL_LOOP_ACCEPT, LL_LOOP_FAILED = 0, 1, 2, 3
LL_MAPPER_IMAGE_MAGIC, LL_MAPPER_IMAGE_VERSION = b"LLMAPIMG", 1
LL_LOOP_IMAGE_MAGIC, LL_LOOP_IMAGE_VERSION, LL_LOOP_IMAGE_VERSION_POLICY, LL_LOOP_IMAGE_VERSION_FEEDBACK = b"LLLOOPIM", 1, 2, 3
LL_LOOP_IMAGE_FEEDBACK, LL_LOOP_IMAGE_SECTIONS_FEEDBACK = 13, 14
LL_LOOP_FEEDBACK_MAX_SEGMENTS = 4096
(LL_LOOP_IMAGE_CONFIG, LL_LOOP_IMAGE_SCALARS, LL_LOOP_IMAGE_CELLS, LL_LOOP_IMAGE_HISTORY, LL_LOOP_IMAGE_OPEN, LL_LOOP_IMAGE_KEYFRAMES, LL_LOOP_IMAGE_POSES,
 LL_LOOP_IMAGE_EDGES, LL_LOOP_IMAGE_IMAGES, LL_LOOP_IMAGE_CLOUDS, LL_LOOP_IMAGE_ACCUMULATED, LL_LOOP_IMAGE_LOOP, LL_LOOP_IMAGE_EVENTS, LL_LOOP_IMAGE_SECTIONS) = range(14)
(LL_IMAGE_CONFIG, LL_IMAGE_SCALARS, LL_IMAGE_HISTORY_CORNER, LL_IMAGE_HISTORY_SURF, LL_IMAGE_SNAPSHOT_CORNER, LL_IMAGE_SNAPSHOT_SURF, LL_IMAGE_CELLS_CORNER,
 LL_IMAGE_CELLS_SURF, LL_IMAGE_SECTIONS) = range(9)

EXPORTS = [
    "ll_config_default", "ll_ctx_create", "ll_ctx_destroy", "ll_ctx_warmup", "ll_last_error", "ll_ctx_stream", "ll_ctx_sync", "ll_extract", "ll_extract_reset", "ll_piece_bounds",
    "ll_get_features", "ll_extract_point_info", "ll_extract_split_idx", "ll_extract_petal_angles", "ll_voxel_downsample", "ll_map_build", "ll_map_release", "ll_map_size",
    "ll_map_build_sharded", "ll_knn", "ll_reg_state_default", "ll_register", "ll_build_blocks", "ll_normal_equations", "ll_solve", "ll_inlier_select", "ll_set_blocks", "ll_solve_fused", "ll_register_dev_counts", "ll_transform",
    "ll_scan_to_pose", "ll_comm_local_handle", "ll_comm_connect", "ll_launch_count", "ll_cellmap_create", "ll_cellmap_release", "ll_cellmap_append",
    "ll_cellmap_assemble", "ll_cellmap_reserve", "ll_cellmap_stats", "ll_voxel_downsample_dev", "ll_transform_dev", "ll_last_features_dev", "ll_mapper_config_default", "ll_mapper_create", "ll_mapper_release",
    "ll_mapper_process_scan", "ll_mapper_pose", "ll_map_rebuild", "ll_debug_solver_cycles", "ll_state_snapshot_bytes", "ll_set_point_layout", "ll_format_pose_log", "ll_reg_state_yaml", "ll_cap_uniform", "ll_map_shard_info", "ll_shard_plan", "ll_align_cfg_default", "ll_scene_align", "ll_frame_to_pose", "ll_features_to_pointcloud2",
    "ll_mapper_process_frame", "ll_voxel_downsample_segments", "ll_register_batch", "ll_mapper_process_frames", "ll_mapper_process_scans",
    "ll_mapper_save", "ll_mapper_load", "ll_mapper_image_info",
    "ll_reloc_index_build", "ll_reloc_index_release", "ll_reloc_index_read", "ll_relocalize", "ll_reloc_scores", "ll_mapper_whole_map", "ll_mapper_set_pose",
    "ll_reloc_field_build", "ll_reloc_field_release", "ll_reloc_field_read", "ll_relocalize_field", "ll_reloc_field_scores",
    "ll_mapper_recovery_default", "ll_mapper_set_recovery", "ll_mapper_recovery_read", "ll_mapper_recovery_last_inputs",
    "ll_pose_graph_create", "ll_pose_graph_release", "ll_pose_graph_optimize", "ll_pose_graph_step", "ll_pose_graph_loop_edge",
    "ll_keyframes_repose", "ll_keyframe_affine",
    "ll_keyframe_create", "ll_keyframe_release", "ll_keyframe_append", "ll_keyframe_analyze", "ll_keyframe_get_info", "ll_keyframe_cells",
    "ll_keyframe_images", "ll_keyframe_cloud", "ll_loop_cfg_default", "ll_loop_search",
    "ll_mapper_loop_closure_default", "ll_mapper_set_loop_closure", "ll_mapper_loop_read", "ll_mapper_loop_result", "ll_mapper_loop_cloud",
    "ll_spin_cfg_default", "ll_spin_create", "ll_spin_release", "ll_spin_extract", "ll_spin_cloud", "ll_spin_point_info", "ll_spin_chains",
    "ll_mapper_process_sweep", "ll_mapper_process_sweeps",
    "ll_mapper_loop_save", "ll_mapper_loop_load", "ll_loop_image_info",
    "ll_mapper_loop_policy_default", "ll_mapper_set_loop_policy", "ll_mapper_loop_edges",
    "ll_mapper_set_loop_feedback", "ll_mapper_loop_correction_read", "ll_loop_correction",
]
LL_SPIN_FULL, LL_SPIN_SHARP, LL_SPIN_LESS_SHARP, LL_SPIN_FLAT, LL_SPIN_LESS_FLAT = 0, 1, 2, 3, 4
LL_CELL_SPHERE, LL_CELL_LINE, LL_CELL_PLANE, LL_CELL_ALL = 0, 1, 2, -1


class SpinCfg(C.Structure):
    """ll_spin_cfg: the Velodyne branch's feature_extraction parameters and the handle's input capacity."""
    _fields_ = [("scan_line", C.c_int), ("minimum_range", C.c_float), ("plane_resolution", C.c_float), ("max_points", C.c_int)]


class Config(C.Structure):
    _fields_ = [("corner_curvature", C.c_float), ("surface_curvature", C.c_float), ("minimum_view_angle", C.c_float), ("livox_min_dis", C.c_float),
                ("livox_min_sigma", C.c_float), ("max_fov_deg", C.c_float), ("time_interval_pts", C.c_float), ("max_scan_points", C.c_int), ("max_features", C.c_int)]


class RegState(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("if_motion_deblur", "current_frame_index", "mapping_init_accumulate_frames", "icp_max_iterations", "cere_max_iterations",
                                       "cere_prerun_times", "icp_plane", "icp_line", "maximum_allow_residual_block", "rng_seed")] + \
               [(n, C.c_double) for n in ("para_max_angular_rate", "para_max_speed", "max_final_cost", "minimum_pt_time_stamp", "maximum_pt_time_stamp",
                                          "minimum_icp_R_diff", "minimum_icp_T_diff", "inliner_dis", "inlier_ratio", "maximum_dis_plane_for_match",
                                          "maximum_dis_line_for_match", "huber_a")] + \
               [("q_w_last", C.c_double * 4), ("t_w_last", C.c_double * 3), ("q_w_curr", C.c_double * 4), ("t_w_curr", C.c_double * 3),
                ("para_buffer_incremental", C.c_double * 7)]


class RegResult(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("status", "registered", "num_residual_blocks", "icp_iterations", "corner_used", "surf_used", "total_lm_iterations",
                                       "total_evaluations")] + \
               [("q_w_curr", C.c_double * 4), ("t_w_curr", C.c_double * 3), ("q_w_incre", C.c_double * 4), ("t_w_incre", C.c_double * 3)] + \
               [(n, C.c_double) for n in ("inlier_threshold", "final_cost", "initial_cost", "angular_diff", "t_diff")] + \
               [("gpu_ms_total", C.c_float), ("gpu_ms_knn", C.c_float), ("gpu_ms_knn_all", C.c_float), ("gpu_ms_solve_all", C.c_float),
                ("gpu_ms_select_all", C.c_float), ("gpu_ms_sort", C.c_float)]


class PipelineCfg(C.Structure):
    _fields_ = [("pieces", C.c_int), ("use_piece", C.c_int), ("extractor_leaf_corner", C.c_float), ("extractor_leaf_surf", C.c_float),
                ("mapping_leaf_corner", C.c_float), ("mapping_leaf_surf", C.c_float), ("whole_frame", C.c_int)]


class PointLayout(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("point_step", "offset_x", "offset_y", "offset_z", "offset_intensity", "intensity_datatype")]


class MapperConfig(C.Structure):
    _fields_ = [("line_resolution", C.c_float), ("plane_resolution", C.c_float), ("cell_resolution", C.c_float), ("threshold_cell_revisit", C.c_int),
                ("maximum_search_range_corner", C.c_float), ("maximum_search_range_surface", C.c_float), ("maximum_in_fov_angle", C.c_float),
                ("down_sample_replace", C.c_int), ("max_cells", C.c_int), ("matching_mode", C.c_int), ("maximum_history_size", C.c_int),
                ("reserve_map_points", C.c_int), ("reserve_store_points", C.c_int),
                ("pipeline", PipelineCfg), ("reg", RegState)]


class MapperStats(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("n_corner", "n_surf", "map_corner", "map_surf", "cells_in_fov_corner", "cells_in_fov_surf", "appended_corner", "appended_surf")] + \
               [(n, C.c_float) for n in ("ms_front_end", "ms_refresh", "ms_register", "ms_append")]


class ImageInfo(C.Structure):
    """ll_image_info: what ll_mapper_image_info reports about a mapper image ([0] corner, [1] surface)."""
    _fields_ = [("bytes", C.c_uint64), ("history_points", C.c_int64 * 2), ("snapshot_points", C.c_int64 * 2), ("cells", C.c_int64 * 2), ("cell_points", C.c_int64 * 2),
                ("version", C.c_uint32), ("matching_mode", C.c_int), ("frame_index", C.c_int), ("have_map", C.c_int), ("map_dirty", C.c_int),
                ("history_segments", C.c_int * 2), ("cell_frame_idx", C.c_int * 2), ("reserved", C.c_int)]


class ShardInfo(C.Structure):
    _fields_ = [("rank", C.c_int), ("world", C.c_int), ("cell_size", C.c_float), ("halo_corner", C.c_float), ("halo_surf", C.c_float), ("origin", C.c_float * 3),
                ("dims", C.c_int * 3), ("kept_corner", C.c_longlong), ("kept_surf", C.c_longlong), ("total_corner", C.c_longlong), ("total_surf", C.c_longlong)]


class AlignCfg(C.Structure):
    _fields_ = [("line_res", C.c_float), ("plane_res", C.c_float), ("maximum_icp_iteration", C.c_int), ("maximum_residual_block", C.c_int),
                ("accepted_threshold", C.c_float), ("rng_seed", C.c_int), ("t_init", C.c_double * 3)]


class RelocCfg(C.Structure):
    """ll_reloc_cfg: the hypotheses of a relocalization (rotations x translation lattice) and the candidate count K."""
    _fields_ = [("n_rot", C.c_int), ("rot_wxyz", C.POINTER(C.c_double)), ("rot_cyclic", C.c_int), ("t0", C.c_double * 3), ("step", C.c_double * 3),
                ("nt", C.c_int * 3), ("max_candidates", C.c_int)]


class RelocCandidate(C.Structure):
    _fields_ = [("q_wxyz", C.c_double * 4), ("t", C.c_double * 3), ("score", C.c_int32), ("hypothesis", C.c_int32)]


class RelocFineCfg(C.Structure):
    """ll_reloc_fine_cfg: the fine search around every candidate (rotation offsets x an odd lattice centred on the candidate)."""
    _fields_ = [("n_rot", C.c_int), ("rot_wxyz", C.POINTER(C.c_double)), ("step", C.c_double * 3), ("nt", C.c_int * 3)]


class RelocFieldCandidate(C.Structure):
    """ll_reloc_field_candidate: a coarse peak, its fine pick and the field score at its refined pose."""
    _fields_ = [("q_wxyz", C.c_double * 4), ("t", C.c_double * 3), ("score", C.c_int32), ("hypothesis", C.c_int32),
                ("fine_q_wxyz", C.c_double * 4), ("fine_t", C.c_double * 3), ("fine_score", C.c_int32), ("fine_index", C.c_int32),
                ("verify_score", C.c_int32), ("reserved", C.c_int32)]


class RecoveryCfg(C.Structure):
    """ll_recovery_cfg: the streaming mapper's tracking-loss detection, relocalization search, acceptance floor and reservations."""
    _fields_ = [("max_inlier_threshold", C.c_double), ("lost_after", C.c_int), ("trunc", C.c_int), ("res", C.c_float), ("score_leaf", C.c_float),
                ("yaw_step_deg", C.c_double), ("t_step", C.c_double), ("window_base", C.c_double), ("window_growth", C.c_double),
                ("max_candidates", C.c_int), ("max_hypotheses", C.c_int), ("fine_yaw_step_deg", C.c_double), ("fine_t_step", C.c_double),
                ("fine_t_half", C.c_double), ("min_verify_fraction", C.c_double), ("reserve_field_voxels", C.c_longlong),
                ("reserve_whole_map_points", C.c_longlong)]


class RecoveryStep(C.Structure):
    """ll_recovery_step: one mapper step while recovery is on (state, detection, and the relocalization attempt when there was one)."""
    _fields_ = [(n, C.c_int32) for n in ("frame_index", "state_before", "state_after", "bad", "bad_steps", "appended", "attempted", "attempt_status")] + \
               [("nt", C.c_int32 * 3), ("n_yaw", C.c_int32)] + [(n, C.c_int32) for n in ("n_cand", "best", "adopted", "grew")] + \
               [("n_score", C.c_int32 * 2), ("score_leaf", C.c_float * 2), ("t0", C.c_double * 3), ("step", C.c_double * 3), ("tilt_wxyz", C.c_double * 4),
                ("verify_fraction", C.c_double), ("q_wxyz", C.c_double * 4), ("t", C.c_double * 3), ("inlier_threshold", C.c_double),
                ("ms_map", C.c_double), ("ms_search", C.c_double)]


class Pose(C.Structure):
    """ll_pose: a pose graph vertex (q as w, x, y, z)."""
    _fields_ = [("q_wxyz", C.c_double * 4), ("t", C.c_double * 3)]


class PgEdge(C.Structure):
    """ll_pg_edge: a pose graph constraint t_be = (q, t) from id_begin to id_end with its information matrix (row-major)."""
    _fields_ = [("id_begin", C.c_int), ("id_end", C.c_int), ("q_wxyz", C.c_double * 4), ("t", C.c_double * 3), ("information", C.c_double * 36)]


class PgSummary(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double)] + \
               [(n, C.c_int) for n in ("iterations", "evaluations", "termination", "border_nodes", "segments", "levels", "free_nodes", "reserved")] + \
               [(n, C.c_longlong) for n in ("cycles_eval", "cycles_elim", "cycles_border", "cycles_total")]


class KeyframeInfo(C.Structure):
    """ll_keyframe_info: what Maps_keyframe::analyze leaves (centre, ROI range, nonzero ratios) and the typed clouds' sizes."""
    _fields_ = [(n, C.c_int) for n in ("cells", "line_cells", "plane_cells", "accumulate_frames")] + \
               [("center", C.c_float * 3), ("roi_range", C.c_float), ("ratio_nonzero_line", C.c_float), ("ratio_nonzero_plane", C.c_float)] + \
               [(n, C.c_size_t) for n in ("line_points", "plane_points", "all_points")]


class LoopCfg(C.Structure):
    """ll_loop_cfg: the gates of service_loop_detection's candidate search."""
    _fields_ = [("minimum_keyframe_differen", C.c_int)] + \
               [(n, C.c_float) for n in ("avail_ratio_plane", "avail_ratio_line", "maximum_roi_difference", "minimum_similarity_linear",
                                         "minimum_similarity_planar")] + [("plane_with_line", C.c_double)]


class LoopClosureCfg(C.Structure):
    """ll_loop_closure_cfg: the streaming mapper's keyframe schedule, search gates, alignment, accumulated-cloud leaf and reservations."""
    _fields_ = [("scans_of_each_keyframe", C.c_int), ("scans_between_two_keyframe", C.c_int), ("loop", LoopCfg),
                ("map_alignment_resolution", C.c_float), ("map_alignment_maximum_icp_iteration", C.c_int), ("map_alignment_inlier_threshold", C.c_float),
                ("scene_alignment_maximum_residual_block", C.c_int), ("surround_pointcloud_resolution", C.c_double), ("incremental_cov", C.c_int),
                ("rng_seed", C.c_int), ("max_cells", C.c_int), ("reserve_map_points", C.c_longlong), ("reserve_history_points", C.c_longlong),
                ("reserve_keyframes", C.c_int)]


class LoopPolicy(C.Structure):
    """ll_loop_policy: how many loops the streaming mapper closes, and the keyframes between the newest keyframes of two loops."""
    _fields_ = [("max_loops", C.c_int32), ("min_keyframes_between_loops", C.c_int32)]


class LoopEvent(C.Structure):
    """ll_loop_event: a processed keyframe, one alignment of a candidate, or the closed loop."""
    _fields_ = [(n, C.c_int32) for n in ("kind", "keyframe", "ending_frame_idx", "n_candidates")] + [("info", KeyframeInfo),
                ("q_wxyz", C.c_double * 4), ("t", C.c_double * 3)] + [(n, C.c_int32) for n in ("his", "scales_run", "decision", "status")] + \
               [("inlier_threshold", C.c_double), ("icp_q_wxyz", C.c_double * 4), ("icp_t", C.c_double * 3), ("edge", PgEdge), ("summary", PgSummary)]


class LoopImageScalars(C.Structure):
    """ll_loop_image_scalars: the loop image's binding stamp (the mapper's state it refers to), closed / stopped and the counts."""
    _fields_ = [(n, C.c_int32) for n in ("frame_index", "matching_mode", "threshold_cell_revisit", "maximum_history_size", "pieces")] + \
               [("cell_resolution", C.c_float), ("last_time_stamp", C.c_double), ("q_w_curr", C.c_double * 4), ("t_w_curr", C.c_double * 3)] + \
               [(n, C.c_int32) for n in ("closed", "stopped", "n_keyframes", "n_open", "n_events", "n_dropped")]


class LoopImageSummary(C.Structure):
    """ll_loop_image_summary: what ll_loop_image_info reports about a loop image."""
    _fields_ = [("bytes", C.c_uint64)] + [(n, C.c_int64) for n in ("cells", "cell_points", "replaced_points", "history_points", "cloud_points",
                                                                    "accumulated_points")] + \
               [("version", C.c_uint32)] + [(n, C.c_int32) for n in ("frame_index", "matching_mode", "closed", "stopped", "keyframes", "open_keyframes",
                                                                     "events", "dropped", "max_incarnation")]


class LoamLivoxError(RuntimeError):
    pass


_LIB = None


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise LoamLivoxError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
                             "There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, sz, ci, cf, cd = C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_double
    L.ll_config_default.argtypes = [C.POINTER(Config)]
    L.ll_ctx_create.argtypes = [C.POINTER(Config), ci, C.POINTER(vp)]
    L.ll_ctx_destroy.argtypes = [vp]
    L.ll_last_error.argtypes = [vp]
    L.ll_last_error.restype = C.c_char_p
    L.ll_ctx_stream.argtypes = [vp]
    L.ll_ctx_stream.restype = vp
    L.ll_ctx_sync.argtypes = [vp]
    L.ll_extract.argtypes = [vp, vp, sz, ci, ci, cd, C.POINTER(ci)]
    L.ll_extract_reset.argtypes = [vp]
    L.ll_piece_bounds.argtypes = [vp, ci, vp, vp]
    L.ll_get_features.argtypes = [vp, cf, cf, vp, C.POINTER(sz), vp, C.POINTER(sz), vp, C.POINTER(sz)]
    L.ll_extract_point_info.argtypes = [vp] + [vp] * 8
    L.ll_extract_split_idx.argtypes = [vp, vp, ci, C.POINTER(ci)]
    L.ll_extract_petal_angles.argtypes = [vp, vp, ci, C.POINTER(ci)]
    L.ll_voxel_downsample.argtypes = [vp, vp, sz, ci, ci, cf, vp, C.POINTER(sz)]
    L.ll_voxel_downsample_segments.argtypes = [vp, vp, sz, vp, ci, cf, vp, vp]
    L.ll_map_build.argtypes = [vp, vp, sz, vp, sz, ci, ci, C.POINTER(vp)]
    L.ll_map_build_sharded.argtypes = [vp, vp, sz, vp, sz, ci, ci, ci, ci, cf, cf, cf, C.POINTER(vp)]
    L.ll_map_shard_info.argtypes = [vp, C.POINTER(ShardInfo), vp, sz]
    L.ll_shard_plan.argtypes = [vp, vp, ci, vp]
    L.ll_align_cfg_default.argtypes = [C.POINTER(AlignCfg)]
    L.ll_scene_align.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, ci, ci, C.POINTER(AlignCfg), C.POINTER(RegResult), C.POINTER(ci)]
    L.ll_map_release.argtypes = [vp]
    L.ll_map_size.argtypes = [vp, ci]
    L.ll_map_size.restype = sz
    L.ll_knn.argtypes = [vp, vp, ci, vp, sz, vp, vp]
    L.ll_reg_state_default.argtypes = [C.POINTER(RegState)]
    L.ll_reg_state_yaml.argtypes = [C.POINTER(RegState), ci]
    L.ll_cap_uniform.argtypes = [ci, ci, ci, ci]
    L.ll_cap_uniform.restype = cf
    L.ll_register.argtypes = [vp, vp, vp, sz, vp, sz, ci, ci, C.POINTER(RegState), C.POINTER(RegResult)]
    L.ll_register_batch.argtypes = [vp, vp, ci, vp, vp, vp, vp, ci, ci, C.POINTER(RegState), C.POINTER(RegResult), vp]
    L.ll_build_blocks.argtypes = [vp, vp, vp, sz, vp, sz, ci, ci, C.POINTER(RegState), vp, vp, vp, C.POINTER(ci), C.POINTER(ci)]
    L.ll_normal_equations.argtypes = [vp, vp, vp]
    L.ll_solve.argtypes = [vp, ci, vp, C.POINTER(cd), C.POINTER(cd), C.POINTER(ci)]
    L.ll_inlier_select.argtypes = [vp, vp, sz, cd, C.POINTER(cd), C.POINTER(ci)]
    L.ll_set_blocks.argtypes = [vp, C.POINTER(RegState), sz, vp, vp, vp, vp]
    L.ll_solve_fused.argtypes = [vp, ci, ci, vp, C.POINTER(cd), C.POINTER(ci), C.POINTER(ci), vp, vp]
    L.ll_register_dev_counts.argtypes = [vp, vp, vp, sz, vp, sz, ci, ci, C.POINTER(RegState), C.POINTER(RegResult)]
    L.ll_transform.argtypes = [vp, vp, vp, vp, sz, ci, ci, vp]
    L.ll_scan_to_pose.argtypes = [vp, vp, vp, sz, ci, ci, cd, C.POINTER(PipelineCfg), C.POINTER(RegState), C.POINTER(RegResult), C.POINTER(ci), C.POINTER(ci)]
    L.ll_frame_to_pose.argtypes = [vp, vp, ci, vp, vp, ci, ci, vp, C.POINTER(PipelineCfg), C.POINTER(RegState), C.POINTER(RegResult), C.POINTER(ci), C.POINTER(ci)]
    L.ll_features_to_pointcloud2.argtypes = [vp, ci, vp, sz, C.POINTER(sz)]
    L.ll_comm_local_handle.argtypes = [vp, vp]
    L.ll_comm_connect.argtypes = [vp, ci, ci, vp]
    L.ll_cellmap_create.argtypes = [vp, cf, ci, ci, C.POINTER(vp)]
    L.ll_cellmap_release.argtypes = [vp]
    L.ll_cellmap_append.argtypes = [vp, vp, vp, sz, ci, ci]
    L.ll_cellmap_assemble.argtypes = [vp, vp, vp, vp, cf, cf, cf, ci, vp, sz, C.POINTER(sz), C.POINTER(ci), C.POINTER(vp)]
    L.ll_ctx_warmup.argtypes = [vp]
    L.ll_cellmap_reserve.argtypes = [vp, vp, C.c_size_t, C.c_size_t]
    L.ll_cellmap_stats.argtypes = [vp, vp, C.POINTER(ci), C.POINTER(ci), C.POINTER(ci)]
    L.ll_voxel_downsample_dev.argtypes = [vp, vp, sz, cf, vp, C.POINTER(sz)]
    L.ll_transform_dev.argtypes = [vp, vp, vp, vp, sz, vp]
    L.ll_last_features_dev.argtypes = [vp, C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.POINTER(sz)]
    L.ll_debug_solver_cycles.argtypes = [vp, vp]
    L.ll_state_snapshot_bytes.argtypes = []
    L.ll_set_point_layout.argtypes = [vp, C.POINTER(PointLayout)]
    L.ll_format_pose_log.argtypes = [C.POINTER(RegResult), C.c_char_p, sz]
    L.ll_map_rebuild.argtypes = [vp, vp, vp, sz, vp, sz, ci, ci]
    L.ll_mapper_config_default.argtypes = [C.POINTER(MapperConfig)]
    L.ll_mapper_create.argtypes = [vp, C.POINTER(MapperConfig), C.POINTER(vp)]
    L.ll_mapper_release.argtypes = [vp]
    L.ll_mapper_process_scan.argtypes = [vp, vp, sz, ci, ci, cd, C.POINTER(RegResult), C.POINTER(MapperStats)]
    L.ll_mapper_process_frame.argtypes = [vp, ci, vp, vp, ci, ci, vp, ci, C.POINTER(RegResult), C.POINTER(MapperStats), ci, C.POINTER(ci)]
    L.ll_mapper_process_frames.argtypes = [vp, ci, ci, vp, vp, ci, ci, vp, ci, C.POINTER(RegResult), C.POINTER(MapperStats), ci, vp, C.POINTER(ci)]
    L.ll_mapper_process_scans.argtypes = [vp, ci, vp, vp, ci, ci, vp, C.POINTER(RegResult), C.POINTER(MapperStats), C.POINTER(ci)]
    L.ll_mapper_pose.argtypes = [vp, vp, vp, C.POINTER(ci)]
    L.ll_mapper_save.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.ll_mapper_load.argtypes = [vp, vp, sz, C.POINTER(MapperConfig), C.POINTER(vp)]
    L.ll_mapper_image_info.argtypes = [vp, sz, C.POINTER(ImageInfo)]
    L.ll_reloc_index_build.argtypes = [vp, vp, cf, ci, ci, C.POINTER(vp)]
    L.ll_reloc_index_release.argtypes = [vp]
    L.ll_reloc_index_read.argtypes = [vp, vp, vp, vp, sz]
    L.ll_relocalize.argtypes = [vp, vp, vp, vp, sz, vp, sz, vp, sz, ci, ci, C.POINTER(RelocCfg), C.POINTER(RegState), C.POINTER(RelocCandidate),
                                C.POINTER(RegResult), vp, C.POINTER(ci), C.POINTER(ci)]
    L.ll_reloc_scores.argtypes = [vp, vp, vp, sz, ci, ci, C.POINTER(RelocCfg), vp]
    L.ll_reloc_field_build.argtypes = [vp, vp, cf, ci, ci, C.POINTER(vp)]
    L.ll_reloc_field_release.argtypes = [vp]
    L.ll_reloc_field_read.argtypes = [vp, ci, vp, vp, vp, sz]
    L.ll_relocalize_field.argtypes = [vp, vp, vp, vp, sz, vp, sz, vp, sz, vp, sz, ci, ci, C.POINTER(RelocCfg), C.POINTER(RelocFineCfg), C.POINTER(RegState),
                                      C.POINTER(RelocFieldCandidate), C.POINTER(RegResult), vp, C.POINTER(ci), C.POINTER(ci)]
    L.ll_reloc_field_scores.argtypes = [vp, vp, vp, sz, vp, sz, ci, ci, C.POINTER(RelocCfg), vp]
    L.ll_mapper_whole_map.argtypes = [vp, C.POINTER(vp)]
    L.ll_mapper_set_pose.argtypes = [vp, vp, vp]
    L.ll_mapper_recovery_default.argtypes = [C.POINTER(RecoveryCfg)]
    L.ll_mapper_set_recovery.argtypes = [vp, C.POINTER(RecoveryCfg)]
    L.ll_mapper_recovery_read.argtypes = [vp, C.POINTER(RecoveryStep), ci, C.POINTER(ci), C.POINTER(ci)]
    L.ll_mapper_recovery_last_inputs.argtypes = [vp, C.POINTER(RelocCfg), C.POINTER(RelocFineCfg), C.POINTER(RegState), vp, vp, vp, vp, vp, sz, vp, vp, ci]
    L.ll_pose_graph_create.argtypes = [vp, ci, ci, C.POINTER(vp)]
    L.ll_pose_graph_release.argtypes = [vp]
    L.ll_pose_graph_optimize.argtypes = [vp, vp, ci, vp, ci, ci, C.POINTER(PgSummary)]
    L.ll_pose_graph_step.argtypes = [vp, vp, ci, vp, ci, cd, C.POINTER(cd), vp, vp, vp, C.POINTER(ci)]
    L.ll_pose_graph_loop_edge.argtypes = [vp, vp, C.POINTER(Pose), ci, C.POINTER(Pose), ci, C.POINTER(PgEdge)]
    L.ll_keyframes_repose.argtypes = [vp, vp, sz, vp, ci, vp, vp, cf, vp, vp]
    L.ll_keyframe_affine.argtypes = [C.POINTER(Pose), C.POINTER(Pose), vp, vp]
    L.ll_keyframe_create.argtypes = [vp, C.POINTER(vp)]
    L.ll_keyframe_release.argtypes = [vp]
    L.ll_keyframe_append.argtypes = [vp, vp, vp, sz, ci, ci, vp, ci]
    L.ll_keyframe_analyze.argtypes = [vp, vp, vp, ci, C.POINTER(KeyframeInfo)]
    L.ll_keyframe_get_info.argtypes = [vp, C.POINTER(KeyframeInfo)]
    L.ll_keyframe_cells.argtypes = [vp, vp, vp, vp, vp, vp, ci, C.POINTER(ci)]
    L.ll_keyframe_images.argtypes = [vp, vp, vp, vp, vp, vp]
    L.ll_keyframe_cloud.argtypes = [vp, vp, ci, vp, sz, C.POINTER(sz), C.POINTER(vp)]
    L.ll_loop_cfg_default.argtypes = [C.POINTER(LoopCfg)]
    L.ll_loop_search.argtypes = [vp, vp, ci, ci, C.POINTER(LoopCfg), vp, vp, vp, C.POINTER(ci)]
    L.ll_mapper_loop_closure_default.argtypes = [C.POINTER(LoopClosureCfg)]
    L.ll_mapper_set_loop_closure.argtypes = [vp, C.POINTER(LoopClosureCfg)]
    L.ll_mapper_loop_read.argtypes = [vp, C.POINTER(LoopEvent), ci, C.POINTER(ci), C.POINTER(ci)]
    L.ll_mapper_loop_result.argtypes = [vp, C.POINTER(ci), C.POINTER(ci), vp, vp, ci, C.POINTER(PgEdge)]
    L.ll_mapper_loop_cloud.argtypes = [vp, ci, vp, sz, C.POINTER(sz), C.POINTER(vp)]
    L.ll_spin_cfg_default.argtypes = [C.POINTER(SpinCfg)]
    L.ll_spin_create.argtypes = [vp, C.POINTER(SpinCfg), C.POINTER(vp)]
    L.ll_spin_release.argtypes = [vp]
    L.ll_spin_extract.argtypes = [vp, vp, sz, ci, ci, vp]
    L.ll_spin_cloud.argtypes = [vp, ci, vp, sz, C.POINTER(sz), C.POINTER(vp)]
    L.ll_spin_point_info.argtypes = [vp, vp, vp, vp, vp, sz, C.POINTER(sz)]
    L.ll_spin_chains.argtypes = [vp, C.POINTER(ci), C.POINTER(ci)]
    L.ll_mapper_process_sweep.argtypes = [vp, vp, vp, sz, ci, ci, C.POINTER(RegResult), C.POINTER(MapperStats)]
    L.ll_mapper_process_sweeps.argtypes = [vp, vp, ci, vp, vp, ci, ci, C.POINTER(RegResult), C.POINTER(MapperStats), C.POINTER(ci)]
    L.ll_mapper_loop_save.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.ll_mapper_loop_load.argtypes = [vp, vp, sz, C.POINTER(LoopClosureCfg)]
    L.ll_loop_image_info.argtypes = [vp, sz, C.POINTER(LoopImageSummary)]
    L.ll_mapper_loop_policy_default.argtypes = [C.POINTER(LoopPolicy)]
    L.ll_mapper_set_loop_policy.argtypes = [vp, C.POINTER(LoopPolicy)]
    L.ll_mapper_loop_edges.argtypes = [vp, vp, ci, C.POINTER(ci)]
    L.ll_mapper_set_loop_feedback.argtypes = [vp, ci]
    L.ll_mapper_loop_correction_read.argtypes = [vp, vp, vp, C.POINTER(ci)]
    L.ll_loop_correction.argtypes = [C.POINTER(Pose), C.POINTER(Pose), vp, ci, ci, vp, vp]
    L.ll_launch_count.argtypes = [vp]
    L.ll_launch_count.restype = C.c_uint64
    _LIB = L
    return L


def default_spin_cfg(**kw) -> SpinCfg:
    c = SpinCfg()
    lib().ll_spin_cfg_default(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def default_loop_cfg(**kw) -> LoopCfg:
    c = LoopCfg()
    lib().ll_loop_cfg_default(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def default_config(**kw) -> Config:
    c = Config()
    lib().ll_config_default(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def default_reg_state(**kw) -> RegState:
    s = RegState()
    lib().ll_reg_state_default(C.byref(s))
    for k, v in kw.items():
        if isinstance(getattr(s, k), C.Array):
            getattr(s, k)[:] = list(v)
        else:
            setattr(s, k, v)
    return s


def yaml_reg_state(realtime: bool = False, **kw) -> RegState:
    """The shipped YAML values exactly (cap 200 / 150, max_allow_final_cost 2.0)."""
    s = RegState()
    lib().ll_reg_state_yaml(C.byref(s), int(bool(realtime)))
    for k, v in kw.items():
        if isinstance(getattr(s, k), C.Array):
            getattr(s, k)[:] = list(v)
        else:
            setattr(s, k, v)
    return s


def _ptr(a):
    """numpy array -> (void*, keepalive); int -> raw (device) pointer."""
    if isinstance(a, (int, np.integer)):
        return C.c_void_p(int(a))
    return C.c_void_p(a.ctypes.data)


def _pts(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] in (4, 8), "points must be [n,4] (XYZI16) or [n,8] (pcl::PointXYZI)"
    return a, (LL_FMT_XYZI16 if a.shape[1] == 4 else LL_FMT_PCL32)
