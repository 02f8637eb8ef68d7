"""ctypes loader for libbadba_b200.so (the C ABI of include/badba.h).

There is deliberately NO fallback: if the CUDA library is missing or cannot be loaded the
import of the product path fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libbadba_b200.so")

ABI_VERSION = 10   # BBA_ABI_VERSION of the include/badba.h this binding types

# bba_pose_variant: the pose kernel's instantiations (surfel tile, precomputed per-surfel frames)
POSE_VARIANT_AUTO, POSE_VARIANT_256_PRE, POSE_VARIANT_512_PRE, POSE_VARIANT_256, POSE_VARIANT_512, POSE_VARIANT_1024 = range(6)
GEOMETRY_PASS_AUTO, GEOMETRY_PASS_SPLIT, GEOMETRY_PASS_ONE = range(3)

OK, ERR_INVALID_ARGUMENT, ERR_CUDA, ERR_STATE, ERR_UNSUPPORTED, ERR_NO_DEVICE = range(6)
STATUS_NAMES = {0: "BBA_OK", 1: "BBA_ERR_INVALID_ARGUMENT", 2: "BBA_ERR_CUDA", 3: "BBA_ERR_STATE",
                4: "BBA_ERR_UNSUPPORTED", 5: "BBA_ERR_NO_DEVICE"}


class Config(C.Structure):
    _fields_ = [("depth_width", C.c_int), ("depth_height", C.c_int), ("color_width", C.c_int), ("color_height", C.c_int),
                ("depth_intrinsics", C.c_float * 4), ("color_intrinsics", C.c_float * 4),
                ("raw_to_float_depth", C.c_float), ("baseline_fx", C.c_float),
                ("sparse_surfel_cell_size", C.c_int), ("max_surfel_count", C.c_uint32), ("max_keyframes", C.c_int),
                ("use_depth_residuals", C.c_int), ("use_descriptor_residuals", C.c_int),
                ("device", C.c_int), ("rank", C.c_int), ("world_size", C.c_int),
                ("min_observation_count_while_bootstrapping_1", C.c_int), ("min_observation_count_while_bootstrapping_2", C.c_int),
                ("min_observation_count", C.c_int), ("surfel_merge_dist_factor", C.c_float)]


PROGRESS_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int)   # bba_ba_options::progress_function


class BAOptions(C.Structure):
    _fields_ = [("optimize_depth_intrinsics", C.c_int), ("optimize_color_intrinsics", C.c_int),
                ("do_surfel_updates", C.c_int), ("optimize_poses", C.c_int), ("optimize_geometry", C.c_int),
                ("min_iterations", C.c_int), ("max_iterations", C.c_int), ("use_pcg", C.c_int),
                ("active_keyframe_window_start", C.c_int), ("active_keyframe_window_end", C.c_int),
                ("increase_ba_iteration_count", C.c_int), ("time_limit_seconds", C.c_double),
                ("pcg_max_inner_iterations", C.c_int), ("pcg_max_keyframes", C.c_int), ("pcg_gauge_keyframe", C.c_int),
                ("progress_function", PROGRESS_FN), ("progress_user", C.c_void_p)]


class PcgProbe(C.Structure):   # bba_pcg_probe
    _fields_ = [("r", C.c_void_p), ("M", C.c_void_p), ("p", C.c_void_p), ("g", C.c_void_p), ("delta", C.c_void_p),
                ("alpha_n", C.c_double), ("alpha_d", C.c_double),
                ("r_step2", C.c_void_p), ("delta_step2", C.c_void_p), ("z", C.c_void_p), ("beta_n", C.c_double),
                ("p_step3", C.c_void_p), ("g_step3", C.c_void_p), ("alpha_d_step3", C.c_double)]


class BAResult(C.Structure):
    _fields_ = [("iterations_done", C.c_int), ("converged", C.c_int),
                ("depth_residual_count", C.c_uint64), ("descriptor_residual_count", C.c_uint64), ("cost", C.c_double),
                ("pose_iterations_total", C.c_int),
                ("ms_surfel_activation", C.c_float), ("ms_geometry_optimization", C.c_float),
                ("ms_pose_optimization", C.c_float), ("ms_intrinsics_optimization", C.c_float),
                ("kernel_launches", C.c_uint64),
                ("pcg_inner_iterations_total", C.c_int), ("pcg_last_r_norm", C.c_float), ("ms_pcg", C.c_float),
                ("surfels_deleted", C.c_uint32), ("surfels_size", C.c_uint32),
                ("surfels_created", C.c_uint32), ("surfels_merged", C.c_uint32)]


class PreprocessOptions(C.Structure):
    _fields_ = [("bilateral_filter_sigma_xy", C.c_float), ("bilateral_filter_sigma_inv_depth", C.c_float),
                ("bilateral_filter_radius_factor", C.c_float), ("max_depth", C.c_float)]


class RawFrameOptions(C.Structure):   # bba_raw_frame_options
    _fields_ = [("base", PreprocessOptions), ("median_filter_and_densify_iterations", C.c_int),
                ("pyramid_level_for_depth", C.c_int), ("pyramid_level_for_color", C.c_int)]


class OdometryOptions(C.Structure):
    _fields_ = [("num_scales", C.c_int), ("use_pyramid_level_0", C.c_int), ("use_gradmag", C.c_int),
                ("test_different_initial_estimates", C.c_int), ("max_iterations_per_scale", C.c_int)]


class OdometryResult(C.Structure):
    _fields_ = [("iterations", C.c_int * 8), ("chose_initial", C.c_int * 8), ("residual_count", C.c_uint32),
                ("residual_sum", C.c_float), ("passes", C.c_uint32), ("kernel_launches", C.c_uint32)]


class MotionModelRecord(C.Structure):
    _fields_ = [("count", C.c_int), ("base_kf_tr_frame", (C.c_float * 7) * 3), ("frame_tr_base_kf", (C.c_float * 7) * 3)]


class PoseConstraint(C.Structure):   # bba_pose_constraint
    _fields_ = [("keyframe_a", C.c_int), ("keyframe_b", C.c_int), ("a_T_b", C.c_float * 7), ("information", C.c_float * 21)]


class RobustLoss(C.Structure):   # bba_robust_loss
    _fields_ = [("type", C.c_int), ("scale", C.c_float)]


class AttitudePrior(C.Structure):   # bba_attitude_prior
    _fields_ = [("reference_direction", C.c_float * 3), ("measured_direction", C.c_float * 3), ("information", C.c_float),
                ("loss", RobustLoss)]


class PoseGraphOptions(C.Structure):   # bba_pose_graph_options
    _fields_ = [("gauge_keyframe", C.c_int), ("max_iterations", C.c_int), ("use_odometry_chain", C.c_int),
                ("odometry_information", C.c_float * 21)]


class PoseGraphResult(C.Structure):   # bba_pose_graph_result
    _fields_ = [("iterations", C.c_int), ("converged", C.c_int), ("linear_iterations", C.c_int), ("held_keyframes", C.c_int),
                ("initial_cost", C.c_double), ("final_cost", C.c_double)]


class ExposureOptions(C.Structure):   # bba_exposure_options
    _fields_ = [("gauge_keyframe", C.c_int), ("min_luma", C.c_int), ("max_luma", C.c_int), ("inlier_threshold", C.c_float),
                ("outer_iterations", C.c_int)]


class PeerHandle(C.Structure):
    _fields_ = [("surfels_ipc", C.c_ubyte * 64), ("surfels_offset", C.c_uint64), ("active_ipc", C.c_ubyte * 64),
                ("active_offset", C.c_uint64), ("pitch_bytes", C.c_uint64), ("surfels_size", C.c_uint32), ("rank", C.c_int32)]


class PoseCoeffs(C.Structure):
    _fields_ = [("H", C.c_float * 21), ("b", C.c_float * 6),
                ("n_pair", C.c_uint64), ("n_inimg", C.c_uint64), ("n_depthok", C.c_uint64),
                ("n_assoc", C.c_uint64), ("n_photo", C.c_uint64),
                ("cost_depth", C.c_double), ("cost_desc1", C.c_double), ("cost_desc2", C.c_double)]


class FrameBuffers(C.Structure):   # bba_frame_buffers
    _fields_ = [("depth", C.c_void_p), ("depth_pitch", C.c_size_t), ("normals", C.c_void_p), ("normals_pitch", C.c_size_t),
                ("color_rgba", C.c_void_p), ("color_pitch", C.c_size_t)]


class FrameOverlapQuery(C.Structure):   # bba_frame_overlap_query
    _fields_ = [("frame", C.c_int), ("global_T_frame", C.c_float * 7), ("min_depth", C.c_float), ("max_depth", C.c_float)]


class FrameOverlap(C.Structure):   # bba_frame_overlap
    _fields_ = [("observed_surfels", C.c_uint32), ("valid_cells", C.c_uint32), ("uncovered_cells", C.c_uint32),
                ("new_surfels", C.c_uint32)]


class OdometryEntry(C.Structure):   # bba_odometry_entry
    _fields_ = [("base_keyframe_id", C.c_int), ("base_frame", C.c_int), ("tracked_frame", C.c_int),
                ("base_T_frame_initial_1", C.c_float * 7), ("base_T_frame_initial_2", C.c_float * 7)]


ODOMETRY_CHUNK_ENTRIES = 64   # BBA_ODOMETRY_CHUNK_ENTRIES

# bba_loop_status
LOOP_ACCEPTED, LOOP_NO_NEIGHBOUR, LOOP_ROTATION_DISAGREES, LOOP_TRANSLATION_DISAGREES, LOOP_CORRECTION_TOO_SMALL = range(5)
LOOP_STATUS_NAMES = {0: "ACCEPTED", 1: "NO_NEIGHBOUR", 2: "ROTATION_DISAGREES", 3: "TRANSLATION_DISAGREES", 4: "CORRECTION_TOO_SMALL"}


class LoopCandidate(C.Structure):   # bba_loop_candidate
    _fields_ = [("current_keyframe_id", C.c_int), ("matched_keyframe_id", C.c_int), ("old_T_cur_initial", C.c_float * 7)]


class LoopVerificationOptions(C.Structure):   # bba_loop_verification_options
    _fields_ = [("odometry", OdometryOptions), ("max_angle_difference", C.c_float), ("max_translation_difference", C.c_float),
                ("max_pixel_distance", C.c_float)]


class LoopVerification(C.Structure):   # bba_loop_verification
    _fields_ = [("status", C.c_int), ("tracked_keyframe_ids", C.c_int * 3), ("cur_T_old_refined", (C.c_float * 7) * 3),
                ("cur_T_old", C.c_float * 7), ("angle_difference", C.c_float), ("translation_difference", C.c_float),
                ("average_pixel_distance", C.c_float), ("pixel_count", C.c_uint32), ("tracking", OdometryResult * 3)]


class PlaceIndexOptions(C.Structure):   # bba_place_index_options
    _fields_ = [("num_ferns", C.c_int), ("min_depth", C.c_float), ("max_depth", C.c_float)]


class PlaceQuery(C.Structure):   # bba_place_query
    _fields_ = [("keyframe_id", C.c_int), ("frame", C.c_int), ("first_keyframe", C.c_int), ("last_keyframe", C.c_int)]


PLACE_MAX_MATCHES = 64   # the largest max_matches of bba_query_place_index


class Profile(C.Structure):
    _fields_ = [("pose_launches", C.c_uint64), ("pose_ms", C.c_double), ("kf_evals", C.c_uint64),
                ("n_pair", C.c_uint64), ("n_inimg", C.c_uint64), ("n_depthok", C.c_uint64),
                ("n_assoc", C.c_uint64), ("n_photo", C.c_uint64),
                ("geometry_launches", C.c_uint64), ("activation_normals_ms", C.c_double),
                ("position_descriptor_ms", C.c_double)]


COLLECTIVE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p)
COLLECTIVE_ALLGATHER, COLLECTIVE_ALLREDUCE_SUM = 0, 1

# every symbol include/badba.h declares: (name, restype, argtypes)
_P = C.c_void_p
_F7 = C.POINTER(C.c_float)
SYMBOLS = {
    "bba_abi_version": (C.c_int, []),
    "bba_create": (C.c_int, [C.POINTER(Config), C.POINTER(_P)]),
    "bba_destroy": (None, [_P]),
    "bba_last_error": (C.c_char_p, [_P]),
    "bba_set_surfels": (C.c_int, [_P, _P, C.c_size_t, C.c_uint32]),
    "bba_set_active_flags": (C.c_int, [_P, _P]),
    "bba_set_surfels_host": (C.c_int, [_P, _P, C.c_size_t, C.c_uint32, _P]),
    "bba_get_surfels_host": (C.c_int, [_P, _P, C.c_size_t, C.c_int, _P]),
    "bba_get_active_flags_host": (C.c_int, [_P, _P, _P]),
    "bba_get_surfels_device": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_size_t), C.POINTER(C.c_uint32)]),
    "bba_add_keyframe": (C.c_int, [_P, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, _F7,
                                   C.c_float, C.c_float, _P, C.POINTER(C.c_int)]),
    "bba_add_keyframe_host": (C.c_int, [_P, _P, _P, _P, _P, _F7, C.c_float, C.c_float, _P, C.POINTER(C.c_int)]),
    "bba_keyframe_count": (C.c_int, [_P]),
    "bba_set_keyframe_pose": (C.c_int, [_P, C.c_int, _F7]),
    "bba_get_keyframe_pose": (C.c_int, [_P, C.c_int, _F7]),
    "bba_set_keyframe_activation": (C.c_int, [_P, C.c_int, C.c_int]),
    "bba_get_keyframe_activation": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int)]),
    "bba_set_keyframe_states": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_get_keyframe_states": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_get_covisibility": (C.c_int, [_P, C.c_int, _P]),
    "bba_set_keyframe_pose_priors": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "bba_clear_keyframe_pose_priors": (C.c_int, [_P, C.c_int, _P]),
    "bba_get_keyframe_pose_prior": (C.c_int, [_P, C.c_int, _P, _P, C.POINTER(C.c_int)]),
    "bba_add_keyframe_pose_constraints": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_remove_keyframe_pose_constraints": (C.c_int, [_P, C.c_int, _P]),
    "bba_get_keyframe_pose_constraints": (C.c_int, [_P, C.c_int, _P, _P, C.POINTER(C.c_int)]),
    "bba_set_keyframe_pose_prior_losses": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_set_keyframe_pose_constraint_losses": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_get_keyframe_pose_prior_loss": (C.c_int, [_P, C.c_int, C.POINTER(RobustLoss)]),
    "bba_get_keyframe_pose_constraint_losses": (C.c_int, [_P, C.c_int, _P, _P, C.POINTER(C.c_int)]),
    "bba_evaluate_keyframe_pose_terms": (C.c_int, [_P, C.c_int, _P, _P, C.c_int, _P, _P, _P]),
    "bba_set_keyframe_attitude_priors": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_clear_keyframe_attitude_priors": (C.c_int, [_P, C.c_int, _P]),
    "bba_get_keyframe_attitude_prior": (C.c_int, [_P, C.c_int, C.POINTER(AttitudePrior), C.POINTER(C.c_int)]),
    "bba_evaluate_keyframe_attitude_priors": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "bba_set_intrinsics": (C.c_int, [_P, _F7, _F7, C.c_float]),
    "bba_get_intrinsics": (C.c_int, [_P, _F7, _F7, C.POINTER(C.c_float)]),
    "bba_host_se3_exp": (None, [_P, _P]),
    "bba_host_se3_log": (None, [_P, _P]),
    "bba_host_se3_compose": (None, [_P, _P, _P]),
    "bba_host_se3_inverse": (None, [_P, _P]),
    "bba_host_pose_update_converged": (C.c_int, [_P]),
    "bba_host_solve_ldlt": (C.c_int, [C.c_int, _P, _P, _P]),
    "bba_host_pose_prior_terms": (None, [_P, _P, _P, _P, _P, C.POINTER(C.c_double)]),
    "bba_host_pose_constraint_terms": (None, [_P, _P, _P, _P, _P, _P, C.POINTER(C.c_double)]),
    "bba_host_robust_loss": (None, [C.c_int, C.c_float, C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "bba_host_attitude_prior_terms": (None, [_P, _P, C.c_float, _P, _P, _P, C.POINTER(C.c_double)]),
    "bba_host_average_pose": (None, [C.c_int, _P, _P]),
    "bba_host_loop_agreement": (C.c_int, [_P, C.c_float, C.c_float, _P, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "bba_host_frusta_intersect": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_float, C.c_float, _P, C.c_float, C.c_float]),
    "bba_host_motion_model_clear": (None, [C.POINTER(MotionModelRecord), _P, _P]),
    "bba_host_motion_model_predict": (C.c_int, [C.POINTER(MotionModelRecord), C.c_int, _P, _P]),
    "bba_host_motion_model_push": (None, [C.POINTER(MotionModelRecord), _P]),
    "bba_host_motion_model_rebase": (None, [C.POINTER(MotionModelRecord)]),
    "bba_host_deform_trajectory": (C.c_int, [C.c_int, _P, _P, _P, C.c_int, C.c_int, _P]),
    "bba_set_residual_types": (C.c_int, [_P, C.c_int, C.c_int]),
    "bba_get_residual_types": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "bba_set_cfactor_host": (C.c_int, [_P, _P, _P]),
    "bba_get_cfactor_host": (C.c_int, [_P, _P, _P]),
    "bba_cfactor_size": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "bba_accumulate_pose_coeffs": (C.c_int, [_P, C.c_int, _F7, C.POINTER(PoseCoeffs), _P]),
    "bba_debug_pose_coeffs_batch": (C.c_int, [_P, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "bba_debug_set_pose_group": (C.c_int, [_P, C.c_int]),
    "bba_debug_set_geometry_pass": (C.c_int, [_P, C.c_int, C.c_int]),
    "bba_estimate_frame_pose": (C.c_int, [_P, C.c_int, _F7, _F7, C.POINTER(C.c_int), C.POINTER(C.c_int), _P]),
    "bba_estimate_frame_pose_for_frame": (C.c_int, [_P, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, _F7, _F7,
                                                    C.POINTER(C.c_int), C.POINTER(C.c_int), _P]),
    "bba_estimate_frame_poses_for_frames": (C.c_int, [_P, C.c_int, C.POINTER(FrameBuffers), C.c_int, _P, _P, _P, _P, _P,
                                                      C.POINTER(PoseCoeffs), _P]),
    "bba_track_frame_pairwise": (C.c_int, [_P, C.POINTER(OdometryOptions), C.c_int, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t,
                                           _F7, _F7, _F7, C.POINTER(OdometryResult), _P]),
    "bba_track_frames_pairwise": (C.c_int, [_P, C.POINTER(OdometryOptions), C.c_int, C.POINTER(FrameBuffers), C.c_int,
                                            C.POINTER(OdometryEntry), _P, C.POINTER(OdometryResult), C.POINTER(C.c_uint32), _P]),
    "bba_track_frame_pairwise_to_frame": (C.c_int, [_P, C.POINTER(OdometryOptions), _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t,
                                                    _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, _F7, _F7, _F7,
                                                    C.POINTER(OdometryResult), _P]),
    "bba_verify_loop_closures": (C.c_int, [_P, C.POINTER(LoopVerificationOptions), C.c_int, C.POINTER(LoopCandidate),
                                           C.POINTER(LoopVerification), _P]),
    "bba_index_keyframes": (C.c_int, [_P, C.POINTER(PlaceIndexOptions), C.c_int, _P, _P]),
    "bba_query_place_index": (C.c_int, [_P, C.c_int, C.POINTER(FrameBuffers), C.c_int, C.POINTER(PlaceQuery), C.c_int, _P, _P, _P, _P]),
    "bba_get_place_index_codes": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P]),
    "bba_get_place_index_options": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "bba_host_place_ferns": (C.c_int, [C.c_int, C.c_int, C.c_int, _P, _P]),
    "bba_odometry_get_level": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, C.POINTER(C.c_int), C.POINTER(C.c_int), _P]),
    "bba_odometry_debug_coeffs": (C.c_int, [_P, C.c_int, C.c_int, _F7, _F7, _P, _P, C.POINTER(C.c_uint32), C.POINTER(C.c_float),
                                            _P, _P, _P]),
    "bba_update_surfel_activation": (C.c_int, [_P, _P]),
    "bba_optimize_geometry_iteration": (C.c_int, [_P, _P]),
    "bba_deform_surfels": (C.c_int, [_P, C.c_int, _P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), _P]),
    "bba_measure_keyframe_covisibility": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, _P]),
    "bba_debug_set_covisibility_chunk": (C.c_int, [_P, C.c_uint32]),
    "bba_estimate_keyframe_exposures": (C.c_int, [_P, C.POINTER(ExposureOptions), C.c_int, _P, _P, _P, _P, _P]),
    "bba_set_keyframe_exposures": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "bba_get_keyframe_exposures": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_debug_get_exposure_system": (C.c_int, [_P, C.c_int, _P, _P]),
    "bba_measure_frame_overlap": (C.c_int, [_P, C.c_int, C.POINTER(FrameBuffers), C.c_int, C.POINTER(FrameOverlapQuery), C.c_int, _P,
                                            C.POINTER(FrameOverlap), _P]),
    "bba_optimize_pose_graph": (C.c_int, [_P, C.POINTER(PoseGraphOptions), C.POINTER(PoseGraphResult), _P]),
    "bba_optimize_intrinsics": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "bba_debug_intrinsics_coeffs": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P]),
    "bba_perform_end_tasks": (C.c_int, [_P, C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), _P]),
    "bba_surfels_size": (C.c_uint32, [_P]),
    "bba_get_ba_iteration_counts": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "bba_set_ba_iteration_counts": (C.c_int, [_P, C.c_int, C.c_int]),
    "bba_create_surfels_for_keyframe": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(C.c_uint32), _P]),
    "bba_merge_surfels_for_keyframe": (C.c_int, [_P, C.c_int, C.POINTER(C.c_uint32), _P]),
    "bba_compact_surfels": (C.c_int, [_P, C.c_uint32, C.c_int, C.POINTER(C.c_uint32), _P]),
    "bba_preprocess_frame": (C.c_int, [_P, C.POINTER(PreprocessOptions), _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t,
                                       _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "bba_preprocess_raw_frame": (C.c_int, [_P, C.POINTER(RawFrameOptions), _P, C.c_size_t, C.c_int, C.c_int, _P, C.c_size_t, C.c_int,
                                           C.c_int, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t,
                                           C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "bba_pcg_debug": (C.c_int, [_P, C.POINTER(BAOptions), C.c_int, C.c_int, C.POINTER(C.c_uint32), C.POINTER(PcgProbe), _P]),
    "bba_bundle_adjust": (C.c_int, [_P, C.POINTER(BAOptions), C.POINTER(BAResult), _P]),
    "bba_peer_export": (C.c_int, [_P, _P]),
    "bba_peer_import": (C.c_int, [_P, _P, C.c_int]),
    "bba_peer_count": (C.c_int, [_P]),
    "bba_peer_unmap": (C.c_int, [_P]),
    "bba_mark_replica_rewritten": (C.c_int, [_P]),
    "bba_set_collective": (C.c_int, [_P, COLLECTIVE_FN, _P]),
    "bba_local_group_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, C.POINTER(_P)]),
    "bba_local_group_reset": (C.c_int, [_P]),
    "bba_local_group_poison": (C.c_int, [_P]),
    "bba_local_group_destroy": (None, [_P]),
    "bba_debug_collective": (C.c_int, [_P, C.c_int, _P, C.c_size_t, _P]),
    "bba_shard_surfel_owner": (C.c_int, [C.c_uint32, C.c_int]),
    "bba_shard_surfel_local_index": (C.c_uint32, [C.c_uint32, C.c_int]),
    "bba_shard_slice_length": (C.c_uint32, [C.c_uint32, C.c_int]),
    "bba_shard_keyframe_owner": (C.c_int, [C.c_int, C.c_int]),
    "bba_balance_keyframes": (None, [_P, C.c_int, C.c_int, _P]),
    "bba_kernel_launch_count": (C.c_uint64, [_P]),
    "bba_update_keyframe_host": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P]),
    "bba_set_deterministic": (C.c_int, [_P, C.c_int]),
    "bba_get_deterministic": (C.c_int, [_P, C.POINTER(C.c_int)]),
    "bba_debug_exact_sum": (C.c_int, [_P, _P, C.c_uint64, C.POINTER(C.c_double), _P]),
    "bba_host_exact_sum": (None, [_P, C.c_size_t, C.POINTER(C.c_double)]),
    "bba_set_profiling": (C.c_int, [_P, C.c_int]),
    "bba_get_profile": (C.c_int, [_P, C.POINTER(Profile), C.c_int]),
}

_lib = None


def load():
    """Loads the shared library and types every exported symbol.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -m badslam_b200.build` "
                          "(there is no CPU / eager fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SYMBOLS.items():
        fn = getattr(lib, name)   # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.bba_abi_version() != ABI_VERSION:
        raise ImportError(f"libbadba_b200.so ABI version {lib.bba_abi_version()}, this binding expects {ABI_VERSION}")
    _lib = lib
    return lib


class BadBAError(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"{STATUS_NAMES.get(status, status)}: {message}")
        self.status = status
