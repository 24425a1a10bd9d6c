"""ctypes binding of the C ABI declared in include/se2gpu.h (the drop-in boundary).

Loading fails loudly if the CUDA library has not been built: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import build as _build

KP_DTYPE = np.dtype([("x", "f4"), ("y", "f4"), ("size", "f4"), ("angle", "f4"), ("response", "f4"),
                     ("octave", "i4"), ("class_id", "i4")])
assert KP_DTYPE.itemsize == 28
BA_STATS_DTYPE = np.dtype([("chi2_before", "f8"), ("chi2_after", "f8"), ("lambda", "f8"), ("rho", "f8"),
                           ("trials", "i4"), ("accepted", "i4"), ("terminate", "i4"), ("pad", "i4")])

ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p)


class GridParams(C.Structure):
    _fields_ = [("min_x", C.c_float), ("min_y", C.c_float), ("inv_w", C.c_float), ("inv_h", C.c_float)]


class BowKF(C.Structure):
    _fields_ = [("angle", C.c_void_p), ("desc", C.c_void_p), ("has_mp", C.c_void_p), ("n", C.c_int),
                ("node", C.c_void_p), ("n_node", C.c_int), ("ptr", C.c_void_p), ("feat", C.c_void_p)]


class BowBatchKF(C.Structure):
    """se2gpu_bow_batch_kf: one side of se2gpu_search_by_bow_batch_device (device pointers)"""
    _fields_ = [("kp", C.c_void_p), ("desc", C.c_void_p), ("has_mp", C.c_void_p), ("cap", C.c_int), ("node", C.c_void_p),
                ("ptr", C.c_void_p), ("feat", C.c_void_p), ("n_node", C.c_void_p)]


class LoopDetectParams(C.Structure):
    """se2gpu_loop_detect_params"""
    _fields_ = [("min_id_offset", C.c_int), ("min_score", C.c_double)]


class LoopVerifyParams(C.Structure):
    """se2gpu_loop_verify_params"""
    _fields_ = [("localizer", C.c_int), ("min_match_mp", C.c_int), ("min_match_kp", C.c_int), ("ratio_min_match_mp", C.c_double)]


class PoseBAParams(C.Structure):
    _fields_ = [("fx", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("Tbc", C.c_float * 16), ("huber_delta", C.c_float),
                ("xrot_info", C.c_float), ("yrot_info", C.c_float), ("z_info", C.c_float), ("iterations", C.c_int)]


class FeatEdgeParams(C.Structure):
    _fields_ = [("Tbc", C.c_float * 16), ("xrot_info", C.c_float), ("yrot_info", C.c_float), ("z_info", C.c_float),
                ("huber_delta", C.c_float), ("iterations", C.c_int * 2), ("chi2_cut", C.c_float), ("min_points", C.c_int * 2)]


class GlobalBAParams(C.Structure):
    _fields_ = [("Tbc", C.c_float * 16), ("xrot_info", C.c_float), ("yrot_info", C.c_float), ("z_info", C.c_float),
                ("iterations", C.c_int)]


class SE3BAParams(C.Structure):
    _fields_ = [("fx", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("Tbc", C.c_float * 16), ("huber_delta", C.c_float),
                ("xrot_info", C.c_float), ("yrot_info", C.c_float), ("z_info", C.c_float), ("iterations", C.c_int),
                ("chi2_cut", C.c_float)]


vp_ = C.c_void_p


class MpKeyframes(C.Structure):
    """se2gpu_mp_keyframes"""
    _fields_ = [("n_kf", C.c_int), ("kf_id", vp_), ("kf_null", vp_), ("Tcw", vp_), ("kp_base", vp_), ("n_slots", C.c_int),
                ("kp", vp_), ("desc", vp_), ("view_mp", vp_), ("view_info", vp_)]


class MpPoints(C.Structure):
    """se2gpu_mp_points"""
    _fields_ = [("n_mp", C.c_int), ("pos", vp_), ("good_prl", vp_), ("null", vp_), ("main_kf", vp_), ("main_desc", vp_),
                ("main_octave", vp_), ("main_measure", vp_), ("level_scale", vp_), ("normal", vp_), ("min_dist", vp_),
                ("max_dist", vp_), ("obs_ptr", vp_), ("obs_kf", vp_), ("obs_idx", vp_)]


MP_MAX_LEVELS = 32   # SE2GPU_MP_MAX_LEVELS


class MpParams(C.Structure):
    """se2gpu_mp_params"""
    _fields_ = [("K", C.c_float * 9), ("lower_depth", C.c_float), ("upper_depth", C.c_float), ("fx", C.c_float),
                ("nlevels", C.c_int), ("scale_factors", C.c_float * MP_MAX_LEVELS)]


class TrackerParams(C.Structure):
    """se2gpu_tracker_params"""
    _fields_ = [("nfeatures", C.c_int), ("scale_factor", C.c_float), ("nlevels", C.c_int), ("fast_th", C.c_int),
                ("K", C.c_float * 9), ("dist", C.c_float * 12), ("ndist", C.c_int), ("grid", GridParams),
                ("lower_depth", C.c_float), ("upper_depth", C.c_float), ("cTb", C.c_float * 16), ("bTc", C.c_float * 16),
                ("odo_noise", C.c_float * 3), ("min_frames", C.c_int), ("max_frames", C.c_int)]


class TrackKF(C.Structure):
    """se2gpu_track_kf"""
    _fields_ = [("d_observed", vp_), ("d_view_mp", vp_), ("n_obs_mp", C.c_int), ("accept_new_kf", C.c_int),
                ("odom", C.c_float * 3)]


TRACK_RESULT_FIELDS = ["frame_id", "first", "n_keypoints", "n_matched", "n_inlier", "n_tracked_old", "n_good_prl",
                       "triangulated", "new_kf", "abort_ba"]


class TrackResult(C.Structure):
    """se2gpu_track_result"""
    _fields_ = [(n, C.c_int) for n in TRACK_RESULT_FIELDS]


class TrackState(C.Structure):
    """se2gpu_track_state"""
    _fields_ = [("d_ref_kp", vp_), ("d_ref_desc", vp_), ("d_ref_n", vp_), ("d_cur_kp", vp_), ("d_cur_desc", vp_),
                ("d_cur_n", vp_), ("d_prev", vp_), ("d_matches", vp_), ("d_local_mps", vp_), ("d_good_prl", vp_),
                ("Tcr", C.c_float * 16), ("pre_meas", C.c_double * 3), ("pre_cov", C.c_double * 9), ("frame_id", C.c_int),
                ("kf_id", C.c_int), ("has_ref", C.c_int), ("n_good_prl", C.c_int)]


class LocMap(C.Structure):
    """se2gpu_loc_map"""
    _fields_ = [("n_kf", C.c_int), ("n_mp", C.c_int), ("kf_Tcw", vp_), ("kf_kp_ptr", vp_), ("kf_obs_mp", vp_), ("kf_obs_ptr", vp_),
                ("kf_obs", vp_), ("kf_cov_ptr", vp_), ("kf_cov", vp_), ("mp_pos", vp_), ("mp_null", vp_), ("mp_good_prl", vp_),
                ("mp_desc", vp_), ("mp_octave", vp_)]


class LocParams(C.Structure):
    """se2gpu_loc_params"""
    _fields_ = [("nfeatures", C.c_int), ("scale_factor", C.c_float), ("nlevels", C.c_int), ("fast_th", C.c_int),
                ("K", C.c_float * 9), ("dist", C.c_float * 12), ("ndist", C.c_int), ("grid", GridParams),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("cTb", C.c_float * 16), ("bTc", C.c_float * 16), ("ba", PoseBAParams), ("inv_level_sigma2", C.c_float * 16),
                ("max_local_mps", C.c_int)]


LOC_RESULT_FIELDS = ["tracked", "first", "n_keypoints", "n_matched", "n_obs_mp", "ba_status", "ba_iterations", "n_local_kfs",
                     "n_local_mps", "overflow"]


class LocResult(C.Structure):
    """se2gpu_loc_result"""
    _fields_ = [(n, C.c_int) for n in LOC_RESULT_FIELDS] + [("Tcw", C.c_float * 16)]


class LocStreamState(C.Structure):
    """se2gpu_loc_stream_state"""
    _fields_ = [("d_kp", vp_), ("d_desc", vp_), ("d_n", vp_), ("d_obs_mp", vp_), ("d_local_mps", vp_), ("d_n_local_mps", vp_),
                ("d_local_kfs", vp_), ("d_covis_kfs", vp_), ("Tcw", C.c_float * 16), ("has_frame", C.c_int), ("tracked", C.c_int),
                ("overflow", C.c_int)]


class Se2GpuError(RuntimeError):
    pass


_lib = None

# every symbol include/se2gpu.h declares (tests/test_abi.py checks the header against this list)
PEER_HANDLE_BYTES = 128   # SE2GPU_BA_PEER_HANDLE_BYTES

SYMBOLS = [
    "se2gpu_device_count", "se2gpu_last_error", "se2gpu_launch_count",
    "se2gpu_orb_create", "se2gpu_orb_create_scored", "se2gpu_orb_destroy", "se2gpu_orb_extract", "se2gpu_orb_extract_device", "se2gpu_orb_submit", "se2gpu_orb_wait",
    "se2gpu_orb_level_dims", "se2gpu_orb_get_level", "se2gpu_orb_profile", "se2gpu_orb_profile_read",
    "se2gpu_orb_debug_nth_element", "se2gpu_orb_debug_nth_element_f32", "se2gpu_orb_set_undistort", "se2gpu_orb_debug_undistort_map",
    "se2gpu_hamming_distance", "se2gpu_match_by_window", "se2gpu_match_by_projection", "se2gpu_search_by_bow",
    "se2gpu_matcher_create", "se2gpu_matcher_destroy", "se2gpu_match_by_window_device", "se2gpu_keypoints_to_points_device",
    "se2gpu_match_by_projection_device", "se2gpu_matcher_match_by_window", "se2gpu_matcher_match_by_projection",
    "se2gpu_matcher_search_by_bow", "se2gpu_matcher_profile", "se2gpu_matcher_profile_read", "se2gpu_matcher_last_rounds",
    "se2gpu_matcher_create_batch", "se2gpu_match_by_window_batch_device", "se2gpu_match_by_projection_batch_device",
    "se2gpu_matcher_last_rounds_batch", "se2gpu_search_by_bow_batch_device", "se2gpu_detect_loop_device", "se2gpu_verify_loop_device",
    "se2gpu_ba_create", "se2gpu_ba_destroy", "se2gpu_ba_set_problem", "se2gpu_ba_optimize", "se2gpu_ba_get",
    "se2gpu_ba_set_shard", "se2gpu_ba_peer_export", "se2gpu_ba_peer_import", "se2gpu_ba_set_stream", "se2gpu_ba_debug_system", "se2gpu_ba_reset", "se2gpu_ba_profile",
    "se2gpu_ba_profile_read", "se2gpu_ba_set_mode", "se2gpu_ba_get_f32", "se2gpu_ba_build_information", "se2gpu_ba_optimize_from", "se2gpu_ba_peer_attach_local",
    "se2gpu_ba_debug_plan", "se2gpu_ba_set_problem_device", "se2gpu_ba_build_information_device", "se2gpu_ba_debug_structure",
    "se2gpu_ba_optimize_batch", "se2gpu_ba_batch_cluster",
    "se2gpu_voc_create", "se2gpu_voc_destroy", "se2gpu_voc_transform", "se2gpu_voc_transform_device", "se2gpu_voc_compute_bow_device",
    "se2gpu_median_descriptor",
    "se2gpu_triangulate", "se2gpu_triangulate_device", "se2gpu_track_triangulate", "se2gpu_track_triangulate_device",
    "se2gpu_xyz_info", "se2gpu_xyz_info_device", "se2gpu_projection_observations", "se2gpu_projection_observations_device",
    "se2gpu_debug_svd4", "se2gpu_remove_outliers", "se2gpu_remove_outliers_device", "se2gpu_fundam_niters_table",
    "se2gpu_fundam_debug_niters",
    "se2gpu_pose_ba", "se2gpu_pose_ba_device", "se2gpu_pose_ba_debug_trace", "se2gpu_localizer_create", "se2gpu_localizer_destroy",
    "se2gpu_localizer_ba_device",
    "se2gpu_feat_edge", "se2gpu_feat_edge_device", "se2gpu_feat_edge_debug_trace",
    "se2gpu_global_ba_create", "se2gpu_global_ba_destroy", "se2gpu_global_ba", "se2gpu_global_ba_device",
    "se2gpu_global_ba_update_points", "se2gpu_global_ba_update_points_device", "se2gpu_global_ba_profile",
    "se2gpu_global_ba_profile_read",
    "se2gpu_se3_ba_create", "se2gpu_se3_ba_destroy", "se2gpu_se3_ba", "se2gpu_se3_ba_device", "se2gpu_se3_ba_debug_trace",
    "se2gpu_mp_add_observations", "se2gpu_mp_erase_observations", "se2gpu_mp_update_measure",
    "se2gpu_mp_add_observations_device", "se2gpu_mp_erase_observations_device", "se2gpu_mp_update_measure_device",
    "se2gpu_track_triangulate_batch_device", "se2gpu_tracker_create", "se2gpu_tracker_destroy", "se2gpu_tracker_step",
    "se2gpu_tracker_first", "se2gpu_tracker_reset", "se2gpu_tracker_state", "se2gpu_tracker_graph_nodes",
    "se2gpu_tracker_debug_eager", "se2gpu_track_host_pose", "se2gpu_track_host_decide",
    "se2gpu_loc_create", "se2gpu_loc_destroy", "se2gpu_loc_step", "se2gpu_loc_relocalize", "se2gpu_loc_state",
    "se2gpu_loc_graph_nodes", "se2gpu_loc_debug_eager", "se2gpu_loc_host_pose",
]


def lib_path() -> str:
    return _build.LIB_PATH


def lib():
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise Se2GpuError(
            f"{path} is missing: build it with `python -m se2lam_b200.build` (or __graft_entry__.build()). "
            "se2lam_b200 has no CPU fallback.")
    L = C.CDLL(path)
    vp, i, f, d, sz = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t
    L.se2gpu_device_count.restype = i
    L.se2gpu_last_error.restype = C.c_char_p
    L.se2gpu_launch_count.restype = C.c_ulonglong
    L.se2gpu_orb_create.restype = vp
    L.se2gpu_orb_create.argtypes = [i, f, i, i, i, i, i, i]
    L.se2gpu_orb_create_scored.restype = vp
    L.se2gpu_orb_create_scored.argtypes = [i, f, i, i, i, i, i, i, i]
    L.se2gpu_orb_destroy.argtypes = [vp]
    L.se2gpu_orb_extract.argtypes = [vp, vp, i, i, i, i, sz, vp, vp, vp]
    L.se2gpu_orb_submit.argtypes = [vp, vp, i, i, i, i, sz, vp, vp, vp]
    L.se2gpu_orb_wait.argtypes = [vp]
    L.se2gpu_orb_extract_device.argtypes = [vp, vp, i, i, i, i, sz, vp, vp, vp, vp]
    L.se2gpu_orb_level_dims.argtypes = [vp, i, C.POINTER(i), C.POINTER(i), C.POINTER(i)]
    L.se2gpu_orb_get_level.argtypes = [vp, i, i, i, vp]
    L.se2gpu_orb_profile.argtypes = [vp, i]
    L.se2gpu_orb_profile_read.argtypes = [vp, vp, vp]
    L.se2gpu_orb_debug_nth_element.argtypes = [vp, vp, vp, i, i]
    L.se2gpu_orb_debug_nth_element_f32.argtypes = [vp, vp, vp, i, vp, i]
    L.se2gpu_orb_set_undistort.argtypes = [vp, vp, vp, i]
    L.se2gpu_orb_debug_undistort_map.argtypes = [vp, vp, i, i, i, vp, vp]
    L.se2gpu_ba_reset.argtypes = [vp]
    L.se2gpu_ba_peer_export.argtypes = [vp, vp]
    L.se2gpu_ba_peer_import.argtypes = [vp, vp, i]
    L.se2gpu_ba_profile.argtypes = [vp, i]
    L.se2gpu_ba_set_mode.argtypes = [vp, i]
    L.se2gpu_ba_profile_read.argtypes = [vp, vp, vp]
    L.se2gpu_hamming_distance.argtypes = [vp, vp, i, vp, i]
    L.se2gpu_match_by_window.argtypes = [vp, vp, i, vp, vp, i, vp, GridParams, i, i, i, i, f, vp, i]
    L.se2gpu_match_by_projection.argtypes = [vp, vp, i, vp, vp, vp, i, vp, vp, GridParams, i, i, f, vp, i]
    L.se2gpu_search_by_bow.argtypes = [C.POINTER(BowKF), C.POINTER(BowKF), i, f, i, vp, i]
    L.se2gpu_matcher_create.restype = vp
    L.se2gpu_matcher_create.argtypes = [i, i, i]
    L.se2gpu_matcher_create_batch.restype = vp
    L.se2gpu_matcher_create_batch.argtypes = [i, i, i, i]
    L.se2gpu_matcher_destroy.argtypes = [vp]
    L.se2gpu_match_by_window_device.argtypes = [vp, vp, vp, i, vp, vp, vp, i, vp, vp, GridParams, i, i, i, i, f, vp, vp, vp]
    L.se2gpu_keypoints_to_points_device.argtypes = [vp, i, vp, vp, vp]
    L.se2gpu_match_by_projection_device.argtypes = [vp, vp, vp, i, vp, vp, vp, vp, i, vp, vp, GridParams, i, i, f, vp, vp, vp]
    L.se2gpu_match_by_window_batch_device.argtypes = [vp, i, vp, vp, i, vp, vp, vp, i, vp, vp, GridParams, i, i, i, i, f, vp, vp, vp]
    L.se2gpu_match_by_projection_batch_device.argtypes = [vp, i, vp, vp, i, vp, vp, vp, vp, i, vp, vp, GridParams, i, i, f, vp, vp, vp]
    L.se2gpu_matcher_match_by_window.argtypes = [vp, vp, vp, i, vp, vp, i, vp, GridParams, i, i, i, i, f, vp]
    L.se2gpu_matcher_match_by_projection.argtypes = [vp, vp, vp, i, vp, vp, vp, i, vp, vp, GridParams, i, i, f, vp]
    L.se2gpu_matcher_search_by_bow.argtypes = [vp, C.POINTER(BowKF), C.POINTER(BowKF), i, f, i, vp]
    L.se2gpu_matcher_profile.argtypes = [vp, i]
    L.se2gpu_matcher_profile_read.argtypes = [vp, vp, vp]
    L.se2gpu_matcher_last_rounds.argtypes = [vp, C.POINTER(i), C.POINTER(i)]
    L.se2gpu_matcher_last_rounds_batch.argtypes = [vp, i, vp, vp]
    L.se2gpu_search_by_bow_batch_device.argtypes = [vp, i, C.POINTER(BowBatchKF), C.POINTER(BowBatchKF), vp, i, f, i, vp, vp, vp]
    L.se2gpu_detect_loop_device.argtypes = [i, vp, vp, vp, i, i, vp, vp, vp, i, vp, vp, C.POINTER(LoopDetectParams), vp, vp, vp, vp]
    L.se2gpu_verify_loop_device.argtypes = [vp, i, C.POINTER(BowBatchKF), C.POINTER(BowBatchKF), vp, vp, C.POINTER(LoopVerifyParams),
                                            vp, vp, vp, vp, vp, vp]
    L.se2gpu_ba_create.restype = vp
    L.se2gpu_ba_create.argtypes = [i, i, i, i, i]
    L.se2gpu_ba_destroy.argtypes = [vp]
    L.se2gpu_ba_set_problem.argtypes = [vp, i, i, i, i] + [vp] * 11 + [d, d, d, vp, d]
    L.se2gpu_ba_optimize.argtypes = [vp, i, vp, vp, vp, vp]
    L.se2gpu_ba_get.argtypes = [vp, vp, vp]
    L.se2gpu_ba_set_shard.argtypes = [vp, i, i, ALLREDUCE_FN, vp]
    L.se2gpu_ba_set_stream.argtypes = [vp, vp]
    L.se2gpu_ba_debug_system.argtypes = [vp, d] + [vp] * 10
    L.se2gpu_ba_debug_plan.argtypes = [vp, vp, i]
    L.se2gpu_ba_get_f32.argtypes = [vp, vp, vp]
    L.se2gpu_ba_optimize_from.argtypes = [vp, i, i, vp, vp, vp, vp]
    L.se2gpu_ba_peer_attach_local.argtypes = [vp, i]
    L.se2gpu_ba_optimize_batch.argtypes = [vp, i, i, vp, vp, vp, vp, vp]
    L.se2gpu_ba_batch_cluster.argtypes = [vp]
    L.se2gpu_ba_build_information.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, i, f, f, f, vp, i]
    L.se2gpu_ba_set_problem_device.argtypes = [vp, i, i, i, i] + [vp] * 11 + [d, d, d, vp, d]
    L.se2gpu_ba_build_information_device.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, i, f, f, f, vp, vp]
    L.se2gpu_ba_debug_structure.argtypes = [vp, i, vp, i]
    L.se2gpu_voc_create.restype = vp
    L.se2gpu_voc_create.argtypes = [i, vp, vp, vp, vp, vp, i, i]
    L.se2gpu_voc_destroy.argtypes = [vp]
    L.se2gpu_voc_transform.argtypes = [vp, vp, i, i, vp, vp, vp]
    L.se2gpu_voc_transform_device.argtypes = [vp, vp, i, i, vp, vp, vp, vp]
    L.se2gpu_voc_compute_bow_device.argtypes = [vp, i, vp, i, vp, i] + [vp] * 8
    L.se2gpu_median_descriptor.argtypes = [vp, vp, i, vp, vp, i]
    L.se2gpu_triangulate.argtypes = [i, vp, vp, vp, i, vp, vp, vp, i]
    L.se2gpu_triangulate_device.argtypes = [i] + [vp] * 7
    L.se2gpu_track_triangulate.argtypes = [vp, i, vp, i, vp, vp, vp, vp, vp, f, f, i, vp, vp, vp, i]
    L.se2gpu_track_triangulate_device.argtypes = [vp, i, vp, vp, vp, vp, vp, vp, vp, f, f, i, vp, vp, vp, vp]
    L.se2gpu_xyz_info.argtypes = [i, vp, vp, vp, vp, i, f, vp, vp, i]
    L.se2gpu_xyz_info_device.argtypes = [i, vp, vp, vp, vp, f, vp, vp, vp]
    L.se2gpu_projection_observations.argtypes = [vp, i] + [vp] * 8 + [i, vp, i, vp, f, f, f, vp, vp, vp, i]
    L.se2gpu_projection_observations_device.argtypes = [vp, i] + [vp] * 11 + [f, f, f, vp, vp, vp, vp]
    L.se2gpu_debug_svd4.argtypes = [i, vp, vp, vp, i]
    L.se2gpu_remove_outliers.argtypes = [i, vp, vp, i, vp, vp, i, vp, vp, vp, vp, i]
    L.se2gpu_remove_outliers_device.argtypes = [i, vp, vp, i, vp, vp, i, vp, vp, vp, vp, vp]
    L.se2gpu_fundam_niters_table.restype = None
    L.se2gpu_fundam_niters_table.argtypes = [vp]
    L.se2gpu_fundam_debug_niters.argtypes = [i, vp, vp, vp, vp, i]
    L.se2gpu_pose_ba.argtypes = [i] + [vp] * 10 + [i]
    L.se2gpu_pose_ba_device.argtypes = [i] + [vp] * 11
    L.se2gpu_pose_ba_debug_trace.argtypes = [i] + [vp] * 11 + [i]
    L.se2gpu_localizer_create.restype = vp
    L.se2gpu_localizer_create.argtypes = [i, i]
    L.se2gpu_localizer_destroy.argtypes = [vp]
    L.se2gpu_localizer_ba_device.argtypes = [vp, vp, i, vp, vp, i, vp, vp, vp, i, vp, vp, i, vp, vp, vp, vp, vp, vp]
    L.se2gpu_feat_edge.argtypes = [i, i] + [vp] * 17 + [i]
    L.se2gpu_feat_edge_device.argtypes = [i, i] + [vp] * 19
    L.se2gpu_feat_edge_debug_trace.argtypes = [i, i] + [vp] * 18 + [i]
    L.se2gpu_global_ba_create.restype = vp
    L.se2gpu_global_ba_create.argtypes = [i]
    L.se2gpu_global_ba_destroy.argtypes = [vp]
    L.se2gpu_global_ba.argtypes = [vp, i, vp, vp, i] + [vp] * 10
    L.se2gpu_global_ba_device.argtypes = [vp, i, vp, vp, i] + [vp] * 12
    L.se2gpu_global_ba_update_points.argtypes = [i, vp, vp, i, vp, vp, i]
    L.se2gpu_global_ba_update_points_device.argtypes = [i] + [vp] * 5
    L.se2gpu_global_ba_profile.argtypes = [vp, i]
    L.se2gpu_global_ba_profile_read.argtypes = [vp, vp]
    L.se2gpu_se3_ba_create.restype = vp
    L.se2gpu_se3_ba_create.argtypes = [i]
    L.se2gpu_se3_ba_destroy.argtypes = [vp]
    L.se2gpu_se3_ba.argtypes = [vp, i, vp, vp, vp, i, vp, vp, vp, vp, i, vp, i] + [vp] * 14
    L.se2gpu_se3_ba_device.argtypes = [vp, i, vp, vp, vp, i, vp, vp, vp, vp, i, vp, i] + [vp] * 15
    L.se2gpu_se3_ba_debug_trace.argtypes = [vp, i, vp, vp, vp, i, vp, vp, vp, vp, i, vp, i] + [vp] * 13
    L.se2gpu_mp_add_observations.argtypes = [vp] * 6 + [i]
    L.se2gpu_mp_erase_observations.argtypes = [vp] * 6 + [i]
    L.se2gpu_mp_update_measure.argtypes = [vp, vp, i, vp, i]
    L.se2gpu_mp_add_observations_device.argtypes = [vp] * 8
    L.se2gpu_mp_erase_observations_device.argtypes = [vp] * 8
    L.se2gpu_mp_update_measure_device.argtypes = [vp, vp, i, vp, vp, vp]
    L.se2gpu_track_triangulate_batch_device.argtypes = [i, vp, i, vp, vp, i, vp, vp, vp, vp, vp, vp, f, f, i, vp, vp, vp, vp]
    L.se2gpu_tracker_create.restype = vp
    L.se2gpu_tracker_create.argtypes = [i, i, i, vp, i]
    L.se2gpu_tracker_destroy.argtypes = [vp]
    L.se2gpu_tracker_step.argtypes = [vp, i, vp, i, i, i, i, sz, vp, vp, vp]
    L.se2gpu_tracker_first.argtypes = [vp, i, vp, i, i, i, i, sz, vp, vp]
    L.se2gpu_tracker_reset.argtypes = [vp, i, vp, vp]
    L.se2gpu_tracker_state.argtypes = [vp, i, vp]
    L.se2gpu_tracker_graph_nodes.argtypes = [vp, vp, vp]
    L.se2gpu_tracker_debug_eager.argtypes = [vp, i]
    L.se2gpu_track_host_pose.argtypes = [vp] * 7
    L.se2gpu_track_host_decide.argtypes = [vp, i, i, i, i, i, vp, vp, i, vp, vp]
    L.se2gpu_loc_create.restype = vp
    L.se2gpu_loc_create.argtypes = [i, i, i, vp, vp, i]
    L.se2gpu_loc_destroy.argtypes = [vp]
    L.se2gpu_loc_step.argtypes = [vp, i, vp, i, i, i, i, sz, vp, vp]
    L.se2gpu_loc_relocalize.argtypes = [vp, i] + [vp] * 7
    L.se2gpu_loc_state.argtypes = [vp, i, vp]
    L.se2gpu_loc_graph_nodes.argtypes = [vp, vp, vp]
    L.se2gpu_loc_debug_eager.argtypes = [vp, i]
    L.se2gpu_loc_host_pose.argtypes = [vp] * 5
    _lib = L
    return L


def last_error() -> str:
    return lib().se2gpu_last_error().decode()


def check(rc: int, what: str) -> int:
    if rc < 0:
        raise Se2GpuError(f"{what} failed ({rc}): {last_error()}")
    return rc


def ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if hasattr(a, "data_ptr"):  # torch tensor
        return C.c_void_p(a.data_ptr())
    return C.c_void_p(int(a))
