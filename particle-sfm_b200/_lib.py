"""ctypes binding of libpsfm_b200.so (the C ABI of include/psfm_b200.h).

The library is the product: there is no Python/NumPy fallback.  Loading fails loudly if
the shared object has not been built (python -m particlesfm_b200.build)."""
import ctypes as C
import os

from . import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
# PSFM_LIB: alternative build of the same library (kernel-tuning experiments only)
LIB_PATH = os.environ.get("PSFM_LIB") or os.path.join(_HERE, "libpsfm_b200.so")
_LIB = None

EXPORTS = [
    "psfm_last_error", "psfm_abi_version", "psfm_device_count", "psfm_set_device", "psfm_launch_count",
    "psfm_traj_default_options", "psfm_traj_optimize", "psfm_traj_optimize_device",
    "psfm_ba_default_options", "psfm_ba_global_options", "psfm_ba_solve", "psfm_ba_create",
    "psfm_ba_set_state", "psfm_ba_run", "psfm_ba_get_state", "psfm_ba_destroy", "psfm_ba_evaluate",
    "psfm_ba_linear_step", "psfm_ba_band_solve", "psfm_measure_dfma", "psfm_ba_default_refine_options",
    "psfm_ba_filter_negative_depth", "psfm_ba_filter_points", "psfm_ba_normalize", "psfm_ba_num_observations",
    "psfm_ba_get_observation_mask", "psfm_ba_get_point_errors", "psfm_ba_iterative_refinement",
    "psfm_ba_create_from_triangulation", "psfm_ba_get_model", "psfm_ba_get_observations",
    "psfm_grid_sample", "psfm_flow_check", "psfm_tracker_step", "psfm_tracker_buffer_inputs",
    "psfm_tracker_create", "psfm_tracker_advance", "psfm_tracker_optimize", "psfm_tracker_get_buffer", "psfm_tracker_set_buffer",
    "psfm_flow_check_device", "psfm_tracker_finish", "psfm_tracker_result", "psfm_tracker_destroy",
    "psfm_tracker_create_mode", "psfm_tracker_track_npy", "psfm_track_npy_create", "psfm_track_npy_data",
    "psfm_track_npy_destroy",
    "psfm_matches_create", "psfm_matches_result", "psfm_matches_destroy", "psfm_tracker_matches",
    "psfm_matches_table", "psfm_match_table_result", "psfm_match_table_verify", "psfm_match_table_destroy",
    "psfm_known_rotation_translations", "psfm_triangulate_tracks",
    "psfm_two_view_relative_poses", "psfm_rotation_default_options", "psfm_estimate_global_rotations",
    "psfm_optimize_pairwise_translations", "psfm_lud_default_options", "psfm_estimate_global_positions",
    "psfm_triangulator_default_options", "psfm_triangulation_create", "psfm_triangulation_result",
    "psfm_triangulation_destroy", "psfm_verification_default_options", "psfm_verify_two_view_geometries",
    "psfm_blocked_cholesky_solve", "psfm_laplacian_solve", "psfm_spd_inverse",
    "psfm_null_vectors", "psfm_verification_local_model", "psfm_verification_minimal", "psfm_verification_cubic",
    "psfm_convert_create", "psfm_convert_result", "psfm_convert_destroy",
    "psfm_colors_create", "psfm_colors_add_images", "psfm_colors_result", "psfm_colors_destroy",
    "psfm_corr_pyramids", "psfm_corr_pyramid_floats", "psfm_corr_lookup", "psfm_flow_upsample", "psfm_flow_to_image",
    "psfm_depth_prepare", "psfm_depth_upsample", "psfm_depth_quantize",
    "psfm_seg_max_window", "psfm_seg_hits", "psfm_seg_shuffle", "psfm_seg_windows", "psfm_seg_depth_resize",
    "psfm_seg_encode", "psfm_seg_merge", "psfm_seg_draw",
    "psfm_dist_get_unique_id", "psfm_dist_init", "psfm_dist_world_size",
    "psfm_dist_rank", "psfm_dist_finalize",
]


class PsfmError(RuntimeError):
    """code: the library's negative status (_abi.PSFM_ERR_*) when a call returned one, else None."""

    def __init__(self, message, code=None):
        super().__init__(message)
        self.code = code


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise PsfmError("libpsfm_b200.so is not built — run `python -m particlesfm_b200.build` "
                        "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    dp, fp, ip = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int32)
    L.psfm_last_error.restype = C.c_char_p
    L.psfm_launch_count.restype = C.c_int64
    L.psfm_traj_default_options.argtypes = [C.POINTER(_abi.TrajOptions)]
    L.psfm_traj_default_options.restype = None
    L.psfm_traj_optimize.argtypes = [dp, dp, dp, dp, fp, C.c_int32, C.c_int32, C.c_int32,
                                     C.POINTER(_abi.TrajOptions), dp, C.POINTER(_abi.TrajSummary)]
    L.psfm_traj_optimize_device.argtypes = [C.c_void_p] * 5 + [C.c_int32, C.c_int32, C.c_int32,
                                                               C.POINTER(_abi.TrajOptions), C.c_void_p,
                                                               C.POINTER(_abi.TrajSummary), C.c_void_p]
    L.psfm_ba_default_options.argtypes = [C.POINTER(_abi.BAOptions)]
    L.psfm_ba_default_options.restype = None
    L.psfm_ba_global_options.argtypes = [C.POINTER(_abi.BAOptions)]
    L.psfm_ba_global_options.restype = None
    L.psfm_ba_solve.argtypes = [C.POINTER(_abi.BAProblemStruct), C.POINTER(_abi.BAOptions),
                                C.POINTER(_abi.BASummary)]
    L.psfm_ba_create.argtypes = [C.POINTER(_abi.BAProblemStruct), C.POINTER(C.c_void_p)]
    L.psfm_ba_set_state.argtypes = [C.c_void_p, dp, dp, dp, dp]
    L.psfm_ba_get_state.argtypes = [C.c_void_p, dp, dp, dp, dp]
    L.psfm_ba_run.argtypes = [C.c_void_p, C.POINTER(_abi.BAOptions), C.POINTER(_abi.BASummary)]
    L.psfm_ba_destroy.argtypes = [C.c_void_p]
    L.psfm_ba_destroy.restype = None
    L.psfm_ba_evaluate.argtypes = [C.c_void_p, C.POINTER(_abi.BAOptions), dp, dp, dp, dp]
    L.psfm_ba_linear_step.argtypes = [C.c_void_p, C.POINTER(_abi.BAOptions), C.c_double, dp, dp, ip]
    L.psfm_measure_dfma.argtypes = [dp, dp]
    u8p = C.POINTER(C.c_uint8)
    L.psfm_grid_sample.argtypes = [fp, C.c_int32, C.c_int32, C.c_int32, dp, C.c_int32, fp]
    L.psfm_flow_check.argtypes = [fp, fp, C.c_int32, C.c_int32, C.c_float, fp, u8p]
    L.psfm_tracker_step.argtypes = [fp, u8p, C.c_int32, C.c_int32, dp, C.c_int32, C.c_int32, dp, u8p, u8p]
    L.psfm_tracker_buffer_inputs.argtypes = [fp, fp, u8p, C.c_int32, C.c_int32, dp, C.c_int32, C.c_double, dp, dp, dp]
    L.psfm_known_rotation_translations.argtypes = [dp, dp, ip, dp, dp, C.c_int32, dp, ip]
    L.psfm_triangulate_tracks.argtypes = [dp, dp, ip, C.c_int32, dp]
    i64p = C.POINTER(C.c_int64)
    L.psfm_two_view_relative_poses.argtypes = [C.c_int32, i64p, fp, ip, dp, C.c_int32, C.c_int64, ip, ip, dp, dp, dp, i64p,
                                               C.POINTER(C.c_uint32), dp, dp, dp, ip, i64p, C.POINTER(C.c_uint8)]
    L.psfm_rotation_default_options.argtypes = [C.POINTER(_abi.RotationOptions)]
    L.psfm_rotation_default_options.restype = None
    L.psfm_estimate_global_rotations.argtypes = [C.c_int32, C.c_int64, ip, dp, ip, C.POINTER(C.c_uint8),
                                                 C.POINTER(_abi.RotationOptions), dp, C.POINTER(C.c_uint8),
                                                 C.POINTER(C.c_uint8), C.POINTER(_abi.RotationSummary)]
    L.psfm_optimize_pairwise_translations.argtypes = [C.c_int32, i64p, fp, ip, dp, C.c_int32, C.c_int64, ip, i64p,
                                                      C.POINTER(C.c_uint32), dp, C.POINTER(C.c_uint8), dp, ip]
    L.psfm_lud_default_options.argtypes = [C.POINTER(_abi.LudOptions)]
    L.psfm_lud_default_options.restype = None
    L.psfm_estimate_global_positions.argtypes = [C.c_int32, C.c_int64, ip, dp, dp, C.POINTER(C.c_uint8),
                                                 C.POINTER(C.c_uint8), C.POINTER(_abi.LudOptions), dp,
                                                 C.POINTER(C.c_uint8), dp, dp, C.POINTER(_abi.PositionSummary)]
    vp = C.c_void_p
    L.psfm_triangulator_default_options.argtypes = [C.POINTER(_abi.TriangulatorOptions)]
    L.psfm_triangulator_default_options.restype = None
    L.psfm_triangulation_create.argtypes = [C.c_int32, i64p, fp, ip, dp, C.c_int32, ip, C.c_int64, ip, i64p,
                                            C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), dp, dp, C.POINTER(C.c_uint8),
                                            C.POINTER(_abi.TriangulatorOptions), C.POINTER(vp), i64p, i64p]
    L.psfm_triangulation_result.argtypes = [vp, dp, i64p, ip, ip, i64p, C.POINTER(_abi.TriangulationSummary)]
    L.psfm_triangulation_destroy.argtypes = [vp]
    L.psfm_triangulation_destroy.restype = None
    L.psfm_verification_default_options.argtypes = [C.POINTER(_abi.VerificationOptions)]
    L.psfm_verification_default_options.restype = None
    u32p = C.POINTER(C.c_uint32)
    L.psfm_verify_two_view_geometries.argtypes = [C.c_int32, i64p, fp, ip, C.c_int32, ip, C.POINTER(C.c_uint8), C.c_int64,
                                                  ip, i64p, u32p, C.POINTER(_abi.VerificationOptions), ip, dp, dp, dp,
                                                  i64p, u32p, ip, C.POINTER(_abi.VerificationSummary)]
    L.psfm_tracker_create.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.POINTER(vp)]
    L.psfm_tracker_advance.argtypes = [vp] * 6 + [ip]
    L.psfm_tracker_optimize.argtypes = [vp, C.POINTER(_abi.TrajOptions), C.POINTER(_abi.TrajSummary)]
    L.psfm_tracker_get_buffer.argtypes = [vp, dp, dp, dp, dp]
    L.psfm_tracker_set_buffer.argtypes = [vp, dp]
    L.psfm_flow_check_device.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_float, vp, vp, vp]
    L.psfm_tracker_finish.argtypes = [vp, C.c_int32, i64p, i64p]
    L.psfm_tracker_result.argtypes = [vp, i64p, i64p, ip, dp]
    L.psfm_tracker_destroy.argtypes = [vp]
    L.psfm_tracker_destroy.restype = None
    L.psfm_tracker_create_mode.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp, C.POINTER(vp)]
    L.psfm_tracker_track_npy.argtypes = [vp, C.POINTER(vp), i64p]
    L.psfm_track_npy_create.argtypes = [i64p, i64p, ip, dp, C.c_int64, C.c_int64, C.POINTER(vp), i64p]
    L.psfm_track_npy_data.argtypes = [vp]
    L.psfm_track_npy_data.restype = vp
    L.psfm_track_npy_destroy.argtypes = [vp]
    L.psfm_track_npy_destroy.restype = None
    L.psfm_matches_create.argtypes = [i64p, C.c_int64, i64p, dp, C.c_int32, C.c_int32, C.POINTER(vp), i64p, i64p]
    L.psfm_matches_result.argtypes = [vp, i64p, dp, i64p, i64p, i64p]
    L.psfm_matches_destroy.argtypes = [vp]
    L.psfm_tracker_matches.argtypes = [vp, C.c_int32, C.c_int32, C.POINTER(vp), i64p, i64p]
    L.psfm_matches_destroy.restype = None
    L.psfm_matches_table.argtypes = [vp, ip, C.POINTER(vp), i64p, i64p, i64p]
    L.psfm_match_table_result.argtypes = [vp, i64p, fp, ip, i64p, u32p]
    L.psfm_match_table_verify.argtypes = [vp, ip, C.c_int32, ip, C.POINTER(C.c_uint8), C.POINTER(_abi.VerificationOptions),
                                          ip, dp, dp, dp, i64p, u32p, ip, C.POINTER(_abi.VerificationSummary)]
    L.psfm_match_table_destroy.argtypes = [vp]
    L.psfm_match_table_destroy.restype = None
    L.psfm_ba_default_refine_options.argtypes = [C.POINTER(_abi.BARefineOptions)]
    L.psfm_ba_default_refine_options.restype = None
    L.psfm_ba_filter_negative_depth.argtypes = [C.c_void_p, i64p]
    L.psfm_ba_filter_points.argtypes = [C.c_void_p, C.c_double, C.c_double, i64p]
    L.psfm_ba_normalize.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double, dp, dp]
    L.psfm_ba_num_observations.argtypes = [C.c_void_p, i64p]
    L.psfm_ba_get_observation_mask.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
    L.psfm_ba_get_point_errors.argtypes = [C.c_void_p, dp]
    L.psfm_ba_iterative_refinement.argtypes = [C.c_void_p, C.POINTER(_abi.BAOptions), C.POINTER(_abi.BARefineOptions),
                                               C.POINTER(_abi.BARefineReport)]
    L.psfm_ba_create_from_triangulation.argtypes = [vp, dp, dp, dp, u8p, u8p, u8p, C.POINTER(vp), ip, ip, i64p]
    L.psfm_ba_get_model.argtypes = [vp, dp, dp, dp, dp, i64p, ip, ip, i64p]
    L.psfm_ba_get_observations.argtypes = [vp, ip, ip, dp, ip]
    L.psfm_ba_band_solve.argtypes = [dp, dp, C.c_int32, C.c_int32, dp]
    L.psfm_blocked_cholesky_solve.argtypes = [dp, dp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, dp]
    L.psfm_laplacian_solve.argtypes = [dp, dp, C.c_int32, dp]
    L.psfm_spd_inverse.argtypes = [dp, C.c_int32, dp]
    L.psfm_null_vectors.argtypes = [C.c_int32, dp, C.c_int64, dp]
    L.psfm_verification_local_model.argtypes = [C.c_int32, fp, C.c_int64, dp, C.c_double, dp, dp, dp]
    L.psfm_verification_minimal.argtypes = [C.c_int32, fp, C.c_int64, dp, ip]
    L.psfm_verification_cubic.argtypes = [dp, C.c_int64, dp, ip]
    L.psfm_convert_create.argtypes = [C.c_int32, ip, C.c_int32, dp, dp, ip, i64p, dp, ip, C.c_int64, dp, u8p, C.c_int64,
                                      C.POINTER(vp), i64p, ip, C.POINTER(_abi.ConvertSummary)]
    L.psfm_convert_result.argtypes = [vp, C.c_int32, C.c_int32, dp, u8p, C.POINTER(_abi.ConvertSummary)]
    L.psfm_convert_destroy.argtypes = [vp]
    L.psfm_convert_destroy.restype = None
    L.psfm_colors_create.argtypes = [C.c_int32, i64p, dp, ip, C.c_int64, C.POINTER(vp), C.POINTER(_abi.ColorsSummary)]
    L.psfm_colors_add_images.argtypes = [vp, C.c_int32, C.c_int32, ip, ip, u8p]
    L.psfm_colors_result.argtypes = [vp, u8p, C.POINTER(_abi.ColorsSummary)]
    L.psfm_colors_destroy.argtypes = [vp]
    L.psfm_colors_destroy.restype = None
    L.psfm_corr_pyramids.argtypes = [vp, vp, C.c_int32, C.c_int32, vp]
    L.psfm_corr_pyramid_floats.argtypes = [C.c_int32, C.c_int32]
    L.psfm_corr_pyramid_floats.restype = C.c_int64
    L.psfm_corr_lookup.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp]
    L.psfm_flow_upsample.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, ip, vp, vp]
    L.psfm_flow_to_image.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, vp, vp]
    L.psfm_depth_prepare.argtypes = [vp] + [C.c_int32] * 6 + [vp, vp]
    L.psfm_depth_upsample.argtypes = [vp] + [C.c_int32] * 6 + [vp, vp, vp]
    L.psfm_depth_quantize.argtypes = [vp] + [C.c_int32] * 3 + [vp, vp, vp]
    L.psfm_seg_max_window.argtypes = []
    L.psfm_seg_hits.argtypes = [vp, vp, C.c_int32, vp, C.c_int32, C.c_int32, vp, vp]
    L.psfm_seg_shuffle.argtypes = [C.c_int32, vp]
    L.psfm_seg_windows.argtypes = [vp, vp, vp, vp, vp, C.c_int32, vp, C.c_int32, vp, vp, vp]
    L.psfm_seg_depth_resize.argtypes = [vp] + [C.c_int32] * 3 + [vp, vp]
    L.psfm_seg_encode.argtypes = [vp, vp, vp, vp] + [C.c_int32] * 3 + [vp] + [C.c_int32] * 3 + [vp, vp, vp]
    L.psfm_seg_merge.argtypes = [vp, vp, C.c_int32, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp]
    L.psfm_seg_draw.argtypes = [vp, vp, vp, vp] + [C.c_int32] * 4 + [vp, C.c_int32, vp] + [C.c_int32] * 3 + [vp, vp, vp]
    L.psfm_dist_get_unique_id.argtypes = [C.POINTER(C.c_uint8)]
    L.psfm_dist_init.argtypes = [C.POINTER(C.c_uint8), C.c_int32, C.c_int32]
    L.psfm_dist_finalize.restype = None
    _LIB = L
    return L


def check(rc, what):
    if rc < 0:
        msg = lib().psfm_last_error().decode("utf-8", "replace")
        raise PsfmError(f"{what} failed with status {rc}: {msg}", rc)
    return rc


def dptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None
