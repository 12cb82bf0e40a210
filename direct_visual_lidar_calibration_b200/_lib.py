"""ctypes loader for libvlcal_nid.so (the C ABI declared in include/vlcal_nid.h). Fails loudly; no fallback."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_PKG = os.path.dirname(os.path.abspath(__file__))
# VLCAL_LIB: an alternative build of the same library (A/B measurements of compile-time kernel shapes, `make -C csrc alt`)
_LIB_PATH = os.environ.get("VLCAL_LIB") or os.path.join(_PKG, "libvlcal_nid.so")
_CSRC = os.path.join(_PKG, "csrc")

OK = 0
ERR_INVALID_ARGUMENT = -1
ERR_UNKNOWN_CAMERA_MODEL = -2
ERR_INTRINSIC_COUNT = -3
ERR_CUDA = -4
ERR_NO_DEVICE = -5
ERR_UNSUPPORTED = -6
ERR_BUSY = -7

MODE_HISTOGRAM = 0
MODE_BSPLINE = 1


class VlcalError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"vlcal error {code}: {message}")
        self.code = code
        self.message = message


def library_path() -> str:
    return _LIB_PATH


def build_library(force: bool = False, jobs: int = 4) -> str:
    """Compile libvlcal_nid.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
    if force:
        subprocess.run(["make", "-C", _CSRC, "clean"], check=True, stdout=subprocess.DEVNULL)
    subprocess.run(["make", "-C", _CSRC, f"-j{jobs}", "-s"], check=True)
    return _LIB_PATH


class NMParams(C.Structure):
    _fields_ = [
        ("init_step", C.c_double), ("alpha", C.c_double), ("gamma", C.c_double), ("rho", C.c_double), ("sigma", C.c_double),
        ("max_iterations", C.c_int), ("convergence_var_thresh", C.c_double),
    ]


class NMResult(C.Structure):
    _fields_ = [
        ("converged", C.c_int), ("num_iterations", C.c_int), ("x", C.c_double * 8), ("y", C.c_double),
        ("num_evaluations", C.c_int), ("num_batches", C.c_int), ("num_evaluations_computed", C.c_int),
    ]


class CalibParams(C.Structure):
    _fields_ = [
        ("max_outer_iterations", C.c_int), ("max_inner_iterations", C.c_int),
        ("delta_trans_thresh", C.c_double), ("delta_rot_thresh", C.c_double),
        ("disable_z_buffer_culling", C.c_int), ("nid_bins", C.c_int),
        ("nelder_mead_init_step", C.c_double), ("nelder_mead_convergence_criteria", C.c_double),
    ]


class Bag(C.Structure):
    _fields_ = [
        ("image", C.c_void_p), ("width", C.c_int), ("height", C.c_int), ("row_stride_bytes", C.c_int),
        ("points_xyzw", C.c_void_p), ("intensities", C.c_void_p), ("n_points", C.c_int64),
    ]


class CalibStats(C.Structure):
    _fields_ = [
        ("outer_iterations", C.c_int), ("total_evaluations", C.c_int), ("total_evaluations_computed", C.c_int), ("total_batches", C.c_int),
        ("inner_iterations", C.c_int * 16), ("inner_final_cost", C.c_double * 16), ("culled_points", C.c_int64 * 16),
        ("kernel_launches", C.c_int64), ("kernel_ms_total", C.c_double),
        ("upload_ms", C.c_double), ("cull_ms", C.c_double), ("solve_ms", C.c_double),
    ]


class BfgsParams(C.Structure):
    _fields_ = [
        ("max_num_iterations", C.c_int), ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double),
        ("sufficient_decrease", C.c_double), ("sufficient_curvature_decrease", C.c_double), ("max_step_expansion", C.c_double), ("max_line_search_steps", C.c_int),
        ("max_translation_from_init", C.c_double), ("max_rotation_from_init", C.c_double),
    ]


class BfgsResult(C.Structure):
    _fields_ = [
        ("iterations", C.c_int), ("evaluations", C.c_int), ("termination", C.c_int), ("line_search_restarts", C.c_int),
        ("initial_cost", C.c_double), ("final_cost", C.c_double), ("gradient_max_norm", C.c_double),
    ]


class PoseEstimationParams(C.Structure):
    _fields_ = [("ransac_iterations", C.c_int), ("ransac_error_thresh", C.c_double), ("robust_kernel_width", C.c_double)]


class PoseEstimationStats(C.Structure):
    _fields_ = [
        ("hypotheses", C.c_int), ("degenerate", C.c_int), ("best_index", C.c_int), ("best_inliers", C.c_int),
        ("lm_iterations", C.c_int), ("final_cost", C.c_double),
    ]


class ScanDesc(C.Structure):
    """vlcal_scan_desc: one PointCloud2 scan inside the concatenated data of a bag."""
    _fields_ = [
        ("byte_offset", C.c_int64), ("n_points", C.c_int64), ("point_step", C.c_int32), ("x_offset", C.c_int32), ("y_offset", C.c_int32),
        ("z_offset", C.c_int32), ("xyz_type", C.c_int32), ("intensity_offset", C.c_int32), ("intensity_type", C.c_int32), ("reserved", C.c_int32),
    ]


class Frame(C.Structure):
    """vlcal_frame: one compressed container frame (zstd or LZ4 frame format) and where its output goes."""
    _fields_ = [
        ("src_offset", C.c_int64), ("src_size", C.c_int64), ("dst_offset", C.c_int64), ("dst_size", C.c_int64), ("codec", C.c_int32),
        ("has_crc32", C.c_int32), ("crc32", C.c_uint32), ("reserved", C.c_int32),
    ]


class SearchSet(C.Structure):
    """vlcal_search_set: pose i = (ib * n_left + il) * n_offset + io is [R | R (center[ib] + offset[io])], R = left[il] base[ib]."""
    _fields_ = [
        ("left", C.POINTER(C.c_double)), ("base", C.POINTER(C.c_double)), ("center", C.POINTER(C.c_double)), ("offset", C.POINTER(C.c_double)),
        ("indices", C.POINTER(C.c_int32)), ("n_left", C.c_int32), ("n_base", C.c_int32), ("n_offset", C.c_int32), ("n_poses", C.c_int64),
    ]


SE3_OBJECTIVE = C.CFUNCTYPE(C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p)
NM_BATCH_FN = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.c_int, C.c_int, C.POINTER(C.c_double), C.c_void_p)
NM_OBSERVE_FN = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.c_int, C.c_double, C.c_void_p)
POSE_CALLBACK = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.c_double, C.c_void_p)
ALLREDUCE_FN = C.CFUNCTYPE(None, C.POINTER(C.c_double), C.c_int, C.c_void_p)

_lib = None


def load_library():
    """Load the product library; raises if it has not been built (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise VlcalError(ERR_CUDA, f"{_LIB_PATH} is missing: build it with __graft_entry__.build() or `make -C {_CSRC}`; there is no CPU fallback")
    L = C.CDLL(_LIB_PATH)
    dp, vp, ip = C.POINTER(C.c_double), C.c_void_p, C.POINTER(C.c_int)
    L.vlcal_nid_version.restype = C.c_char_p
    L.vlcal_nid_last_error.restype = C.c_char_p
    L.vlcal_nid_device_count.restype = C.c_int
    L.vlcal_camera_model_id.argtypes = [C.c_char_p]
    L.vlcal_camera_num_params.argtypes = [C.c_int, ip, ip]
    L.vlcal_camera_project.argtypes = [C.c_int, dp, C.c_int, dp, C.c_int, dp, dp]
    L.vlcal_se3_expmap_gtsam.argtypes = [dp, dp]
    L.vlcal_estimate_camera_fov.argtypes = [C.c_int, dp, C.c_int, dp, C.c_int, C.c_int, C.c_int, dp]
    L.vlcal_outer_step_delta.argtypes = [dp, dp, dp, dp]
    L.vlcal_nid_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, dp, C.c_int, dp, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int64, C.c_int, C.c_double]
    L.vlcal_nid_destroy.argtypes = [vp]
    L.vlcal_nid_destroy.restype = None
    L.vlcal_nid_evaluate.argtypes = [vp, dp, C.c_int, dp, vp]
    L.vlcal_nid_evaluate_async.argtypes = [vp, dp, C.c_int]
    L.vlcal_nid_wait.argtypes = [vp, dp, vp]
    L.vlcal_nid_score_poses.argtypes = [C.POINTER(vp), C.c_int, dp, C.c_int, dp]
    L.vlcal_nid_sweep_poses.argtypes = [C.POINTER(vp), C.c_int, dp, C.c_int64, dp, vp]
    L.vlcal_nid_debug_sweep_kernel.argtypes = [C.POINTER(vp), C.c_int, dp, C.c_int64, dp, vp]
    L.vlcal_nid_sweep_search_set.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(SearchSet), dp]
    L.vlcal_nid_sweep_search_set_inliers.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(SearchSet), dp, C.POINTER(C.c_int64)]
    L.vlcal_search_set_poses.argtypes = [C.c_int, C.POINTER(SearchSet), dp]
    L.vlcal_nid_sweep_max_points.restype = C.c_int64
    L.vlcal_nid_sweep_launch_shape.argtypes = [vp, ip, ip]
    L.vlcal_nid_sweep_last_kernel_ms.restype = C.c_double
    L.vlcal_nid_debug_sweep_last_deferred.restype = C.c_int64
    L.vlcal_nid_set_poses_per_pass.argtypes = [vp, C.c_int]
    L.vlcal_nid_get_profile_passes.argtypes = [vp, C.POINTER(C.c_int64)]
    L.vlcal_nid_get_profile_delta.argtypes = [vp, C.POINTER(C.c_int64)]
    L.vlcal_nid_debug_solve_stamps.argtypes = [vp, C.c_int, C.POINTER(C.c_uint64), ip]
    L.vlcal_nid_debug_block_times.argtypes = [vp, C.c_int, C.POINTER(C.c_uint64), ip]
    L.vlcal_nid_evaluate_bspline.argtypes = [vp, dp, C.c_int, dp, vp, vp]
    L.vlcal_nid_evaluate_bspline_grad.argtypes = [vp, dp, C.c_int, dp, dp, vp]
    L.vlcal_nid_num_points.argtypes = [vp]
    L.vlcal_nid_num_points.restype = C.c_int64
    L.vlcal_nid_bins.argtypes = [vp]
    L.vlcal_nid_max_fov.argtypes = [vp]
    L.vlcal_nid_max_fov.restype = C.c_double
    L.vlcal_nid_points_are_f32.argtypes = [vp]
    L.vlcal_nid_max_poses_per_launch.restype = C.c_int
    L.vlcal_nid_set_profiling.argtypes = [vp, C.c_int]
    L.vlcal_nid_get_profile.argtypes = [vp, C.POINTER(C.c_int64), dp, C.POINTER(C.c_int64)]
    L.vlcal_nid_reset_profile.argtypes = [vp]
    L.vlcal_nid_set_kernel_variant.argtypes = [vp, C.c_int]
    L.vlcal_nid_debug_timeline.argtypes = [vp, dp, C.c_int, dp]
    L.vlcal_nid_reorder_for_pose.argtypes = [vp, dp]
    L.vlcal_nid_filter_enabled.argtypes = [vp]
    L.vlcal_nid_debug_filter_check.argtypes = [vp, dp, C.c_int, C.POINTER(C.c_uint64), dp]
    L.vlcal_nid_debug_filter_check_delta.argtypes = [vp, dp, C.c_int, C.POINTER(C.c_uint64), dp]
    L.vlcal_nid_p2p_create.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(vp), vp]
    L.vlcal_nid_p2p_connect.argtypes = [vp, vp]
    L.vlcal_nid_p2p_attach.argtypes = [vp, vp]
    L.vlcal_nid_p2p_destroy.argtypes = [vp]
    L.vlcal_nid_p2p_destroy.restype = None
    L.vlcal_nid_p2p_set_default.argtypes = [vp]
    L.vlcal_nid_set_solver_mode.argtypes = [C.c_int]
    L.vlcal_nid_debug_record_solve_trace.argtypes = [C.c_int]
    L.vlcal_nid_debug_last_solve_trace.argtypes = [C.c_int, dp, ip]
    L.vlcal_nid_debug_last_points_per_lane.argtypes = [vp, ip]
    L.vlcal_view_cull.argtypes = [C.c_int, C.c_int, dp, C.c_int, dp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, vp, C.c_int64, dp, vp, C.POINTER(C.c_int64)]
    L.vlcal_debug_view_cull_points.argtypes = [C.c_int, C.c_int, dp, C.c_int, dp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, vp, vp, C.c_int64, dp, vp,
                                               C.POINTER(C.c_int64), ip]
    L.vlcal_generate_lidar_image.argtypes = [C.c_int, C.c_int, dp, C.c_int, dp, C.c_int, C.c_int, C.c_int, dp, vp, vp, C.c_int64, vp, vp]
    viewer = [C.c_int, C.c_int, dp, C.c_int, dp, C.c_int, C.c_int, C.c_int, vp, C.c_int, dp, vp, vp, C.c_int64]
    L.vlcal_turbo_colormap.argtypes = [vp]
    L.vlcal_colorize_points.argtypes = viewer + [C.c_float, vp, dp]
    L.vlcal_render_overlay.argtypes = viewer + [C.c_int, C.c_float, vp, vp, dp]
    L.vlcal_agreement_map.argtypes = viewer + [C.c_int, C.c_int, C.c_float, dp, vp, vp, vp]
    L.vlcal_nm_default_params.argtypes = [C.POINTER(NMParams)]
    L.vlcal_nm_default_params.restype = None
    L.vlcal_nelder_mead_batched.argtypes = [C.c_int, NM_BATCH_FN, NM_OBSERVE_FN, vp, dp, C.POINTER(NMParams), C.POINTER(NMResult)]
    L.vlcal_calib_default_params.argtypes = [C.POINTER(CalibParams)]
    L.vlcal_calib_default_params.restype = None
    L.vlcal_estimate_pose_nelder_mead_ctx.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(CalibParams), dp, POSE_CALLBACK, ALLREDUCE_FN, vp, dp, C.POINTER(NMResult)]
    L.vlcal_estimate_poses_nelder_mead_ctx.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(CalibParams), C.c_int, dp, vp, dp, C.POINTER(NMResult)]
    common = [C.c_int, C.c_int, dp, C.c_int, dp, C.c_int, C.POINTER(Bag), C.c_int, C.POINTER(CalibParams), dp, POSE_CALLBACK, ALLREDUCE_FN, vp, C.c_int, dp]
    L.vlcal_estimate_pose_nelder_mead.argtypes = common + [C.POINTER(NMResult), C.POINTER(CalibStats)]
    L.vlcal_calibrate_nelder_mead.argtypes = common + [C.POINTER(CalibStats)]
    L.vlcal_bfgs_default_params.argtypes = [C.POINTER(BfgsParams)]
    L.vlcal_bfgs_default_params.restype = None
    L.vlcal_bfgs_minimize_se3.argtypes = [SE3_OBJECTIVE, vp, C.POINTER(BfgsParams), dp, POSE_CALLBACK, vp, dp, C.POINTER(BfgsResult)]
    L.vlcal_estimate_pose_bfgs_ctx.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(BfgsParams), dp, POSE_CALLBACK, ALLREDUCE_FN, vp, dp, C.POINTER(BfgsResult)]
    L.vlcal_pose_estimation_default_params.argtypes = [C.POINTER(PoseEstimationParams)]
    L.vlcal_pose_estimation_default_params.restype = None
    cam = [C.c_int, dp, C.c_int, dp, C.c_int]
    L.vlcal_estimate_pose_from_correspondences.argtypes = [C.c_int] + cam + [dp, dp, C.c_int64, C.POINTER(PoseEstimationParams), dp, vp, C.POINTER(PoseEstimationStats)]
    L.vlcal_estimate_directions.argtypes = cam + [dp, C.c_int64, dp]
    L.vlcal_pose_debug_score_pairs.argtypes = [C.c_int] + cam + [dp, dp, C.c_int64, vp, C.c_int, C.c_double, vp, vp, dp]
    L.vlcal_pose_debug_sample_pairs.argtypes = [C.c_int64, C.c_int, vp]
    L.vlcal_pose_debug_refine.argtypes = cam + [dp, dp, C.c_int64, C.c_double, dp, dp, ip, dp]
    i64p = C.POINTER(C.c_int64)
    L.vlcal_approximate_voxel_grid.argtypes = [C.c_int, vp, C.c_int64, C.c_double, vp, i64p, i64p, dp]
    L.vlcal_equalize_intensities.argtypes = [C.c_int, vp, C.c_int64, vp, dp]
    L.vlcal_lidar_fov_candidates.argtypes = [C.c_int, vp, C.c_int64, vp, i64p, ip, dp]
    L.vlcal_min_bearing_cosine.argtypes = [C.c_int, vp, C.c_int64, dp]
    L.vlcal_bag_integrate.argtypes = [C.c_int, vp, C.c_int64, C.POINTER(ScanDesc), C.c_int64, C.c_double, C.c_double, vp, i64p, i64p, dp]
    L.vlcal_decode_frames.argtypes = [C.c_int, vp, C.c_int64, C.POINTER(Frame), C.c_int, vp, C.c_int64, C.POINTER(C.c_int32), dp]
    _lib = L
    return L


def check(rc: int):
    if rc != OK:
        msg = load_library().vlcal_nid_last_error().decode(errors="replace")
        raise VlcalError(rc, msg)


def set_solver_mode(mode: int):
    """0 auto (persistent kernel where possible), 1 host loop, 3 persistent kernel (see include/vlcal_nid.h); any other mode raises VlcalError."""
    check(load_library().vlcal_nid_set_solver_mode(int(mode)))


def device_count() -> int:
    return int(load_library().vlcal_nid_device_count())
