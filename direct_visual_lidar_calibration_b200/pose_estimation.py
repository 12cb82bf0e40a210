"""vlcal::PoseEstimation mirror (reference: include/vlcal/common/estimate_pose.hpp, src/vlcal/common/estimate_pose.cpp):
the initial guess of T_camera_lidar from 2D-3D correspondences that initial_guess_auto computes.

The RANSAC over rotation hypotheses is scored on the GPU (one launch for all hypotheses, csrc/pose_estimation.cu); the
bearings, the hypothesis sampling and the robust Levenberg-Marquardt refinement run on the host inside the library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .camera import GenericCamera, _dp


class PoseEstimationParams:
    """estimate_pose.hpp:10-14.  The reference's PoseEstimation ignores the params it is given (estimate_pose.cpp:16) and
    always runs these defaults; here they take effect."""

    def __init__(self, ransac_iterations: int = 8192, ransac_error_thresh: float = 5.0, robust_kernel_width: float = 10.0):
        self.ransac_iterations = ransac_iterations
        self.ransac_error_thresh = ransac_error_thresh
        self.robust_kernel_width = robust_kernel_width


def _cam_args(proj: GenericCamera):
    return (proj.model_id, _dp(proj.intrinsics), proj.intrinsics.size, _dp(proj.distortion), proj.distortion.size)


def _inputs(kp0, points):
    kp = np.ascontiguousarray(np.asarray(kp0, dtype=np.float64).reshape(-1, 2))
    pts = np.asarray(points, dtype=np.float64)
    if pts.ndim != 2 or pts.shape[1] not in (3, 4):
        raise ValueError("points must be (M,3) or (M,4)")
    pts = np.ascontiguousarray(pts[:, :3])
    if kp.shape[0] != pts.shape[0]:
        raise ValueError(f"{kp.shape[0]} keypoints but {pts.shape[0]} points")
    return kp, pts


class PoseEstimation:
    """PoseEstimation(params).estimate(proj, kp0 (M,2), points (M,3)) -> (T_camera_lidar 4x4, inliers bool (M,)).

    `inliers` marks the correspondences the RANSAC winner's rotation reprojects within ransac_error_thresh.  After a call,
    `stats` holds the solver's counters (hypotheses, degenerate, best_index, best_inliers, lm_iterations, final_cost).
    Raises VlcalError for fewer than 2 correspondences and when no hypothesis has an inlier."""

    def __init__(self, params: PoseEstimationParams | None = None, device: int = -1):
        self.params = params or PoseEstimationParams()
        self.device = device
        self.stats: dict = {}

    def estimate(self, proj: GenericCamera, kp0, points):
        L = _lib.load_library()
        kp, pts = _inputs(kp0, points)
        p = _lib.PoseEstimationParams(int(self.params.ransac_iterations), float(self.params.ransac_error_thresh), float(self.params.robust_kernel_width))
        T = np.empty(16)
        mask = np.zeros(max(kp.shape[0], 1), dtype=np.uint8)
        st = _lib.PoseEstimationStats()
        _lib.check(L.vlcal_estimate_pose_from_correspondences(
            self.device, *_cam_args(proj), _dp(kp), _dp(pts), kp.shape[0], C.byref(p), _dp(T), mask.ctypes.data, C.byref(st)))
        self.stats = {name: getattr(st, name) for name, _ in _lib.PoseEstimationStats._fields_}
        return T.reshape(4, 4).T.copy(), mask[: kp.shape[0]].astype(bool)


def estimate_directions(proj: GenericCamera, pixels) -> np.ndarray:
    """estimate_direction (estimate_fov.cpp:17-34) for each pixel (N,2) -> unit bearings (N,3); host NelderMead<2>."""
    L = _lib.load_library()
    px = np.ascontiguousarray(np.asarray(pixels, dtype=np.float64).reshape(-1, 2))
    out = np.empty((px.shape[0], 3))
    _lib.check(L.vlcal_estimate_directions(*_cam_args(proj), _dp(px), px.shape[0], _dp(out)))
    return out


def sample_pairs(n_correspondences: int, iterations: int) -> np.ndarray:
    """The (iterations, 2) correspondence index pairs the RANSAC draws for M correspondences."""
    out = np.empty((max(iterations, 1), 2), dtype=np.int32)
    _lib.check(_lib.load_library().vlcal_pose_debug_sample_pairs(int(n_correspondences), int(iterations), out.ctypes.data))
    return out[:iterations]


def score_pairs(proj: GenericCamera, kp0, points, pairs, ransac_error_thresh: float, device: int = -1, timing: dict | None = None):
    """The RANSAC scoring launch on given index pairs -> (inlier counts int32 (H,), degenerate bool (H,)).
    With `timing`, timing["kernel_ms"] receives the launch's time between CUDA events."""
    L = _lib.load_library()
    kp, pts = _inputs(kp0, points)
    pr = np.ascontiguousarray(np.asarray(pairs, dtype=np.int32).reshape(-1, 2))
    counts = np.empty(max(pr.shape[0], 1), dtype=np.int32)
    degenerate = np.empty(max(pr.shape[0], 1), dtype=np.uint8)
    ms = C.c_double()
    _lib.check(L.vlcal_pose_debug_score_pairs(
        device, *_cam_args(proj), _dp(kp), _dp(pts), kp.shape[0], pr.ctypes.data, pr.shape[0], float(ransac_error_thresh), counts.ctypes.data, degenerate.ctypes.data,
        C.byref(ms) if timing is not None else None))
    if timing is not None:
        timing["kernel_ms"] = ms.value
    return counts[: pr.shape[0]], degenerate[: pr.shape[0]].astype(bool)


def refine(proj: GenericCamera, kp0, points, init_T_camera_lidar, robust_kernel_width: float = 10.0):
    """The Levenberg-Marquardt refinement alone (host) -> (T_camera_lidar, iterations, final cost)."""
    L = _lib.load_library()
    kp, pts = _inputs(kp0, points)
    T0 = np.ascontiguousarray(np.asarray(init_T_camera_lidar, dtype=np.float64).T.reshape(-1))
    T = np.empty(16)
    it, cost = C.c_int(), C.c_double()
    _lib.check(L.vlcal_pose_debug_refine(*_cam_args(proj), _dp(kp), _dp(pts), kp.shape[0], float(robust_kernel_width), _dp(T0), _dp(T), C.byref(it), C.byref(cost)))
    return T.reshape(4, 4).T.copy(), it.value, cost.value
