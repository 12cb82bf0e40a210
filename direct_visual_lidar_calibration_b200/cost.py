"""vlcal::CostCalculatorNID mirror (reference: include/vlcal/calib/cost_calculator_nid.hpp, src/vlcal/calib/cost_calculator_nid.cpp)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .camera import GenericCamera, _dp


def T_to_colmajor(T) -> np.ndarray:
    """(…,4,4) row-major numpy transform(s) -> (…,16) column-major doubles (Eigen::Isometry3d::matrix().data())."""
    T = np.asarray(T, dtype=np.float64)
    return np.ascontiguousarray(np.swapaxes(T.reshape(-1, 4, 4), 1, 2)).reshape(-1, 16)


def colmajor_to_T(v) -> np.ndarray:
    return np.swapaxes(np.asarray(v, dtype=np.float64).reshape(-1, 4, 4), 1, 2).copy()


class VisualLiDARData:
    """vlcal::VisualLiDARData {cv::Mat image (CV_8UC1); FrameCPU::Ptr points} (visual_lidar_data.hpp:10-23).

    points: (N,4) float64 homogeneous (x,y,z,1) = Eigen::Vector4d; (N,3) input gets w=1 appended.
    intensities: (N,) float64 (frame.hpp:66,69)."""

    def __init__(self, image, points, intensities):
        self.image = np.ascontiguousarray(image, dtype=np.uint8)
        if self.image.ndim != 2:
            raise ValueError("image must be a single-channel uint8 array (cv::imread(path, 0))")
        pts = np.asarray(points, dtype=np.float64)
        if pts.ndim != 2 or pts.shape[1] not in (3, 4):
            raise ValueError("points must be (N,3) or (N,4)")
        if pts.shape[1] == 3:
            pts = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1)
        self.points = np.ascontiguousarray(pts)
        self.intensities = np.ascontiguousarray(np.asarray(intensities, dtype=np.float64).reshape(-1))
        if self.intensities.shape[0] != self.points.shape[0]:
            raise ValueError("intensities / points size mismatch")

    def size(self) -> int:
        return int(self.points.shape[0])


class NIDCostParams:
    """vlcal::NIDCostParams (cost_calculator_nid.cpp:7-9)."""

    def __init__(self, bins: int = 16):
        self.bins = bins


class CostCalculatorNID:
    """vlcal::CostCalculatorNID(proj, data, params) with calculate(T_camera_lidar) (cost_calculator_nid.cpp:13-67),
    plus calculate_batch(Ts) which scores many poses in one pass over the cloud."""

    def __init__(self, proj: GenericCamera, data: VisualLiDARData, params: NIDCostParams | None = None, device: int = -1, max_fov: float | None = None):
        params = params or NIDCostParams()
        L = _lib.load_library()
        self._L = L
        self._ctx = C.c_void_p()
        self.params = params
        self.proj = proj
        self.data = data
        h, w = data.image.shape
        _lib.check(
            L.vlcal_nid_create(
                C.byref(self._ctx), device, _lib.MODE_HISTOGRAM, proj.model_id, _dp(proj.intrinsics), proj.intrinsics.size, _dp(proj.distortion), proj.distortion.size,
                data.image.ctypes.data, w, h, data.image.strides[0], data.points.ctypes.data, data.intensities.ctypes.data, data.size(), params.bins,
                -1.0 if max_fov is None else float(max_fov),
            )
        )

    # --- reference surface ---------------------------------------------------------------
    def calculate(self, T_camera_lidar) -> float:
        return float(self.calculate_batch(np.asarray(T_camera_lidar, dtype=np.float64).reshape(1, 4, 4))[0])

    # --- batched surface ------------------------------------------------------------------
    def calculate_batch(self, Ts, return_hist: bool = False):
        Tc = T_to_colmajor(Ts)
        P = Tc.shape[0]
        out = np.empty(P)
        bins = self.params.bins
        hist = np.empty((P, bins * bins), dtype=np.int32) if return_hist else None
        _lib.check(self._L.vlcal_nid_evaluate(self._ctx, _dp(Tc), P, _dp(out), hist.ctypes.data if return_hist else None))
        if return_hist:
            # storage index = image_bin + lidar_bin*bins -> [P, lidar_bin, image_bin] -> [P, image_bin, lidar_bin]
            return out, np.swapaxes(hist.reshape(P, bins, bins), 1, 2).copy()
        return out

    @property
    def max_fov(self) -> float:
        return float(self._L.vlcal_nid_max_fov(self._ctx))

    @property
    def points_are_f32(self) -> bool:
        return bool(self._L.vlcal_nid_points_are_f32(self._ctx))

    def reorder_for_pose(self, T_camera_lidar):
        """Group the cloud by projected image tile at this pose (values are unchanged; gathers coalesce)."""
        _lib.check(self._L.vlcal_nid_reorder_for_pose(self._ctx, _dp(T_to_colmajor(T_camera_lidar))))

    def attach_peer_exchange(self, px):
        """Multi-GPU, one bag per rank: evaluations return the sum over ranks (fused in-kernel exchange)."""
        _lib.check(self._L.vlcal_nid_p2p_attach(self._ctx, px.handle if px is not None else None))

    def debug_timeline(self, Ts):
        Tc = T_to_colmajor(Ts)
        out = np.zeros(12)
        _lib.check(self._L.vlcal_nid_debug_timeline(self._ctx, _dp(Tc), Tc.shape[0], _dp(out)))
        keys = ["main_done", "merged", "ticket", "finalize_done", "published", "host_launch_call", "host_total", "fin_zeroed", "fin_marginals", "fin_terms", "p2p_enter", "p2p_arrived"]
        return dict(zip(keys, out[:12]))

    @property
    def filter_enabled(self) -> bool:
        return bool(self._L.vlcal_nid_filter_enabled(self._ctx))

    def debug_filter_check(self, Ts, delta=False):
        """Test hook: (point_poses, deferred_to_exact, mismatches, max |uv32-uv64|/bound).  delta: equirectangular delta
        step -- in every group of 8 poses, the most central pose is the anchor and the others are first-order updates from it."""
        Tc = T_to_colmajor(Ts)
        counts = (C.c_uint64 * 3)()
        ratio = C.c_double()
        fn = self._L.vlcal_nid_debug_filter_check_delta if delta else self._L.vlcal_nid_debug_filter_check
        _lib.check(fn(self._ctx, _dp(Tc), Tc.shape[0], counts, C.byref(ratio)))
        return int(counts[0]), int(counts[1]), int(counts[2]), float(ratio.value)

    @property
    def handle(self):
        return self._ctx

    def set_profiling(self, enable: bool):
        _lib.check(self._L.vlcal_nid_set_profiling(self._ctx, int(enable)))

    def set_kernel_variant(self, variant: int):
        _lib.check(self._L.vlcal_nid_set_kernel_variant(self._ctx, int(variant)))

    def reset_profile(self):
        _lib.check(self._L.vlcal_nid_reset_profile(self._ctx))

    def profile(self):
        launches, poses, ms, passes, delta = C.c_int64(), C.c_int64(), C.c_double(), C.c_int64(), (C.c_int64 * 4)()
        _lib.check(self._L.vlcal_nid_get_profile(self._ctx, C.byref(launches), C.byref(ms), C.byref(poses)))
        _lib.check(self._L.vlcal_nid_get_profile_passes(self._ctx, C.byref(passes)))
        _lib.check(self._L.vlcal_nid_get_profile_delta(self._ctx, delta))
        # persistent kernel: passes (and their poses) that took the equirectangular delta step; point-poses deferred to
        # the exact path in the other passes and in the delta passes
        return {"kernel_launches": launches.value, "kernel_ms_total": ms.value, "poses_total": poses.value, "passes": passes.value,
                "delta_passes": delta[0], "delta_poses": delta[1], "deferred_plain": delta[2], "deferred_delta": delta[3]}

    def set_poses_per_pass(self, k: int):
        """Poses per pass over the cloud in pose-list evaluations (1..8, default 8); measurement hook, results unchanged."""
        _lib.check(self._L.vlcal_nid_set_poses_per_pass(self._ctx, int(k)))

    def arm_solve_stamps(self, capacity: int = 64):
        """The next persistent solve on this cost object records %globaltimer stamps for its first `capacity` batches."""
        _lib.check(self._L.vlcal_nid_debug_solve_stamps(self._ctx, int(capacity), None, None))

    def solve_stamps(self, capacity: int = 64):
        """(n, 8) uint64 nanosecond stamps per batch: block 0 enters, main loop done, merged + arrived, finalizer saw all
        blocks, score published, block 0 saw all scores, next poses ready, unused."""
        buf = (C.c_uint64 * (8 * capacity))()
        n = C.c_int()
        _lib.check(self._L.vlcal_nid_debug_solve_stamps(self._ctx, int(capacity), buf, C.byref(n)))
        return np.ctypeslib.as_array(buf).reshape(capacity, 8)[: n.value].copy()

    def last_points_per_lane(self) -> int:
        """Points per lane (2 or 4) of the kernel instance the last persistent launch on this cost object ran (0: none yet)."""
        k = C.c_int()
        _lib.check(self._L.vlcal_nid_debug_last_points_per_lane(self._ctx, C.byref(k)))
        return int(k.value)

    def block_times(self, capacity: int = 2048):
        """(n_blocks, 4) uint64 ns stamps of one batch of the last stamped persistent solve: enter, zeroed, main loop done, arrived."""
        buf = (C.c_uint64 * (4 * capacity))()
        n = C.c_int()
        _lib.check(self._L.vlcal_nid_debug_block_times(self._ctx, int(capacity), buf, C.byref(n)))
        return np.ctypeslib.as_array(buf).reshape(capacity, 4)[: n.value].copy()

    def close(self):
        if self._ctx:
            self._L.vlcal_nid_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def score_poses(costs, Ts) -> np.ndarray:
    """sum over the cost objects (bags) of calculate(T) for every pose of a list of any length, in ONE persistent launch
    (the objective of visual_camera_calibration.cpp:105-110 over a pose grid)."""
    Tc = T_to_colmajor(Ts)
    P = Tc.shape[0]
    out = np.empty(P)
    handles = (C.c_void_p * len(costs))(*[c.handle for c in costs])
    _lib.check(_lib.load_library().vlcal_nid_score_poses(handles, len(costs), _dp(Tc), P, _dp(out)))
    return out


class NIDCost:
    """vlcal::NIDCost(proj, normalized_image, points, bins) -- value of operator()<double> (nid_cost.hpp:23-107), the
    B-spline soft-histogram NID of the BFGS branch.  `image` is the uint8 image; the reference's CV_64F image is
    image * (1/255.0) (visual_camera_calibration.cpp:203-204), which is what the kernel's bin plane is built from.

    evaluate(T_params) with T_params = (P,7) [qx qy qz qw tx ty tz] (Sophus::SE3d storage) -> (ok[P], nid[P])."""

    def __init__(self, proj: GenericCamera, data: VisualLiDARData, bins: int = 16, device: int = -1):
        L = _lib.load_library()
        self._L = L
        self._ctx = C.c_void_p()
        self.bins = bins
        self.data = data
        h, w = data.image.shape
        _lib.check(
            L.vlcal_nid_create(
                C.byref(self._ctx), device, _lib.MODE_BSPLINE, proj.model_id, _dp(proj.intrinsics), proj.intrinsics.size, _dp(proj.distortion), proj.distortion.size,
                data.image.ctypes.data, w, h, data.image.strides[0], data.points.ctypes.data, data.intensities.ctypes.data, data.size(), bins, 0.0,
            )
        )

    def evaluate(self, T_params, return_hist: bool = False):
        tp = np.ascontiguousarray(np.asarray(T_params, dtype=np.float64)).reshape(-1, 7)
        P = tp.shape[0]
        nid = np.empty(P)
        ok = np.empty(P, dtype=np.int32)
        hist = np.empty((P, self.bins * self.bins)) if return_hist else None
        _lib.check(self._L.vlcal_nid_evaluate_bspline(self._ctx, _dp(tp), P, _dp(nid), ok.ctypes.data, hist.ctypes.data if return_hist else None))
        if return_hist:
            return ok.astype(bool), nid, np.swapaxes(hist.reshape(P, self.bins, self.bins), 1, 2).copy()
        return ok.astype(bool), nid

    @property
    def handle(self):
        return self._ctx

    def evaluate_with_gradient(self, T_params):
        """NIDCost::operator()<ceres::Jet<double, 7>>: (ok[P], nid[P], grad[P, 7]) with grad = d NID / d [qx qy qz qw tx ty tz]."""
        tp = np.ascontiguousarray(np.asarray(T_params, dtype=np.float64)).reshape(-1, 7)
        P = tp.shape[0]
        nid = np.empty(P)
        grad = np.empty((P, 7))
        ok = np.empty(P, dtype=np.int32)
        _lib.check(self._L.vlcal_nid_evaluate_bspline_grad(self._ctx, _dp(tp), P, _dp(nid), _dp(grad), ok.ctypes.data))
        return ok.astype(bool), nid, grad

    def __call__(self, T_params7):
        ok, nid = self.evaluate(np.asarray(T_params7).reshape(1, 7))
        return bool(ok[0]), float(nid[0])

    def close(self):
        if self._ctx:
            self._L.vlcal_nid_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
