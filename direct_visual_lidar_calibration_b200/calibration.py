"""vlcal::VisualCameraCalibration mirror (reference: include/vlcal/calib/visual_camera_calibration.hpp,
src/vlcal/calib/visual_camera_calibration.cpp): the NID_NELDER_MEAD branch (:70-139, trajectory-exact, the hot path) and
the NID_BFGS branch (:187-238: mode-B value + gradient on the GPU, Ceres-free BFGS -- see bfgs.py)."""
from __future__ import annotations

import ctypes as C
import enum
import math

import numpy as np

from . import _lib
from .camera import GenericCamera, _dp
from .cost import T_to_colmajor, VisualLiDARData, colmajor_to_T


class RegistrationType(enum.Enum):  # visual_camera_calibration.hpp:8
    NID_BFGS = 0
    NID_NELDER_MEAD = 1


def se3_expmap(x) -> np.ndarray:
    """gtsam::Pose3::Expmap(x).matrix() (x = omega, v)."""
    x = np.ascontiguousarray(np.asarray(x, dtype=np.float64)).reshape(6)
    T = np.empty(16)
    _lib.check(_lib.load_library().vlcal_se3_expmap_gtsam(_dp(x), _dp(T)))
    return colmajor_to_T(T)[0]


def estimate_camera_fov(proj: GenericCamera, image_size) -> float:
    """vlcal::estimate_camera_fov(proj, {W,H}) (src/vlcal/common/estimate_fov.cpp:36-51)."""
    out = C.c_double()
    _lib.check(_lib.load_library().vlcal_estimate_camera_fov(proj.model_id, _dp(proj.intrinsics), proj.intrinsics.size, _dp(proj.distortion), proj.distortion.size, int(image_size[0]), int(image_size[1]), C.byref(out)))
    return float(out.value)


def outer_step_delta(T, new_T):
    """(delta_t, delta_r) of the outer loop (visual_camera_calibration.cpp:50-54): new_T^-1 * T as isometries, its
    translation norm and AngleAxisd angle -- the same bits the Nelder-Mead branch's outer loop decides on."""
    dt, dr = C.c_double(), C.c_double()
    _lib.check(_lib.load_library().vlcal_outer_step_delta(_dp(T_to_colmajor(T)), _dp(T_to_colmajor(new_T)), C.byref(dt), C.byref(dr)))
    return float(dt.value), float(dr.value)


class VisualCameraCalibrationParams:
    def __init__(self):  # visual_camera_calibration.hpp:12-26
        self.max_outer_iterations = 10
        self.max_inner_iterations = 256
        self.delta_trans_thresh = 0.1
        self.delta_rot_thresh = 0.5 * math.pi / 180.0
        self.disable_z_buffer_culling = False
        self.nid_bins = 16
        # the reference's default is NID_BFGS (visual_camera_calibration.hpp:22, src/calibrate.cpp:176); the hot path of this
        # repository is the Nelder-Mead branch, which stays the default here
        self.registration_type = RegistrationType.NID_NELDER_MEAD
        self.bfgs_params = None  # _lib.BfgsParams; None = Ceres' documented defaults (bfgs.default_bfgs_params())
        self.nelder_mead_init_step = 1e-3
        self.nelder_mead_convergence_criteria = 1e-8
        self.callback = None  # callable(T_camera_lidar[4,4]) on every best-cost improvement

    def to_c(self) -> _lib.CalibParams:
        return _lib.CalibParams(
            self.max_outer_iterations, self.max_inner_iterations, self.delta_trans_thresh, self.delta_rot_thresh,
            int(self.disable_z_buffer_culling), self.nid_bins, self.nelder_mead_init_step, self.nelder_mead_convergence_criteria,
        )


def _make_bags(dataset):
    arr = (_lib.Bag * len(dataset))()
    for i, d in enumerate(dataset):
        h, w = d.image.shape
        arr[i].image = d.image.ctypes.data
        arr[i].width, arr[i].height, arr[i].row_stride_bytes = w, h, d.image.strides[0]
        arr[i].points_xyzw = d.points.ctypes.data
        arr[i].intensities = d.intensities.ctypes.data
        arr[i].n_points = d.size()
    return arr


def _stats_dict(st: _lib.CalibStats):
    k = min(st.outer_iterations, 16)
    return {
        "outer_iterations": int(st.outer_iterations), "total_evaluations": int(st.total_evaluations),
        "total_evaluations_computed": int(st.total_evaluations_computed), "total_batches": int(st.total_batches),
        "inner_iterations": list(st.inner_iterations[:k]), "inner_final_cost": list(st.inner_final_cost[:k]), "culled_points": list(st.culled_points[:k]),
        "kernel_launches": int(st.kernel_launches), "kernel_ms_total": float(st.kernel_ms_total),
        "upload_ms": float(st.upload_ms), "cull_ms": float(st.cull_ms), "solve_ms": float(st.solve_ms),
    }


class VisualCameraCalibration:
    """VisualCameraCalibration(proj, dataset, params).calibrate(init_T_camera_lidar) -> T_camera_lidar (4x4).

    allreduce: optional callable(np.ndarray) -> None that sums the per-pose partial costs over all ranks in place
    (multi-GPU bag sharding: each rank passes only its local bags)."""

    def __init__(self, proj: GenericCamera, dataset, params: VisualCameraCalibrationParams | None = None, device: int = -1, allreduce=None, profiling: bool = False):
        self.proj = proj
        self.dataset = list(dataset)
        self.params = params or VisualCameraCalibrationParams()
        self.device = device
        self.allreduce = allreduce
        self.profiling = profiling
        self.stats = None
        self.trace = []  # (T, cost) on each best-cost improvement

    def _callbacks(self):
        def _pose_cb(Tp, cost, _user):
            T = colmajor_to_T(np.ctypeslib.as_array(Tp, shape=(16,)))[0]
            self.trace.append((T, float(cost)))
            if self.params.callback:
                self.params.callback(T)

        def _allreduce(vals, count, _user):
            a = np.ctypeslib.as_array(vals, shape=(count,))
            self.allreduce(a)

        cb = _lib.POSE_CALLBACK(_pose_cb)
        ar = _lib.ALLREDUCE_FN(_allreduce) if self.allreduce else _lib.ALLREDUCE_FN()
        return cb, ar

    def _check_type(self):
        if self.params.registration_type != RegistrationType.NID_NELDER_MEAD:
            raise _lib.VlcalError(_lib.ERR_UNSUPPORTED, "this entry point is the Nelder-Mead branch; use calibrate() / estimate_pose_bfgs() for RegistrationType.NID_BFGS")

    def estimate_pose_bfgs(self, init_T_camera_lidar):
        """One inner BFGS solve (visual_camera_calibration.cpp:187-238): cull every bag at the start pose (:196), build one
        NIDCost per bag on the image / 255 (:198-206), minimise their sum (:208-228).  Returns (T, result dict)."""
        from . import bfgs
        from .cost import NIDCost
        from .culling import ViewCulling, ViewCullingParams

        first = self.dataset[0]
        culling = ViewCulling(self.proj, (first.image.shape[1], first.image.shape[0]), ViewCullingParams(not self.params.disable_z_buffer_culling), device=self.device)
        costs = []
        for d in self.dataset:
            pts, ins = culling.cull(d.points, d.intensities, init_T_camera_lidar)
            costs.append(NIDCost(self.proj, VisualLiDARData(d.image, pts, ins), self.params.nid_bins, device=self.device))

        def _cb(T, cost):
            self.trace.append((T, cost))
            if self.params.callback:
                self.params.callback(T)

        try:
            T, r = bfgs.estimate_pose_bfgs_on_costs(costs, init_T_camera_lidar, self.params.bfgs_params, _cb, self.allreduce)
        finally:
            for c in costs:
                c.close()
        return T, r

    def _calibrate_bfgs(self, init_T_camera_lidar) -> np.ndarray:
        """Outer loop of visual_camera_calibration.cpp:35-68 around estimate_pose_bfgs."""
        T = np.array(init_T_camera_lidar, dtype=np.float64).reshape(4, 4)
        inner = []
        for _ in range(self.params.max_outer_iterations):
            new_T, r = self.estimate_pose_bfgs(T)
            inner.append(r)
            delta_t, delta_r = outer_step_delta(T, new_T)
            T = new_T
            if delta_t < self.params.delta_trans_thresh and delta_r < self.params.delta_rot_thresh:
                break
        self.stats = {"outer_iterations": len(inner), "inner": inner, "total_evaluations": sum(r["evaluations"] for r in inner)}
        return T

    def calibrate(self, init_T_camera_lidar) -> np.ndarray:
        if self.params.registration_type == RegistrationType.NID_BFGS:
            return self._calibrate_bfgs(init_T_camera_lidar)
        L = _lib.load_library()
        bags = _make_bags(self.dataset)
        cb, ar = self._callbacks()
        p = self.params.to_c()
        T0 = T_to_colmajor(init_T_camera_lidar)
        out = np.empty(16)
        st = _lib.CalibStats()
        _lib.check(
            L.vlcal_calibrate_nelder_mead(
                self.device, self.proj.model_id, _dp(self.proj.intrinsics), self.proj.intrinsics.size, _dp(self.proj.distortion), self.proj.distortion.size,
                bags, len(self.dataset), C.byref(p), _dp(T0), cb, ar, None, int(self.profiling), _dp(out), C.byref(st),
            )
        )
        self.stats = _stats_dict(st)
        return colmajor_to_T(out)[0]

    def estimate_pose_nelder_mead(self, init_T_camera_lidar):
        """One inner solve (visual_camera_calibration.cpp:70-139). Returns (T, nm_result dict)."""
        self._check_type()
        L = _lib.load_library()
        bags = _make_bags(self.dataset)
        cb, ar = self._callbacks()
        p = self.params.to_c()
        T0 = T_to_colmajor(init_T_camera_lidar)
        out = np.empty(16)
        st = _lib.CalibStats()
        res = _lib.NMResult()
        _lib.check(
            L.vlcal_estimate_pose_nelder_mead(
                self.device, self.proj.model_id, _dp(self.proj.intrinsics), self.proj.intrinsics.size, _dp(self.proj.distortion), self.proj.distortion.size,
                bags, len(self.dataset), C.byref(p), _dp(T0), cb, ar, None, int(self.profiling), _dp(out), C.byref(res), C.byref(st),
            )
        )
        self.stats = _stats_dict(st)
        r = {
            "converged": bool(res.converged), "num_iterations": int(res.num_iterations), "x": np.array(res.x[:6]), "y": float(res.y),
            "num_evaluations": int(res.num_evaluations), "num_batches": int(res.num_batches), "num_evaluations_computed": int(res.num_evaluations_computed),
        }
        return colmajor_to_T(out)[0], r


def record_solve_trace(enable: bool):
    """Test hook: keep (True) or stop keeping (False) the evaluations of the calling thread's inner solves for
    last_solve_trace(); off by default."""
    _lib.check(_lib.load_library().vlcal_nid_debug_record_solve_trace(int(enable)))


def last_solve_trace() -> np.ndarray:
    """(n, 7) rows {x[6], y}: every evaluation of the calling thread's last Nelder-Mead inner solve, in the reference's
    order, as its best-cost callback logic saw them (test hook; needs record_solve_trace(True) before the solve)."""
    L = _lib.load_library()
    n = C.c_int()
    _lib.check(L.vlcal_nid_debug_last_solve_trace(0, None, C.byref(n)))
    rows = np.zeros((n.value, 7))
    _lib.check(L.vlcal_nid_debug_last_solve_trace(n.value, _dp(rows), C.byref(n)))
    return rows


def estimate_pose_on_costs(costs, init_T_camera_lidar, params: VisualCameraCalibrationParams | None = None, allreduce=None, callback=None):
    """Nelder-Mead over already-built CostCalculatorNID objects (the `costs` vector of visual_camera_calibration.cpp:75-127)."""
    L = _lib.load_library()
    params = params or VisualCameraCalibrationParams()
    handles = (C.c_void_p * len(costs))(*[c.handle for c in costs])

    def _pose_cb(Tp, cost, _user):
        callback(colmajor_to_T(np.ctypeslib.as_array(Tp, shape=(16,)))[0], float(cost))

    def _allreduce(vals, count, _user):
        allreduce(np.ctypeslib.as_array(vals, shape=(count,)))

    # no callback: the null one, so the library knows that nobody observes the evaluations (it then skips scoring the
    # centroid of every iteration, whose value feeds no decision)
    cb = _lib.POSE_CALLBACK(_pose_cb) if callback else _lib.POSE_CALLBACK()
    ar = _lib.ALLREDUCE_FN(_allreduce) if allreduce else _lib.ALLREDUCE_FN()
    p = params.to_c()
    T0 = T_to_colmajor(init_T_camera_lidar)
    out = np.empty(16)
    res = _lib.NMResult()
    _lib.check(L.vlcal_estimate_pose_nelder_mead_ctx(handles, len(costs), C.byref(p), _dp(T0), cb, ar, None, _dp(out), C.byref(res)))
    r = {
        "converged": bool(res.converged), "num_iterations": int(res.num_iterations), "x": np.array(res.x[:6]), "y": float(res.y),
        "num_evaluations": int(res.num_evaluations), "num_batches": int(res.num_batches), "num_evaluations_computed": int(res.num_evaluations_computed),
    }
    return colmajor_to_T(out)[0], r


def estimate_poses_on_costs(costs, init_Ts, bag_mask=None, params: VisualCameraCalibrationParams | None = None):
    """S independent Nelder-Mead solves over already-built CostCalculatorNID objects in ONE persistent launch: solve s
    starts from init_Ts[s] and sums the costs b with bag_mask[s, b] (default: all), each exactly as
    estimate_pose_on_costs([costs[b] for b in its bags], init_Ts[s], params) would run it.  Returns (T (S, 4, 4), list of
    result dicts)."""
    L = _lib.load_library()
    params = params or VisualCameraCalibrationParams()
    T0 = T_to_colmajor(init_Ts)
    S = T0.shape[0]
    mask = np.ones((S, len(costs)), dtype=np.uint8) if bag_mask is None else np.ascontiguousarray(np.asarray(bag_mask, dtype=bool).astype(np.uint8))
    if mask.shape != (S, len(costs)):
        raise ValueError(f"bag_mask must be ({S}, {len(costs)})")
    handles = (C.c_void_p * len(costs))(*[c.handle for c in costs])
    p = params.to_c()
    out = np.empty((S, 16))
    res = (_lib.NMResult * S)()
    _lib.check(L.vlcal_estimate_poses_nelder_mead_ctx(handles, len(costs), C.byref(p), S, _dp(T0), mask.ctypes.data, _dp(out), res))
    rs = [
        {"converged": bool(r.converged), "num_iterations": int(r.num_iterations), "x": np.array(r.x[:6]), "y": float(r.y),
         "num_evaluations": int(r.num_evaluations), "num_batches": int(r.num_batches), "num_evaluations_computed": int(r.num_evaluations_computed)}
        for r in res
    ]
    return colmajor_to_T(out), rs
