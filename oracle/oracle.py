"""ctypes binding of the CPU ORACLE (oracle/vlcal_oracle.c) -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package (direct_visual_lidar_calibration_b200) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libvlcal_oracle.so")

CAMERA_MODELS = ["plumb_bob", "fisheye", "atan", "omnidir", "equirectangular", "rational_polynomial"]


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in ("vlcal_oracle.c", "vlcal_oracle_grad.c", "vlcal_oracle.h")]
    stale = (not os.path.exists(_LIB_PATH)) or any(os.path.exists(p) and os.path.getmtime(p) > os.path.getmtime(_LIB_PATH) for p in srcs)
    if force or stale:
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


class Camera(C.Structure):
    _fields_ = [("model", C.c_int), ("n_intr", C.c_int), ("n_dist", C.c_int), ("intr", C.c_double * 5), ("dist", C.c_double * 8)]


class NMParams(C.Structure):
    _fields_ = [
        ("init_step", C.c_double),
        ("alpha", C.c_double),
        ("gamma", C.c_double),
        ("rho", C.c_double),
        ("sigma", C.c_double),
        ("max_iterations", C.c_int),
        ("convergence_var_thresh", C.c_double),
    ]


class NMResult(C.Structure):
    _fields_ = [("converged", C.c_int), ("num_iterations", C.c_int), ("x", C.c_double * 8), ("y", C.c_double), ("num_evaluations", C.c_int)]


NM_FUNC = C.CFUNCTYPE(C.c_double, C.POINTER(C.c_double), C.c_void_p)


class Bag(C.Structure):
    _fields_ = [
        ("image", C.c_void_p),
        ("width", C.c_int),
        ("height", C.c_int),
        ("row_stride", C.c_int),
        ("points_xyzw", C.c_void_p),
        ("intensities", C.c_void_p),
        ("n", C.c_int64),
    ]


class CalibParams(C.Structure):
    _fields_ = [
        ("max_outer_iterations", C.c_int),
        ("max_inner_iterations", C.c_int),
        ("delta_trans_thresh", C.c_double),
        ("delta_rot_thresh", C.c_double),
        ("disable_z_buffer_culling", C.c_int),
        ("nid_bins", C.c_int),
        ("nelder_mead_init_step", C.c_double),
        ("nelder_mead_convergence_criteria", C.c_double),
    ]


class CalibStats(C.Structure):
    _fields_ = [
        ("outer_iterations", C.c_int),
        ("total_evaluations", C.c_int),
        ("inner_iterations", C.c_int * 16),
        ("inner_final_cost", C.c_double * 16),
        ("best_cost_last", C.c_double),
    ]


class Trace(C.Structure):
    _fields_ = [("evals", C.c_void_p), ("capacity", C.c_int), ("count", C.c_int)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        dp = C.POINTER(C.c_double)
        L.orc_create_camera.argtypes = [C.c_char_p, dp, C.c_int, dp, C.c_int, C.POINTER(Camera)]
        L.orc_create_camera.restype = C.c_int
        L.orc_project.argtypes = [C.POINTER(Camera), dp, dp]
        L.orc_project_n.argtypes = [C.POINTER(Camera), dp, C.c_int64, dp]
        L.orc_project_n.restype = None
        L.orc_se3_expmap_gtsam.argtypes = [dp, dp]
        L.orc_isometry_mul.argtypes = [dp, dp, dp]
        L.orc_isometry_inverse.argtypes = [dp, dp]
        L.orc_rotation_angle.argtypes = [dp]
        L.orc_rotation_angle.restype = C.c_double
        L.orc_estimate_camera_fov.argtypes = [C.POINTER(Camera), C.c_int, C.c_int]
        L.orc_estimate_camera_fov.restype = C.c_double
        L.orc_nm_default_params.argtypes = [C.POINTER(NMParams)]
        L.orc_nelder_mead.argtypes = [C.c_int, NM_FUNC, C.c_void_p, dp, C.POINTER(NMParams), C.POINTER(NMResult)]
        nid_args = [C.POINTER(Camera), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_double, dp, C.c_void_p]
        L.orc_nid_calculate.argtypes = nid_args
        L.orc_nid_calculate.restype = C.c_double
        L.orc_nid_calculate_omp.argtypes = nid_args
        L.orc_nid_calculate_omp.restype = C.c_double
        L.orc_nid_from_hist.argtypes = [C.c_void_p, C.c_int, dp, dp, dp, dp]
        L.orc_nid_from_hist.restype = C.c_double
        L.orc_view_cull.argtypes = [C.POINTER(Camera), C.c_int, C.c_int, C.c_double, C.c_int, C.c_void_p, C.c_int64, dp, C.c_void_p]
        L.orc_view_cull.restype = C.c_int64
        L.orc_generate_lidar_image.argtypes = [C.POINTER(Camera), C.c_int, C.c_int, dp, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.orc_generate_lidar_image.restype = None
        L.orc_set_bag_threads.argtypes = [C.c_int]
        L.orc_set_bag_threads.restype = None
        L.orc_nid_cost_bspline.argtypes = [C.POINTER(Camera), C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, dp, dp, C.c_void_p]
        L.orc_nid_cost_bspline.restype = C.c_int
        L.orc_nid_cost_bspline_grad.argtypes = [C.POINTER(Camera), C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, dp, dp, C.c_void_p, C.c_void_p]
        L.orc_nid_cost_bspline_grad.restype = C.c_int
        L.orc_calib_default_params.argtypes = [C.POINTER(CalibParams)]
        L.orc_estimate_pose_nelder_mead.argtypes = [C.POINTER(Camera), C.POINTER(Bag), C.c_int, C.POINTER(CalibParams), dp, dp, C.POINTER(NMResult), C.POINTER(Trace)]
        L.orc_calibrate.argtypes = [C.POINTER(Camera), C.POINTER(Bag), C.c_int, C.POINTER(CalibParams), dp, dp, C.POINTER(CalibStats), C.POINTER(Trace)]
        _lib = L
    return _lib


def _dp(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _f64(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


def T_to_colmajor(T) -> np.ndarray:
    """4x4 (row-major numpy) -> 16 doubles column-major (Eigen storage)."""
    return np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(4, 4).T).reshape(16)


def colmajor_to_T(v) -> np.ndarray:
    return np.asarray(v, dtype=np.float64).reshape(4, 4).T.copy()


def create_camera(model: str, intrinsics, distortion):
    """Mirror of camera::create_camera; returns None where the reference returns nullptr."""
    cam = Camera()
    intr = _f64(intrinsics).reshape(-1)
    dist = _f64(distortion).reshape(-1)
    intr_p = _dp(intr) if intr.size else C.POINTER(C.c_double)()
    dist_p = _dp(dist) if dist.size else C.POINTER(C.c_double)()
    rc = lib().orc_create_camera(model.encode(), intr_p, int(intr.size), dist_p, int(dist.size), C.byref(cam))
    return cam if rc == 0 else None


def project(cam: Camera, p) -> np.ndarray:
    pts = _f64(p).reshape(-1, 3)
    out = np.empty((pts.shape[0], 2))
    lib().orc_project_n(C.byref(cam), _dp(pts), pts.shape[0], _dp(out))  # orc_project per point
    return out if np.asarray(p).ndim > 1 else out[0]


def se3_expmap(x) -> np.ndarray:
    x = _f64(x).reshape(6)
    T = np.empty(16)
    lib().orc_se3_expmap_gtsam(_dp(x), _dp(T))
    return colmajor_to_T(T)


def isometry_mul(A, B) -> np.ndarray:
    a, b, c = T_to_colmajor(A), T_to_colmajor(B), np.empty(16)
    lib().orc_isometry_mul(_dp(a), _dp(b), _dp(c))
    return colmajor_to_T(c)


def rotation_angle(T) -> float:
    a = T_to_colmajor(T)
    return float(lib().orc_rotation_angle(_dp(a)))


def estimate_camera_fov(cam: Camera, width: int, height: int) -> float:
    return float(lib().orc_estimate_camera_fov(C.byref(cam), int(width), int(height)))


def nelder_mead(f, x0, init_step=0.1, max_iterations=1024, convergence_var_thresh=1e-5):
    x0 = _f64(x0).reshape(-1)
    n = int(x0.size)
    p = NMParams()
    lib().orc_nm_default_params(C.byref(p))
    p.init_step, p.max_iterations, p.convergence_var_thresh = init_step, max_iterations, convergence_var_thresh
    calls = []

    def _cb(xp, _user):
        x = np.array([xp[i] for i in range(n)])
        y = float(f(x))
        calls.append((x, y))
        return y

    r = NMResult()
    lib().orc_nelder_mead(n, NM_FUNC(_cb), None, _dp(x0), C.byref(p), C.byref(r))
    return {
        "converged": bool(r.converged),
        "num_iterations": int(r.num_iterations),
        "x": np.array(r.x[:n]),
        "y": float(r.y),
        "num_evaluations": int(r.num_evaluations),
        "calls": calls,
    }


def _check_inputs(image, points_xyzw, intensities):
    image = np.ascontiguousarray(image, dtype=np.uint8)
    pts = _f64(points_xyzw).reshape(-1, 4)
    ins = _f64(intensities).reshape(-1)
    assert pts.shape[0] == ins.shape[0]
    return image, pts, ins


def nid_calculate(cam, image, points_xyzw, intensities, bins, max_fov, T, omp=False):
    """CostCalculatorNID::calculate. Returns (nid, hist[bins(image), bins(lidar)])."""
    image, pts, ins = _check_inputs(image, points_xyzw, intensities)
    H, W = image.shape
    hist = np.zeros(bins * bins, dtype=np.int32)
    t = T_to_colmajor(T)
    fn = lib().orc_nid_calculate_omp if omp else lib().orc_nid_calculate
    nid = fn(C.byref(cam), image.ctypes.data, W, H, image.strides[0], pts.ctypes.data, ins.ctypes.data, pts.shape[0], int(bins), float(max_fov), _dp(t), hist.ctypes.data)
    # storage index = image_bin + lidar_bin*bins  ->  [lidar_bin, image_bin] -> transpose to [image_bin, lidar_bin]
    return float(nid), hist.reshape(bins, bins).T.copy()


def nid_from_hist(hist_image_by_lidar):
    h = np.asarray(hist_image_by_lidar, dtype=np.int32)
    bins = h.shape[0]
    flat = np.ascontiguousarray(h.T).reshape(-1)  # index = image_bin + lidar_bin*bins
    vals = [C.c_double() for _ in range(4)]
    nid = lib().orc_nid_from_hist(flat.ctypes.data, bins, *[C.byref(v) for v in vals])
    return float(nid), tuple(float(v.value) for v in vals)


def view_cull(cam, width, height, max_fov, enable_depth, points_xyzw, T):
    pts = _f64(points_xyzw).reshape(-1, 4)
    idx = np.empty(max(pts.shape[0], 1), dtype=np.int32)
    t = T_to_colmajor(T)
    m = lib().orc_view_cull(C.byref(cam), int(width), int(height), float(max_fov), int(bool(enable_depth)), pts.ctypes.data, pts.shape[0], _dp(t), idx.ctypes.data)
    return idx[:m].copy()


def generate_lidar_image(cam, width, height, T, points_xyzw, intensities):
    """generate_lidar_image (generate_lidar_image.cpp:8-41) -> (intensity image float64 (H,W), index map int32 (H,W))."""
    pts, ins = _f64(points_xyzw).reshape(-1, 4), _f64(intensities).reshape(-1)
    inten = np.empty((height, width))
    index = np.empty((height, width), dtype=np.int32)
    t = T_to_colmajor(T)
    lib().orc_generate_lidar_image(C.byref(cam), int(width), int(height), _dp(t), pts.ctypes.data, ins.ctypes.data, pts.shape[0], inten.ctypes.data, index.ctypes.data)
    return inten, index


def nid_cost_bspline(cam, image_u8, points_xyzw, intensities, bins, T_params7):
    image, pts, ins = _check_inputs(image_u8, points_xyzw, intensities)
    img64 = np.ascontiguousarray(image.astype(np.float64) * (1.0 / 255.0))  # convertTo(CV_64FC1, 1/255)
    H, W = image.shape
    tp = _f64(T_params7).reshape(7)
    out = C.c_double(float("nan"))
    hist = np.zeros(bins * bins)
    ok = lib().orc_nid_cost_bspline(C.byref(cam), img64.ctypes.data, W, H, pts.ctypes.data, ins.ctypes.data, pts.shape[0], int(bins), _dp(tp), C.byref(out), hist.ctypes.data)
    return bool(ok), float(out.value), hist.reshape(bins, bins).T.copy()


def nid_cost_bspline_grad(cam, image_u8, points_xyzw, intensities, bins, T_params7, return_hist=False):
    """NIDCost::operator()<Jet<double, 7>> -> (ok, nid, grad[7] w.r.t. qx qy qz qw tx ty tz[, hist[bins(image), bins(lidar), 8]])."""
    image, pts, ins = _check_inputs(image_u8, points_xyzw, intensities)
    img64 = np.ascontiguousarray(image.astype(np.float64) * (1.0 / 255.0))
    H, W = image.shape
    tp = _f64(T_params7).reshape(7)
    out = C.c_double(float("nan"))
    grad = np.full(7, np.nan)
    hist = np.zeros(bins * bins * 8)
    ok = lib().orc_nid_cost_bspline_grad(C.byref(cam), img64.ctypes.data, W, H, pts.ctypes.data, ins.ctypes.data, C.c_int64(pts.shape[0]), int(bins), _dp(tp), C.byref(out), grad.ctypes.data,
                                         hist.ctypes.data if return_hist else None)
    if return_hist:
        return bool(ok), float(out.value), grad, hist.reshape(bins, bins, 8).transpose(1, 0, 2).copy()
    return bool(ok), float(out.value), grad


def set_bag_threads(n: int):
    """Threads of the objective's loop over bags (0 = one per bag like the reference's OpenMP loop, 1 = serial)."""
    lib().orc_set_bag_threads(int(n))


def default_calib_params() -> CalibParams:
    p = CalibParams()
    lib().orc_calib_default_params(C.byref(p))
    return p


def _make_bags(bags):
    keep = []
    arr = (Bag * len(bags))()
    for i, (image, points_xyzw, intensities) in enumerate(bags):
        image, pts, ins = _check_inputs(image, points_xyzw, intensities)
        keep.append((image, pts, ins))
        arr[i].image = image.ctypes.data
        arr[i].width, arr[i].height, arr[i].row_stride = image.shape[1], image.shape[0], image.strides[0]
        arr[i].points_xyzw = pts.ctypes.data
        arr[i].intensities = ins.ctypes.data
        arr[i].n = pts.shape[0]
    return arr, keep


def estimate_pose_nelder_mead(cam, bags, init_T, params=None, trace_capacity=4096):
    """bags: list of (image_u8[H,W], points_xyzw[N,4], intensities[N]). Returns dict."""
    params = params or default_calib_params()
    arr, keep = _make_bags(bags)
    t0 = T_to_colmajor(init_T)
    out = np.empty(16)
    r = NMResult()
    tr_buf = np.zeros((trace_capacity, 7))
    tr = Trace(tr_buf.ctypes.data, trace_capacity, 0)
    lib().orc_estimate_pose_nelder_mead(C.byref(cam), arr, len(bags), C.byref(params), _dp(t0), _dp(out), C.byref(r), C.byref(tr))
    return {
        "T": colmajor_to_T(out),
        "x": np.array(r.x[:6]),
        "y": float(r.y),
        "num_iterations": int(r.num_iterations),
        "converged": bool(r.converged),
        "num_evaluations": int(r.num_evaluations),
        "trace": tr_buf[: min(tr.count, trace_capacity)].copy(),
    }


def calibrate(cam, bags, init_T, params=None, trace_capacity=16384):
    params = params or default_calib_params()
    arr, keep = _make_bags(bags)
    t0 = T_to_colmajor(init_T)
    out = np.empty(16)
    st = CalibStats()
    tr_buf = np.zeros((trace_capacity, 7))
    tr = Trace(tr_buf.ctypes.data, trace_capacity, 0)
    lib().orc_calibrate(C.byref(cam), arr, len(bags), C.byref(params), _dp(t0), _dp(out), C.byref(st), C.byref(tr))
    k = st.outer_iterations
    return {
        "T": colmajor_to_T(out),
        "outer_iterations": int(k),
        "total_evaluations": int(st.total_evaluations),
        "inner_iterations": list(st.inner_iterations[:k]),
        "inner_final_cost": list(st.inner_final_cost[:k]),
        "trace": tr_buf[: min(tr.count, trace_capacity)].copy(),
    }
