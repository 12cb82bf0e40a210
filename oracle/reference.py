"""ctypes binding of oracle/_ref/libvlcal_ref.so -- the REFERENCE's own sources of the NID path, compiled from a
reference checkout against the stand-in headers in oracle/ref_standin/ (oracle/ref_shim.cpp,
`make -C oracle ref REF=<checkout>`, or build() with VLCAL_REFERENCE=<checkout> in the environment).

TEST INFRASTRUCTURE ONLY: tests/golden/make_reference_outputs.py uses it to record what the reference returns on the test
inputs (tests/golden/reference_outputs.json), which tests/test_reference_pin.py pins the oracle against.  The library is
git-ignored.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libvlcal_ref.so")
REFERENCE_ROOT = os.environ.get("VLCAL_REFERENCE", "")  # a checkout of koide3/direct_visual_lidar_calibration

NM_FUNC = C.CFUNCTYPE(C.c_double, C.POINTER(C.c_double), C.c_void_p)
_lib = None


def build() -> str | None:
    """(Re)build when the reference tree is present; returns the library path, or None when there is neither a
    reference tree nor a prebuilt library."""
    if REFERENCE_ROOT and os.path.isdir(os.path.join(REFERENCE_ROOT, "src")):
        subprocess.run(["make", "-C", _HERE, "-s", "ref", f"REF={REFERENCE_ROOT}"], check=True)
    return LIB_PATH if os.path.exists(LIB_PATH) else None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB_PATH)
        L.ref_create_camera.restype = C.c_void_p
        L.ref_create_camera.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.ref_free_camera.argtypes = [C.c_void_p]
        L.ref_project.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.ref_estimate_camera_fov.restype = C.c_double
        L.ref_estimate_camera_fov.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ref_nelder_mead.restype = C.c_int
        L.ref_nelder_mead.argtypes = [C.c_int, NM_FUNC, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.ref_nid_calculate.restype = C.c_int
        L.ref_nid_calculate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.ref_view_cull.restype = C.c_int64
        L.ref_view_cull.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.ref_generate_lidar_image.restype = C.c_int
        L.ref_generate_lidar_image.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.ref_nid_cost_bspline.restype = C.c_int
        L.ref_nid_cost_bspline.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.POINTER(C.c_double)]
        L.ref_calibrate_nelder_mead.restype = C.c_int
        L.ref_calibrate_nelder_mead.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.ref_nid_cost_bspline_jet.restype = C.c_int
        L.ref_nid_cost_bspline_jet.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.POINTER(C.c_double), C.c_void_p]
        _lib = L
    return _lib


def _f64(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float64)


class Camera:
    """camera::create_camera(model, intrinsics, distortion); `.handle` is None where the reference returns nullptr."""

    def __init__(self, model: str, intrinsics, distortion):
        intr, dist = _f64(intrinsics).reshape(-1), _f64(distortion).reshape(-1)
        self.handle = lib().ref_create_camera(model.encode(), intr.ctypes.data, intr.size, dist.ctypes.data, dist.size)

    def __del__(self):
        if getattr(self, "handle", None):
            lib().ref_free_camera(self.handle)
            self.handle = None


def project(cam: Camera, points_xyz) -> np.ndarray:
    p = _f64(points_xyz).reshape(-1, 3)
    uv = np.empty((p.shape[0], 2))
    lib().ref_project(cam.handle, p.shape[0], p.ctypes.data, uv.ctypes.data)
    return uv


def estimate_camera_fov(cam: Camera, width: int, height: int) -> float:
    return float(lib().ref_estimate_camera_fov(cam.handle, int(width), int(height)))


def nelder_mead(f, x0, init_step=0.1, alpha=1.0, gamma=2.0, rho=0.5, sigma=0.5, max_iterations=1024, convergence_var_thresh=1e-5):
    """dfo::NelderMead<N>::optimize (N in {2, 3, 6}); `calls` lists the objective evaluations in order."""
    x0 = _f64(x0).reshape(-1)
    n = int(x0.size)
    calls = []

    def _cb(xp, _user):
        x = np.array([xp[i] for i in range(n)])
        y = float(f(x))
        calls.append((x, y))
        return y

    params = _f64([init_step, alpha, gamma, rho, sigma, max_iterations, convergence_var_thresh])
    out_x = np.empty(n)
    y, conv, its = C.c_double(), C.c_int(), C.c_int()
    rc = lib().ref_nelder_mead(n, NM_FUNC(_cb), None, x0.ctypes.data, params.ctypes.data, out_x.ctypes.data, C.byref(y), C.byref(conv), C.byref(its))
    assert rc == 0, f"dfo::NelderMead<{n}> is not instantiated in ref_shim.cpp"
    return {"converged": bool(conv.value), "num_iterations": int(its.value), "x": out_x, "y": float(y.value), "num_evaluations": len(calls), "calls": calls}


def _colmajor(T) -> np.ndarray:
    return np.ascontiguousarray(_f64(T).reshape(4, 4).T).reshape(-1)


def nid_calculate(cam: Camera, image, points_xyzw, intensities, bins, Ts) -> np.ndarray:
    """CostCalculatorNID(proj, data, {bins}).calculate(T) for every T of Ts (row-major 4x4 each)."""
    image = np.ascontiguousarray(image, dtype=np.uint8)
    pts, ins = _f64(points_xyzw).reshape(-1, 4), _f64(intensities).reshape(-1)
    Ts = _f64(Ts).reshape(-1, 4, 4)
    tc = np.concatenate([_colmajor(T) for T in Ts])
    out = np.empty(Ts.shape[0])
    H, W = image.shape
    lib().ref_nid_calculate(cam.handle, image.ctypes.data, W, H, image.strides[0], pts.ctypes.data, ins.ctypes.data, pts.shape[0], int(bins), Ts.shape[0], tc.ctypes.data, out.ctypes.data)
    return out


def view_cull(cam: Camera, width, height, enable_depth, points_xyzw, T) -> np.ndarray:
    pts = _f64(points_xyzw).reshape(-1, 4)
    idx = np.empty(max(pts.shape[0], 1), dtype=np.int32)
    t = _colmajor(T)
    m = lib().ref_view_cull(cam.handle, int(width), int(height), int(bool(enable_depth)), pts.ctypes.data, pts.shape[0], t.ctypes.data, idx.ctypes.data)
    return idx[:m].copy()


def generate_lidar_image(cam: Camera, width, height, T, points_xyzw, intensities):
    """vlcal::generate_lidar_image(proj, {W,H}, T, points) -> (intensity image float64 (H,W), index map int32 (H,W))."""
    pts, ins = _f64(points_xyzw).reshape(-1, 4), _f64(intensities).reshape(-1)
    inten = np.empty((height, width))
    index = np.empty((height, width), dtype=np.int32)
    t = _colmajor(T)
    lib().ref_generate_lidar_image(cam.handle, int(width), int(height), t.ctypes.data, pts.ctypes.data, ins.ctypes.data, pts.shape[0], inten.ctypes.data, index.ctypes.data)
    return inten, index


def nid_cost_bspline(cam: Camera, image_u8, points_xyzw, intensities, bins, T_params7):
    """NIDCost(proj, image / 255 as CV_64FC1, points, bins)(T_params7, &residual) -> (ok, residual)."""
    image = np.ascontiguousarray(image_u8, dtype=np.uint8)
    img64 = np.ascontiguousarray(image.astype(np.float64) * (1.0 / 255.0))  # convertTo(CV_64FC1, 1 / 255.0)
    pts, ins = _f64(points_xyzw).reshape(-1, 4), _f64(intensities).reshape(-1)
    tp = _f64(T_params7).reshape(7)
    out = C.c_double(float("nan"))
    H, W = image.shape
    ok = lib().ref_nid_cost_bspline(cam.handle, img64.ctypes.data, W, H, pts.ctypes.data, ins.ctypes.data, pts.shape[0], int(bins), tp.ctypes.data, C.byref(out))
    return bool(ok), float(out.value)


def calibrate_nelder_mead(cam: Camera, bags, init_T, max_outer_iterations=10, max_inner_iterations=256, delta_trans_thresh=0.1, delta_rot_thresh=0.5 * np.pi / 180.0,
                          disable_z_buffer_culling=False, nid_bins=16, nelder_mead_init_step=1e-3, nelder_mead_convergence_criteria=1e-8, callback_capacity=8192):
    """VisualCameraCalibration(proj, dataset, params).calibrate(init_T), NID_NELDER_MEAD branch.
    bags: list of (image_u8[H, W], points_xyzw[N, 4], intensities[N]), all images of one size.  Returns the final pose and the
    poses handed to params.callback (every new best cost, visual_camera_calibration.cpp:112-116)."""
    keep = []
    for image, pts, ins in bags:
        keep.append((np.ascontiguousarray(image, dtype=np.uint8), _f64(pts).reshape(-1, 4), _f64(ins).reshape(-1)))
    n = len(keep)
    H, W = keep[0][0].shape
    images = (C.c_void_p * n)(*[k[0].ctypes.data for k in keep])
    strides = (C.c_int * n)(*[k[0].strides[0] for k in keep])
    points = (C.c_void_p * n)(*[k[1].ctypes.data for k in keep])
    intens = (C.c_void_p * n)(*[k[2].ctypes.data for k in keep])
    counts = (C.c_int64 * n)(*[k[1].shape[0] for k in keep])
    calib = _f64([max_outer_iterations, max_inner_iterations, delta_trans_thresh, delta_rot_thresh, 1.0 if disable_z_buffer_culling else 0.0, nid_bins, nelder_mead_init_step,
                  nelder_mead_convergence_criteria])
    t0 = _colmajor(init_T)
    out = np.empty(16)
    cb = np.zeros((callback_capacity, 16))
    count = C.c_int(0)
    lib().ref_calibrate_nelder_mead(cam.handle, n, images, W, H, strides, points, intens, counts, calib.ctypes.data, t0.ctypes.data, out.ctypes.data, cb.ctypes.data, callback_capacity,
                                    C.byref(count))
    k = min(count.value, callback_capacity)
    return {"T": out.reshape(4, 4).T.copy(), "callback_T": cb[:k].reshape(k, 4, 4).transpose(0, 2, 1).copy(), "num_callbacks": count.value}


def nid_cost_bspline_jet(cam: Camera, image_u8, points_xyzw, intensities, bins, T_params7):
    """NIDCost::operator()<ceres::Jet<double, 7>> -> (ok, residual, d residual / d(qx qy qz qw tx ty tz))."""
    image = np.ascontiguousarray(image_u8, dtype=np.uint8)
    img64 = np.ascontiguousarray(image.astype(np.float64) * (1.0 / 255.0))
    pts, ins = _f64(points_xyzw).reshape(-1, 4), _f64(intensities).reshape(-1)
    tp = _f64(T_params7).reshape(7)
    out = C.c_double(float("nan"))
    grad = np.full(7, np.nan)
    H, W = image.shape
    ok = lib().ref_nid_cost_bspline_jet(cam.handle, img64.ctypes.data, W, H, pts.ctypes.data, ins.ctypes.data, pts.shape[0], int(bins), tp.ctypes.data, C.byref(out), grad.ctypes.data)
    return bool(ok), float(out.value), grad
