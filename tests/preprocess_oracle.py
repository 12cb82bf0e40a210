"""ctypes wrapper of tests/cpp/preprocess_oracle.c, the sequential CPU checker of preprocess_map's point stages (built on
first use into a temporary directory), plus the Eigen stand-in's virtual-camera rotation (tests/cpp/virtual_rotation_check.cpp)
and a CPU pipeline of the whole preprocess_map from these, the oracle's generate_lidar_image and cv2."""
import ctypes as C
import json
import math
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="preprocess_oracle_"), "libpreprocess_oracle.so")
        subprocess.run(
            ["/usr/bin/gcc", "-O2", "-std=c11", "-D_DEFAULT_SOURCE", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-o", out,
             os.path.join(_HERE, "cpp", "preprocess_oracle.c"), "-lm"],
            check=True,
        )
        L = C.CDLL(out)
        vp = C.c_void_p
        L.orc_approximate_voxel_grid.argtypes = [vp, C.c_int64, C.c_double, vp]
        L.orc_approximate_voxel_grid.restype = C.c_int64
        L.orc_voxel_grid_fov.argtypes = [vp, C.c_int64, vp, C.POINTER(C.c_int)]
        L.orc_voxel_grid_fov.restype = C.c_int64
        L.orc_rank_equalize.argtypes = [vp, C.c_int64, vp]
        L.orc_rank_equalize.restype = None
        L.orc_min_bearing_cosine.argtypes = [vp, C.c_int64]
        L.orc_min_bearing_cosine.restype = C.c_double
        L.orc_virtual_lidar_rotation.argtypes = [C.c_int, vp]
        L.orc_virtual_lidar_rotation.restype = None
        _lib = L
    return _lib


def _f32(a, cols):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(-1, cols))


def approximate_voxel_grid(points_xyzi, leaf_size):
    p = _f32(points_xyzi, 4)
    out = np.empty((max(p.shape[0], 1), 4), np.float32)
    m = lib().orc_approximate_voxel_grid(p.ctypes.data, p.shape[0], float(leaf_size), out.ctypes.data)
    return out[:m].copy()


def voxel_grid_fov(points_xyz):
    p = _f32(np.asarray(points_xyz, dtype=np.float32)[:, :3], 3)
    out = np.empty((max(p.shape[0], 1), 3), np.float32)
    unfiltered = C.c_int()
    m = lib().orc_voxel_grid_fov(p.ctypes.data, p.shape[0], out.ctypes.data, C.byref(unfiltered))
    return out[:m].copy(), bool(unfiltered.value)


def rank_equalize(intensities):
    v = np.ascontiguousarray(np.asarray(intensities, dtype=np.float32).reshape(-1))
    out = np.empty(v.shape[0])
    lib().orc_rank_equalize(v.ctypes.data, v.shape[0], out.ctypes.data)
    return out


def min_bearing_cosine(vertices):
    v = _f32(vertices, 3)
    return lib().orc_min_bearing_cosine(v.ctypes.data, v.shape[0])


def virtual_lidar_rotation(wide: bool) -> np.ndarray:
    R = np.empty(9)
    lib().orc_virtual_lidar_rotation(1 if wide else 0, R.ctypes.data)
    return R.reshape(3, 3)


def standin_rotation_check():
    """-> (quaternion (w, x, y, z), images of e_k under it (3, 3), images of e_k under AngleAxisd(-pi/2, X) (3, 3)), as the
    Eigen stand-in computes them."""
    d = tempfile.mkdtemp(prefix="vrot_")
    exe = os.path.join(d, "vrot")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", f"-I{os.path.join(_ROOT, 'oracle', 'ref_standin')}", "-o", exe,
                    os.path.join(_HERE, "cpp", "virtual_rotation_check.cpp")], check=True)
    lines = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split("\n")
    q = [float.fromhex(t) for t in lines[0].split()]
    rows = [[float.fromhex(t) for t in ln.split()] for ln in lines[1:4]]
    return q, np.array([r[:3] for r in rows]), np.array([r[3:] for r in rows])


def preprocess_map_cpu(oracle, map_cloud_xyzi, image_path, dst_path, map_path, camera_model, intrinsics, distortion, voxel_resolution=0.002):
    """preprocess_map from the sequential checker, the hull of the product's host code (scipy qhull), the oracle's
    generate_lidar_image and cv2 -> writes the same five files into dst_path."""
    import cv2

    from direct_visual_lidar_calibration_b200 import io as vio
    from direct_visual_lidar_calibration_b200 import preprocess as P

    os.makedirs(dst_path, exist_ok=True)
    cv2.imwrite(os.path.join(dst_path, "000000.png"), cv2.equalizeHist(cv2.imread(image_path, 0)))
    filtered = approximate_voxel_grid(map_cloud_xyzi, voxel_resolution)
    inten = rank_equalize(filtered[:, 3])
    vio.save_ply_binary(os.path.join(dst_path, "000000.ply"), filtered[:, :3], inten)
    cand, _ = voxel_grid_fov(filtered[:, :3])
    fov = math.acos(min_bearing_cosine(P.hull_vertices(cand)))
    wide = not (fov < 150.0 * math.pi / 180.0)
    if wide:
        W, H, model, intr = 1920, 960, "equirectangular", [1920.0, 960.0]
    else:
        W, H = 1024, 1024
        fx = W / (2.0 * math.tan(fov / 2.0))
        model, intr = "plumb_bob", [fx, fx, W / 2.0, H / 2.0]
    R = virtual_lidar_rotation(wide)
    T = np.eye(4)
    T[:3, :3] = R.T
    for i in range(3):
        T[i, 3] = -((R[0, i] * 0.0 + R[1, i] * 0.0) + R[2, i] * 0.0)
    pts = np.concatenate([filtered[:, :3].astype(np.float64), np.ones((filtered.shape[0], 1))], axis=1)
    cam = oracle.create_camera(model, intr, [])
    img, idx = oracle.generate_lidar_image(cam, W, H, T, pts, inten)
    cv2.imwrite(os.path.join(dst_path, "000000_lidar_intensities.png"), np.clip(np.rint(img * 255.0), 0, 255).astype(np.uint8))
    vio.save_lidar_indices(os.path.join(dst_path, "000000_lidar_indices.png"), idx)
    config = {
        "camera": {"camera_model": camera_model, "distortion_coeffs": list(distortion), "intrinsics": list(intrinsics)},
        "meta": {"bag_names": ["000000"], "camera_info_topic": "N/A", "data_path": map_path, "image_topic": "N/A", "intensity_channel": "N/A", "points_topic": "N/A"},
    }
    with open(os.path.join(dst_path, "calib.json"), "w") as f:
        f.write(json.dumps(config, indent=2, sort_keys=True) + "\n")
    return {"filtered": filtered, "intensities": inten, "fov": fov, "model": model, "intrinsics": intr}
