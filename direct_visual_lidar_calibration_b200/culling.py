"""vlcal::ViewCulling mirror (reference: include/vlcal/calib/view_culling.hpp, src/vlcal/calib/view_culling.cpp)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .camera import GenericCamera, _dp
from .cost import T_to_colmajor


class ViewCullingParams:
    def __init__(self, enable_depth_buffer_culling: bool = True):  # view_culling.hpp:10-12
        self.enable_depth_buffer_culling = enable_depth_buffer_culling


class ViewCulling:
    """ViewCulling(proj, image_size=(W,H), params).cull(points, T_camera_lidar) -> kept indices (ascending)."""

    def __init__(self, proj: GenericCamera, image_size, params: ViewCullingParams | None = None, device: int = -1):
        self.proj = proj
        self.image_size = (int(image_size[0]), int(image_size[1]))
        self.params = params or ViewCullingParams()
        self.device = device

    def cull_indices(self, points, T_camera_lidar, max_fov: float | None = None) -> np.ndarray:
        L = _lib.load_library()
        pts = np.asarray(points, dtype=np.float64)
        if pts.shape[1] == 3:
            pts = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1)
        pts = np.ascontiguousarray(pts)
        idx = np.empty(max(pts.shape[0], 1), dtype=np.int32)
        kept = C.c_int64()
        T = T_to_colmajor(T_camera_lidar)
        _lib.check(
            L.vlcal_view_cull(
                self.device, self.proj.model_id, _dp(self.proj.intrinsics), self.proj.intrinsics.size, _dp(self.proj.distortion), self.proj.distortion.size,
                self.image_size[0], self.image_size[1], -1.0 if max_fov is None else float(max_fov), int(self.params.enable_depth_buffer_culling),
                pts.ctypes.data, pts.shape[0], _dp(T), idx.ctypes.data, C.byref(kept),
            )
        )
        return idx[: kept.value].copy()

    def cull(self, points, intensities, T_camera_lidar):
        """Returns (points[idx], intensities[idx]) like FrameCPU sample() (frame_cpu.cpp:281-331)."""
        idx = self.cull_indices(points, T_camera_lidar)
        return np.asarray(points)[idx], np.asarray(intensities)[idx]

    def debug_culled_points(self, points, intensities, T_camera_lidar, max_fov: float | None = None, keep_all: bool = False):
        """Test hook: the culled cloud as the solver's cost objects hold it on the device -> ((kept, 4) float64 rows
        (x, y, z, intensity) in device order, points_are_f32).  keep_all=False: the kept points grouped by 32 x 8-pixel
        tile at T_camera_lidar; keep_all=True: every point grouped the same way, those out of view last (reorder_for_pose)."""
        L = _lib.load_library()
        pts = np.asarray(points, dtype=np.float64)
        if pts.shape[1] == 3:
            pts = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1)
        pts = np.ascontiguousarray(pts)
        ins = np.ascontiguousarray(np.asarray(intensities, dtype=np.float64).reshape(-1))
        out = np.empty((max(pts.shape[0], 1), 4))
        kept, f32 = C.c_int64(), C.c_int()
        T = T_to_colmajor(T_camera_lidar)
        _lib.check(
            L.vlcal_debug_view_cull_points(
                self.device, self.proj.model_id, _dp(self.proj.intrinsics), self.proj.intrinsics.size, _dp(self.proj.distortion), self.proj.distortion.size,
                self.image_size[0], self.image_size[1], -1.0 if max_fov is None else float(max_fov), int(self.params.enable_depth_buffer_culling),
                int(bool(keep_all)), pts.ctypes.data, ins.ctypes.data, pts.shape[0], _dp(T), _dp(out), C.byref(kept), C.byref(f32),
            )
        )
        return out[: kept.value].copy(), bool(f32.value)


def generate_lidar_image(proj: GenericCamera, image_size, T_camera_lidar, points, intensities, device: int = -1):
    """vlcal::generate_lidar_image(proj, image_size=(W,H), T_camera_lidar, points) (src/vlcal/preprocess/generate_lidar_image.cpp:8-41)
    -> (intensity image float64 (H,W), point-index map int32 (H,W)); identical to the reference's images."""
    L = _lib.load_library()
    pts = np.asarray(points, dtype=np.float64)
    if pts.shape[1] == 3:
        pts = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1)
    pts = np.ascontiguousarray(pts)
    ins = np.ascontiguousarray(np.asarray(intensities, dtype=np.float64).reshape(-1))
    W, H = int(image_size[0]), int(image_size[1])
    inten = np.empty((H, W))
    index = np.empty((H, W), dtype=np.int32)
    T = T_to_colmajor(T_camera_lidar)
    _lib.check(
        L.vlcal_generate_lidar_image(
            device, proj.model_id, _dp(proj.intrinsics), proj.intrinsics.size, _dp(proj.distortion), proj.distortion.size, W, H, _dp(T),
            pts.ctypes.data, ins.ctypes.data, pts.shape[0], inten.ctypes.data, index.ctypes.data,
        )
    )
    return inten, index
