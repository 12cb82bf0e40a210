"""vlcal::PointsColorUpdater mirror (reference: include/vlcal/common/points_color_updater.hpp,
src/vlcal/common/points_color_updater.cpp) and the LiDAR overlay of the headless viewer (csrc/viewer.cu)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .camera import GenericCamera, _dp
from .cost import T_to_colmajor, VisualLiDARData


def turbo_colormap() -> np.ndarray:
    """The 256 x 3 uint8 RGB Turbo table the kernels colour intensities with (the published table; needs no device)."""
    table = np.empty((256, 3), dtype=np.uint8)
    _lib.check(_lib.load_library().vlcal_turbo_colormap(table.ctypes.data))
    return table


def _viewer_args(proj: GenericCamera, data: VisualLiDARData, T_camera_lidar, device: int):
    h, w = data.image.shape
    T = T_to_colmajor(T_camera_lidar)
    return [device, proj.model_id, _dp(proj.intrinsics), proj.intrinsics.size, _dp(proj.distortion), proj.distortion.size, w, h, data.image.ctypes.data, data.image.strides[0],
            _dp(T), data.points.ctypes.data, data.intensities.ctypes.data, data.size()]


class PointsColorUpdater:
    """vlcal::PointsColorUpdater(proj, image, points) (points_color_updater.hpp) with the points' intensities passed
    beside them: update(T_camera_lidar, blend_weight) -> (N, 4) float32 RGBA, gray * w + turbo(intensity) * (1 - w) with
    alpha 1 for a point that projects into the image inside the viewer's field of view, zeros for any other."""

    def __init__(self, proj: GenericCamera, image, points, intensities, device: int = -1):
        self.proj = proj
        self.data = VisualLiDARData(image, points, intensities)
        self.device = device
        self.kernel_ms = 0.0  # of the last update()

    def update(self, T_camera_lidar, blend_weight: float) -> np.ndarray:
        colors = np.empty((self.data.size(), 4), dtype=np.float32)
        ms = C.c_double()
        args = _viewer_args(self.proj, self.data, T_camera_lidar, self.device)
        _lib.check(_lib.load_library().vlcal_colorize_points(*args, float(np.float32(blend_weight)), colors.ctypes.data, C.byref(ms)))
        self.kernel_ms = ms.value
        return colors


def render_overlay(proj: GenericCamera, image, T_camera_lidar, points, intensities, point_radius: int = 1, blend_weight: float = 0.7, device: int = -1, return_kernel_ms: bool = False):
    """The cloud drawn into the camera image -> (BGR uint8 (H, W, 3), winning point index per pixel int32 (H, W), -1 where
    none).  Per pixel the nearest of the points whose (2 point_radius + 1)^2 square covers it wins, of equal squared
    ranges the last index (the rules and the field of view of generate_lidar_image, whose index map point_radius 0
    returns); a covered pixel is turbo(intensity) * (1 - w) + gray * w, an uncovered one stays gray."""
    data = VisualLiDARData(image, points, intensities)
    h, w = data.image.shape
    bgr = np.empty((h, w, 3), dtype=np.uint8)
    index = np.empty((h, w), dtype=np.int32)
    ms = C.c_double()
    args = _viewer_args(proj, data, T_camera_lidar, device)
    _lib.check(_lib.load_library().vlcal_render_overlay(*args, int(point_radius), float(np.float32(blend_weight)), bgr.ctypes.data, index.ctypes.data, C.byref(ms)))
    return (bgr, index, ms.value) if return_kernel_ms else (bgr, index)


def agreement_map(proj: GenericCamera, image, T_camera_lidar, points, intensities, bins: int = 16, point_radius: int = 1, blend_weight: float = 0.7, device: int = -1):
    """Where the LiDAR and the camera disagree at T_camera_lidar -> (pointwise mutual information per point (N,) float64,
    NaN where the NID histogram does not count the point; joint histogram (bins, bins) [image_bin, lidar_bin] int32, as
    CostCalculatorNID.calculate_batch returns it; BGR uint8 (H, W, 3); winning point per pixel int32 (H, W)).  The image is
    the overlay of render_overlay with turbo(0.5 + PMI / 4) in place of turbo(intensity)."""
    data = VisualLiDARData(image, points, intensities)
    h, w = data.image.shape
    pmi = np.empty(data.size())
    hist = np.empty(bins * bins, dtype=np.int32)
    bgr = np.empty((h, w, 3), dtype=np.uint8)
    index = np.empty((h, w), dtype=np.int32)
    args = _viewer_args(proj, data, T_camera_lidar, device)
    _lib.check(_lib.load_library().vlcal_agreement_map(*args, int(bins), int(point_radius), float(np.float32(blend_weight)), _dp(pmi), hist.ctypes.data, bgr.ctypes.data, index.ctypes.data))
    return pmi, hist.reshape(bins, bins).T.copy(), bgr, index
