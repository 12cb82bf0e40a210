"""GPU-native (H100) NID LiDAR-camera registration engine (hot path of koide3/direct_visual_lidar_calibration).

The compute lives in ``libvlcal_nid.so`` (hand-written sm_90a CUDA behind the C ABI of ``include/vlcal_nid.h``);
this package is the thin host-side mirror of the reference's interface for that path:

  create_camera                 <- camera::create_camera             (src/camera/create_camera.cpp:34-50)
  VisualLiDARData               <- vlcal::VisualLiDARData            (include/vlcal/common/visual_lidar_data.hpp)
  NIDCostParams, CostCalculatorNID <- vlcal::CostCalculatorNID       (include/vlcal/calib/cost_calculator_nid.hpp)
  NIDCost                       <- vlcal::NIDCost (value only)        (include/vlcal/costs/nid_cost.hpp)
  ViewCullingParams, ViewCulling   <- vlcal::ViewCulling             (include/vlcal/calib/view_culling.hpp)
  NelderMead                    <- dfo::NelderMead<N>                (include/dfo/nelder_mead.hpp)
  VisualCameraCalibrationParams, VisualCameraCalibration <- vlcal::VisualCameraCalibration
                                                                     (include/vlcal/calib/visual_camera_calibration.hpp)
  PoseEstimationParams, PoseEstimation <- vlcal::PoseEstimation      (include/vlcal/common/estimate_pose.hpp)
  PointsColorUpdater            <- vlcal::PointsColorUpdater         (include/vlcal/common/points_color_updater.hpp)

There is no CPU fallback: without the built library or without a CUDA device every compute call raises.
"""
from ._lib import VlcalError, build_library, device_count, library_path, load_library, set_solver_mode
from .camera import GenericCamera, create_camera
from .cost import CostCalculatorNID, NIDCost, NIDCostParams, VisualLiDARData, score_poses
from .culling import ViewCulling, ViewCullingParams, generate_lidar_image
from .nelder_mead import NelderMead, NelderMeadParams
from . import bfgs
from .calibration import RegistrationType, VisualCameraCalibration, VisualCameraCalibrationParams, estimate_camera_fov, se3_expmap
from .pose_estimation import PoseEstimation, PoseEstimationParams
from .points_color_updater import PointsColorUpdater, render_overlay, turbo_colormap

__all__ = [
    "score_poses",
    "generate_lidar_image",
    "VlcalError", "build_library", "device_count", "library_path", "load_library", "set_solver_mode",
    "GenericCamera", "create_camera",
    "CostCalculatorNID", "NIDCost", "NIDCostParams", "VisualLiDARData",
    "ViewCulling", "ViewCullingParams",
    "NelderMead", "NelderMeadParams",
    "RegistrationType", "VisualCameraCalibration", "VisualCameraCalibrationParams", "estimate_camera_fov", "se3_expmap",
    "PoseEstimation", "PoseEstimationParams",
    "PointsColorUpdater", "render_overlay", "turbo_colormap",
]
