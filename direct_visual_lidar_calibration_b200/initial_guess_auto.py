"""`initial_guess_auto` on the preprocessed-dataset contract of the reference (src/initial_guess_auto.cpp).

    python -m direct_visual_lidar_calibration_b200.initial_guess_auto <data_path> [--ransac_iterations N]
        [--ransac_error_thresh PX] [--robust_kernel_width PX] [--device D]

Reads calib.json, each bag's <bag>.ply, <bag>_lidar_indices.png (from preprocess) and <bag>_matches.json (from
find_matches_superglue.py), estimates T_camera_lidar from the 2D-3D correspondences of all bags (PoseEstimation: rotation
RANSAC scored on the GPU, then a robust reprojection fit) and writes results.init_T_lidar_camera_auto back; other keys stay
as they are.  `calibrate` then starts from it.  No viewer."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

from . import create_camera
from . import io as vio
from .pose_estimation import PoseEstimation, PoseEstimationParams


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="initial_guess_auto")
    ap.add_argument("data_path", help="directory that contains preprocessed data")
    ap.add_argument("--ransac_iterations", type=int, default=8192, help="iterations for RANSAC")
    # The reference's CLI declares a default of 10.0 here, but its PoseEstimation ignores the params it is given
    # (estimate_pose.cpp:16) and always runs with 5.0: the default below is the value the reference actually uses.
    ap.add_argument("--ransac_error_thresh", type=float, default=5.0, help="reprojection error threshold [pix]")
    ap.add_argument("--robust_kernel_width", type=float, default=10.0, help="Cauchy kernel width for fine estimation [pix]")
    ap.add_argument("--device", type=int, default=-1, help="CUDA device (-1: the current one)")
    args = ap.parse_args(argv)

    if not os.path.exists(os.path.join(args.data_path, "calib.json")):
        print(f"error: failed to open {args.data_path}/calib.json", file=sys.stderr)
        return 1
    config = vio.load_calib_json(args.data_path)
    cam = config["camera"]
    proj = create_camera(cam["camera_model"], cam["intrinsics"], cam["distortion_coeffs"])
    if proj is None:
        return 1

    kp0, points = [], []
    for name in config["meta"]["bag_names"]:  # :51-55, concatenated in bag order
        cloud, _ = vio.load_ply(os.path.join(args.data_path, name + ".ply"))
        k, p = vio.read_correspondences(args.data_path, name, cloud)
        kp0.append(k)
        points.append(p)
    kp0 = np.concatenate(kp0)
    points = np.concatenate(points)

    params = PoseEstimationParams(args.ransac_iterations, args.ransac_error_thresh, args.robust_kernel_width)
    estimator = PoseEstimation(params, device=args.device)
    T_camera_lidar, _ = estimator.estimate(proj, kp0, points)
    st = estimator.stats
    print(f"num_inliers: {st['best_inliers']} / {kp0.shape[0]}")
    print(f"degenerate hypotheses: {st['degenerate']} / {st['hypotheses']}, LM iterations: {st['lm_iterations']}, final cost: {st['final_cost']:.6g}")
    print("--- T_camera_lidar ---")
    print(np.array2string(T_camera_lidar, precision=6, suppress_small=True))

    T_lidar_camera = vio.invert_isometry(T_camera_lidar)  # :127-136
    print("--- T_lidar_camera ---")
    print(np.array2string(T_lidar_camera, precision=6, suppress_small=True))
    config.setdefault("results", {})["init_T_lidar_camera_auto"] = vio.T_to_tum(T_lidar_camera)
    vio.save_calib_json(args.data_path, config)
    print(f"saved to {args.data_path}/calib.json")
    return 0


if __name__ == "__main__":
    sys.exit(main())
