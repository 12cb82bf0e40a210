"""`viewer` without a window: what the reference's viewer shows (src/viewer.cpp), written to files.

    python -m direct_visual_lidar_calibration_b200.viewer <data_path> [--dst_path DIR] [--transformation auto|manual|result]
           [--blend_weight 0.7] [--point_radius 1] [--first_n_bags N] [--device D]

Reads <data_path>/calib.json (+ <bag>.png / <bag>.ply) and writes to DIR (default <data_path>; calib.json is only read):

  <bag>_colored.ply    the cloud coloured with the camera image through the selected pose: PointsColorUpdater::update
                       (points_color_updater.cpp:37-61) on the GPU, as uchar red green blue alpha after intensity
  <bag>_overlay.png    the cloud drawn into the camera image with hidden points removed (the z-buffer of
                       generate_lidar_image with a point radius): image edges should meet range and intensity edges
  viewer_report.json   the NID of CostCalculatorNID::calculate (full cloud, 16 bins) of every transformation calib.json
                       holds, per bag and summed, and the inlier count of the selected one -- "did calibrate improve on
                       the initial guess, on every bag?" as numbers

Transformations are found as viewer.cpp:49-83 finds them; the last one found is selected unless --transformation names
another.  The interactive window, the 3-D view and the icosphere (draw_sphere = false in viewer.cpp:95) have no
counterpart here."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

from . import io as vio
from .camera import create_camera
from .cost import CostCalculatorNID, NIDCostParams, score_poses
from .points_color_updater import PointsColorUpdater, render_overlay

# results key, label (viewer.cpp:49-74, in that order), --transformation name
TRANSFORMATIONS = [
    ("init_T_lidar_camera_auto", "INIT_GUESS (AUTO)", "auto"),
    ("init_T_lidar_camera", "INIT_GUESS (MANUAL)", "manual"),
    ("T_lidar_camera", "CALIBRATION_RESULT", "result"),
]


def _tum2pose(values) -> np.ndarray:
    """tum2pose of viewer.cpp:42-47: Eigen::Quaterniond(w, x, y, z).toRotationMatrix() as stored, not normalised."""
    x, y, z, w = (float(v) for v in values[3:7])
    T = np.eye(4)
    T[:3, :3] = [
        [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)],
    ]
    T[:3, 3] = values[0:3]
    return T


def find_transformations(config: dict, select: str | None = None):
    """viewer.cpp:49-83 -> (labels, T_lidar_camera (K, 4, 4), index of the selected one): every transformation calib.json
    holds, in the reference's order; the last one is selected unless `select` (auto / manual / result) names another that
    was found (ValueError if it was not).  None found: the reference's error line, identity under the label NONE."""
    results = config.get("results", {})
    labels, poses, names = [], [], []
    for key, label, name in TRANSFORMATIONS:
        if key in results:
            labels.append(label)
            poses.append(_tum2pose(results[key]))
            names.append(name)
    if not labels:
        print("error: no transformation found in calib.json!!", file=sys.stderr)
        labels, poses, names = ["NONE"], [np.eye(4)], [None]
    selected = len(labels) - 1
    if select is not None:
        if select not in names:
            raise ValueError(f"calib.json holds no {select} transformation (found: {', '.join(labels)})")
        selected = names.index(select)
    return labels, np.stack(poses), selected


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="viewer")
    ap.add_argument("data_path", help="directory that contains preprocessed data")
    ap.add_argument("--dst_path", default=None, help="directory the files are written to (default: data_path)")
    ap.add_argument("--transformation", choices=[t[2] for t in TRANSFORMATIONS], default=None, help="the transformation to look through (default: the last one found)")
    ap.add_argument("--blend_weight", type=float, default=0.7, help="weight of the camera image in the colours, 0 to 1")
    ap.add_argument("--point_radius", type=int, default=1, help="a point covers (2r+1)^2 pixels of the overlay, 0 to 8")
    ap.add_argument("--first_n_bags", type=int, default=None, help="use only the first N bags")
    ap.add_argument("--device", type=int, default=-1)
    args = ap.parse_args(argv)

    try:
        config = vio.load_calib_json(args.data_path)
    except OSError:
        print(f"error: failed to open {args.data_path}/calib.json", file=sys.stderr)  # viewer.cpp:19-22 (which aborts)
        return 1
    try:
        labels, T_lidar_camera, selected = find_transformations(config, args.transformation)
    except ValueError as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    if not 0.0 <= args.blend_weight <= 1.0 or not 0 <= args.point_radius <= 8:
        print("error: --blend_weight must be in [0, 1] and --point_radius in [0, 8]", file=sys.stderr)
        return 1
    cam = config["camera"]
    proj = create_camera(cam["camera_model"], cam["intrinsics"], cam["distortion_coeffs"])
    if proj is None:
        return 1
    bag_names = list(config["meta"]["bag_names"])
    if args.first_n_bags is not None:
        bag_names = bag_names[: args.first_n_bags]
    dst = args.dst_path or args.data_path
    os.makedirs(dst, exist_ok=True)
    T_camera_lidar = np.stack([vio.invert_isometry(T) for T in T_lidar_camera])  # viewer.cpp:96
    print(f"selected transformation: {labels[selected]}")

    import cv2

    nid = np.empty((len(bag_names), len(labels)))
    inliers = []
    for b, name in enumerate(bag_names):
        print(f"loading {args.data_path}/{name}.(png|ply)")
        data = vio.load_visual_lidar_data(args.data_path, name)
        colors = PointsColorUpdater(proj, data.image, data.points, data.intensities, args.device).update(T_camera_lidar[selected], args.blend_weight)
        vio.save_ply_binary(os.path.join(dst, name + "_colored.ply"), data.points[:, :3], data.intensities, colors=colors)
        bgr, _ = render_overlay(proj, data.image, T_camera_lidar[selected], data.points, data.intensities, args.point_radius, args.blend_weight, args.device)
        if not cv2.imwrite(os.path.join(dst, name + "_overlay.png"), bgr):
            raise OSError(f"failed to write {name}_overlay.png")
        cost = CostCalculatorNID(proj, data, NIDCostParams(16), device=args.device)
        nid[b] = score_poses([cost], T_camera_lidar)
        _, hist = cost.calculate_batch(T_camera_lidar[selected : selected + 1], return_hist=True)
        inliers.append(int(hist.sum()))
        cost.close()

    width = max(len(n) for n in bag_names + ["sum"])
    print(" " * width + "".join(f"  {lab:>20s}" for lab in labels))
    for name, row in zip(bag_names + ["sum"], list(nid) + [nid.sum(axis=0)]):
        print(f"{name:<{width}s}" + "".join(f"  {v:20.12f}" for v in row))

    def numbers(a):
        return [None if np.isnan(v) else float(v) for v in a]  # NaN: no point of the bag is in view at that pose

    report = {
        "labels": labels,
        "T_lidar_camera": [[float(v) for v in config["results"][key]] for key, label, _ in TRANSFORMATIONS if label in labels] or [vio.T_to_tum(np.eye(4))],
        "selected": labels[selected],
        "bag_names": bag_names,
        "nid": [numbers(row) for row in nid],
        "nid_sum": numbers(nid.sum(axis=0)),
        "selected_inliers": inliers,
        "blend_weight": float(np.float32(args.blend_weight)),
        "point_radius": args.point_radius,
    }
    with open(os.path.join(dst, "viewer_report.json"), "w") as f:
        f.write(json.dumps(report, indent=2) + "\n")
    print(f"saved to {dst}/(<bag>_colored.ply|<bag>_overlay.png|viewer_report.json)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
