#!/usr/bin/env python
"""GPU probe of the equirectangular delta step (tools/, builder-run): runs the solves of one resident bench.py step of a
config (same inputs, culling and start poses) and prints one JSON line with the share of passes that took the delta step
and the share of point-poses deferred to the exact path, in those passes and in the others."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C2", "C3"])
    args = ap.parse_args()

    import torch

    import bench
    import direct_visual_lidar_calibration_b200 as V
    from direct_visual_lidar_calibration_b200 import calibration as VC

    torch.cuda.init()
    cfg = bench.CONFIGS[args.config]
    bag = bench.make_inputs(argparse.Namespace(config=args.config, points=None), 0)
    cam = V.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    data = V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])
    idx = V.ViewCulling(cam, (bag["width"], bag["height"]), V.ViewCullingParams(True)).cull_indices(data.points, bag["T_init"])
    cost = V.CostCalculatorNID(cam, V.VisualLiDARData(bag["image"], data.points[idx], data.intensities[idx]), V.NIDCostParams(16))
    cost.reorder_for_pose(bag["T_init"])
    n = len(idx)
    params = V.VisualCameraCalibrationParams()
    cost.reset_profile()
    for T0 in bag["starts"][: cfg["solves_per_step"]]:
        VC.estimate_pose_on_costs([cost], T0, params)
    p = cost.profile()
    plain_pp = (p["poses_total"] - p["delta_poses"]) * n
    out = {"config": args.config, "points": n, **p, "delta_pass_share": p["delta_passes"] / max(1, p["passes"]),
           "deferred_share_all": (p["deferred_plain"] + p["deferred_delta"]) / max(1, p["poses_total"] * n),
           "deferred_share_delta_passes": p["deferred_delta"] / max(1, p["delta_poses"] * n), "deferred_share_other_passes": p["deferred_plain"] / max(1, plain_pp),
           "library": V.library_path()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
