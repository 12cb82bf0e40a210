#!/usr/bin/env python
"""Measure the solve axis of the persistent kernel and a whole `assess` run on the GPU.

  1. C3-sized data (synthetic.config_c3: Livox-Avia-like cloud, 3840x1920 equirectangular): S multi-start Nelder-Mead
     solves in ONE launch (vlcal_estimate_poses_nelder_mead_ctx) against the same S solves as back-to-back single-solve
     launches (vlcal_estimate_pose_nelder_mead_ctx), alternating, results compared bit for bit.
  2. The wall time of assess() on a 3-bag dataset (culling, profiles and stencils, the solves).

Prints one JSON line with the card's name and power limit beside the numbers.

    python tools/assess_probe.py [--points 5000000] [--solves 16] [--repeats 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from direct_visual_lidar_calibration_b200 import CostCalculatorNID, VisualLiDARData, create_camera  # noqa: E402
from direct_visual_lidar_calibration_b200 import assess as A  # noqa: E402
from direct_visual_lidar_calibration_b200 import calibration as VC  # noqa: E402
from direct_visual_lidar_calibration_b200 import synthetic as S  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=5_000_000)
    ap.add_argument("--solves", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--assess_points", type=int, default=1_000_000)
    args = ap.parse_args()

    bag = S.config_c3(args.points)
    cam = create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    T = bag["T_gt"]
    from direct_visual_lidar_calibration_b200.culling import ViewCulling

    pts, ins = ViewCulling(cam, (bag["width"], bag["height"])).cull(bag["points"], bag["intensities"], T)
    cost = CostCalculatorNID(cam, VisualLiDARData(bag["image"], pts, ins))
    starts = A.random_starts(T, args.solves, 0.5, 0.02, seed=0)
    params = VC.VisualCameraCalibrationParams()
    VC.estimate_poses_on_costs([cost], starts[:1], None, params)  # warm-up: module load, occupancy query
    VC.estimate_pose_on_costs([cost], starts[0], params)
    t_many, t_single = [], []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        Ts, rs = VC.estimate_poses_on_costs([cost], starts, None, params)
        t_many.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        singles = [VC.estimate_pose_on_costs([cost], s, params) for s in starts]
        t_single.append(time.perf_counter() - t0)
    # the solve-axis kernel (with its register spills) against the single-solve kernel on the same work: one solve each
    t_axis1, t_plain1 = [], []
    for _ in range(args.repeats):
        for s in starts[:4]:
            t0 = time.perf_counter()
            VC.estimate_poses_on_costs([cost], s[None], None, params)
            t_axis1.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            VC.estimate_pose_on_costs([cost], s, params)
            t_plain1.append(time.perf_counter() - t0)
    same = all(np.array_equal(r["x"], r1["x"]) and r["num_evaluations"] == r1["num_evaluations"] for r, (_, r1) in zip(rs, singles))
    iters = [r["num_iterations"] for r in rs]
    cost.close()

    bags = [S.make_bag("equirect_3840x1920", "avia", args.assess_points, config_index=2, bag_index=b) for b in range(3)]
    data = [VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    t0 = time.perf_counter()
    rep = A.assess(cam, data, ["0", "1", "2"], T, starts=args.solves)
    t_assess = time.perf_counter() - t0

    print(json.dumps({
        "card": card(),
        "c3_points": args.points, "culled_points": int(len(pts)), "solves": args.solves, "iterations": iters,
        "one_launch_s": sorted(t_many), "back_to_back_s": sorted(t_single), "speedup_median": float(np.median(t_single) / np.median(t_many)),
        "bit_identical": bool(same),
        "one_solve_axis_kernel_s_sum": float(np.sum(t_axis1)), "one_solve_plain_kernel_s_sum": float(np.sum(t_plain1)),
        "assess_3_bags_points_per_bag": args.assess_points, "assess_wall_s": t_assess, "assess_warnings": rep["warnings"],
    }))


if __name__ == "__main__":
    main()
