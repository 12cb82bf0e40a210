#!/usr/bin/env python
"""GPU probe of the persistent kernel (tools/, builder-run): solve time per config / solver mode / kernel variant,
in-kernel %globaltimer stamps of the batch phases, pose-list throughput.  Writes JSON lines to stdout."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--modes", default="1,3")
    ap.add_argument("--stamps", action="store_true")
    ap.add_argument("--grid-poses", type=int, default=0, help="also time a pose list of this length (pose-list mode)")
    ap.add_argument("--tag", default="")
    args = ap.parse_args()

    import torch

    import direct_visual_lidar_calibration_b200 as V
    from direct_visual_lidar_calibration_b200 import calibration as VC
    from direct_visual_lidar_calibration_b200 import synthetic as S

    torch.cuda.init()
    if args.config == "C2":
        bag = S.make_bag("pinhole_1920x1080", "os1_64", 1_000_000, config_index=1)
        bag["T_init"] = S.perturb(S.gt_T_camera_lidar(), (0.5, 0.5, 0.5), (0.02, 0.02, 0.02))
    elif args.config == "C3":
        bag = S.make_bag("equirect_3840x1920", "avia", 5_000_000, config_index=2)
        bag["T_init"] = S.perturb(bag["T_gt"], (0.5, 0.5, 0.5), (0.02, 0.02, 0.02))
    elif args.config == "C3F":
        bag = S.make_bag("fisheye_1920x1080", "avia", 5_000_000, config_index=2)
        bag["T_init"] = S.perturb(bag["T_gt"], (0.5, 0.5, 0.5), (0.02, 0.02, 0.02))
    else:  # C5: the C3 cloud under the pinhole camera
        bag = S.make_bag("pinhole_1920x1080", "avia", 5_000_000, config_index=4)
        bag["T_init"] = S.perturb(bag["T_gt"], (0.5, 0.5, 0.5), (0.02, 0.02, 0.02))
    cam = V.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    W, H = bag["width"], bag["height"]
    data = V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])
    cull = V.ViewCulling(cam, (W, H), V.ViewCullingParams(True))
    idx = cull.cull_indices(data.points, bag["T_init"])
    culled = V.VisualLiDARData(bag["image"], data.points[idx], data.intensities[idx])
    cost = V.CostCalculatorNID(cam, culled, V.NIDCostParams(16))
    cost.reorder_for_pose(bag["T_init"])
    params = V.VisualCameraCalibrationParams()
    n_culled = culled.size()
    base = {"config": args.config, "points": data.size(), "culled": n_culled, "tag": args.tag, "env": {k: v for k, v in os.environ.items() if k.startswith("VLCAL_")}}

    ref = None
    for mode in [int(m) for m in args.modes.split(",")]:
        V.set_solver_mode(mode)
        for _ in range(2):
            T, r = VC.estimate_pose_on_costs([cost], bag["T_init"], params)
        cost.set_profiling(True)
        cost.reset_profile()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.reps):
            T, r = VC.estimate_pose_on_costs([cost], bag["T_init"], params)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / args.reps
        prof = cost.profile()
        cost.set_profiling(False)
        same = None
        if ref is None:
            ref = (T, r)
        else:
            same = bool(np.array_equal(T, ref[0]) and r["y"] == ref[1]["y"] and r["num_evaluations"] == ref[1]["num_evaluations"])
        line = dict(base, what="solve", mode=mode, ms_per_solve=1e3 * dt, evals=r["num_evaluations"], evals_per_s=r["num_evaluations"] / dt, batches=r["num_batches"],
                    us_per_batch=1e6 * dt / max(1, r["num_batches"]), computed=r["num_evaluations_computed"], gpp_per_s=n_culled * r["num_evaluations_computed"] / dt * 1e-9,
                    kernel_ms_per_solve=prof["kernel_ms_total"] / args.reps, passes=prof["passes"] / args.reps, launches=prof["kernel_launches"] / args.reps, y=r["y"], same_as_first_mode=same)
        print(json.dumps(line), flush=True)
    V.set_solver_mode(0)

    if args.stamps:
        V.set_solver_mode(3)
        cost.arm_solve_stamps(64)
        VC.estimate_pose_on_costs([cost], bag["T_init"], params)
        st = cost.solve_stamps(64).astype(np.int64)
        V.set_solver_mode(0)
        if len(st):
            rel = (st - st[:, :1]) * 1e-3  # us since block 0 entered the batch
            names = ["enter", "main_done", "arrived", "fin_all_arrived", "fin_published", "scores_seen", "poses_ready", "nm_stepped"]
            rows = rel[1:, :8]  # skip the 7-pose first batch
            med = {n: float(np.median(rows[:, i])) for i, n in enumerate(names)}
            nxt = (st[1:, 0] - st[:-1, 0]) * 1e-3
            print(json.dumps(dict(base, what="stamps_us_median", batches=int(len(st)), phases=med, batch_period_us=float(np.median(nxt)))), flush=True)
            bt = cost.block_times().astype(np.int64)
            if len(bt):
                t0 = bt[:, 0].min()
                rel = (bt - t0) * 1e-3
                q = lambda v: [float(np.percentile(v, p)) for p in (0, 10, 50, 90, 100)]
                print(json.dumps(dict(base, what="block_times_us_p0_p10_p50_p90_p100", blocks=int(len(bt)), enter=q(rel[:, 0]), zeroed=q(rel[:, 1]), main_done=q(rel[:, 2]), arrived=q(rel[:, 3]),
                                      main_duration=q(rel[:, 2] - rel[:, 1]))), flush=True)

    if args.grid_poses > 0:
        rng = np.random.default_rng(0)
        Ts = np.stack([S.perturb(bag["T_init"], tuple(rng.uniform(-4, 4, 3)), tuple(rng.uniform(-0.1, 0.1, 3))) for _ in range(args.grid_poses)])
        full = V.CostCalculatorNID(cam, data, V.NIDCostParams(16))
        full.reorder_for_pose(bag["T_init"])
        for c, name in ((full, "full_cloud"), (cost, "culled_cloud")):
            V.score_poses([c], Ts[:64])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = V.score_poses([c], Ts)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            n = c.data.size()
            print(json.dumps(dict(base, what="pose_list", cloud=name, n_points=n, poses=len(Ts), seconds=dt, poses_per_s=len(Ts) / dt, gpp_per_s=n * len(Ts) / dt * 1e-9, nan=int(np.isnan(out).sum()))), flush=True)
        c.set_kernel_variant(4)
        t0 = time.perf_counter()
        old = c.calculate_batch(Ts[:256])
        dt = time.perf_counter() - t0
        print(json.dumps(dict(base, what="pose_list_round1_kernel", poses=256, seconds=dt, gpp_per_s=c.data.size() * 256 / dt * 1e-9, equal=bool(np.array_equal(old, out[:256], equal_nan=True)))), flush=True)


if __name__ == "__main__":
    main()
