#!/usr/bin/env python
"""GPU probe of the equirectangular delta step (tools/, builder-run): runs the solves of one resident bench.py step of a
config (same inputs, culling and start poses) and prints one JSON line with the share of passes that took the delta step
and the share of point-poses deferred to the exact path, in those passes and in the others.

--replay DIR also replays the same solves through the batched host loop (NelderMead.optimize_batched scoring each batch
with calculate_batch, which walks the resident solve's trajectory), records every candidate batch into DIR/batches.npz
(poses [n][8][12] row-major 3x4, counts [n]) and adds to the JSON line, per anchor (pose 0, the rule of
lean_filter.cuh:lean_delta_anchor), the share of batches inside the gate.  tools/lean_deferral_host.py --batches predicts
the deferral rates of those batches on the CPU."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# lean_filter.cuh: LEAN_DELTA_MAX_DR / _DT and LEAN_DELTA_T_SCALE, as the gate compares them (fp32)
MAX_DR, MAX_DT = np.float32(4e-3), np.float32(2e-2)
T_SCALE = np.float32(4e-3 / 2e-2)


def anchor_of(rows):
    """lean_delta_anchor on rows [n][12]: the pose with the smallest largest fp32 gate entry to the others, lowest index on ties."""
    r = rows.astype(np.float32).reshape(len(rows), 3, 4)
    d = np.abs(r[:, None] - r[None, :])                     # [i][j][row][col]
    d[..., 3] *= T_SCALE
    score = d.max(axis=(1, 2, 3))
    return int(np.flatnonzero(score == score.min())[0])


def in_gate(rows, a):
    """every pose within lean_delta_pose's spread of pose a (at least two poses)"""
    if len(rows) < 2:
        return False
    q = np.abs((rows - rows[a]).astype(np.float32)).reshape(len(rows), 3, 4)
    return bool((q[..., :3] <= MAX_DR).all() and (q[..., 3] <= MAX_DT).all())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C2", "C3"])
    ap.add_argument("--replay", default=None, help="directory for batches.npz: replay the solves and report the gate per anchor")
    args = ap.parse_args()

    import torch

    import bench
    import direct_visual_lidar_calibration_b200 as V
    from direct_visual_lidar_calibration_b200 import calibration as VC
    from direct_visual_lidar_calibration_b200 import nelder_mead as NM

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
    starts = bag["starts"][: cfg["solves_per_step"]]
    cost.reset_profile()
    for T0 in starts:
        VC.estimate_pose_on_costs([cost], T0, params)
    p = cost.profile()
    plain_pp = (p["poses_total"] - p["delta_poses"]) * n
    out = {"config": args.config, "points": n, **p, "delta_pass_share": p["delta_passes"] / max(1, p["passes"]),
           "deferred_share_all": (p["deferred_plain"] + p["deferred_delta"]) / max(1, p["poses_total"] * n),
           "deferred_share_delta_passes": p["deferred_delta"] / max(1, p["delta_poses"] * n), "deferred_share_other_passes": p["deferred_plain"] / max(1, plain_pp),
           "library": V.library_path()}
    if args.replay:
        batches = []
        nm_params = NM.NelderMeadParams(init_step=params.nelder_mead_init_step, max_iterations=params.max_inner_iterations,
                                        convergence_var_thresh=params.nelder_mead_convergence_criteria)
        for T0 in starts:
            def score(X, T0=T0):
                Ts = np.stack([T0 @ VC.se3_expmap(x) for x in X])
                batches.append(np.stack([T[:3, :4].reshape(12) for T in Ts]))
                return cost.calculate_batch(Ts)

            NM.NelderMead(nm_params).optimize_batched(score, np.zeros(6))
        counts = np.array([len(b) for b in batches])
        poses = np.zeros((len(batches), 8, 12))
        for i, b in enumerate(batches):
            poses[i, : len(b)] = b
        os.makedirs(args.replay, exist_ok=True)
        np.savez(os.path.join(args.replay, "batches.npz"), poses=poses, counts=counts)
        anchors = [anchor_of(b) for b in batches]
        gate0 = np.array([in_gate(b, 0) for b in batches])
        gate_rule = np.array([in_gate(b, a) for b, a in zip(batches, anchors)])
        out["replay"] = {"batches": len(batches), "batch_sizes": {int(k): int((counts == k).sum()) for k in np.unique(counts)},
                         "in_gate_anchor_pose0": int(gate0.sum()), "in_gate_anchor_rule": int(gate_rule.sum()),
                         "refused_pose0_inside_with_rule": int((~gate0 & gate_rule).sum()), "inside_pose0_refused_with_rule": int((gate0 & ~gate_rule).sum()),
                         "anchor_index_histogram": {int(k): int(v) for k, v in zip(*np.unique(anchors, return_counts=True))}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
