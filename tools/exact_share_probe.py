#!/usr/bin/env python
"""GPU probe of the exact path's share of a persistent-kernel pass (tools/, builder-run).

Runs, for each library given with --libs (VLCAL_LIB, one subprocess per library and round, alternating):
  * the solves of one resident bench.py step of the config (same inputs, culling and start poses): pass time and the
    point-poses deferred to the exact path (delta_stats: plain passes, delta passes);
  * two fixed pose lists, the same work for every library: batches of 4 poses 1e-3 apart (Nelder-Mead's initial simplex,
    the equirectangular delta step) and batches of 4 poses ~1e-2 apart (the plain classifier), 4 poses per pass.
Prints one JSON line per run and a summary line with the median pass time per library and workload, relative to the
first library.  Comparing a build whose exact drain does nothing with the normal build gives the exact path's share of a
pass; comparing two normal builds gives what a change of the error bound does to the deferral rate and the pass time."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def fixed_lists(bag, n_batches):
    from direct_visual_lidar_calibration_b200 import synthetic as S

    rng = np.random.default_rng(7)
    lists = {}
    for name, rot_deg, trans in (("delta", 0.057, 1e-3), ("plain", 0.8, 3e-2)):  # 1e-3 rad ~ 0.057 deg; 0.8 deg > the 4e-3 gate
        Ts = []
        for b in range(n_batches):
            c = bag["starts"][b % len(bag["starts"])]
            c = S.perturb(c, tuple(rng.uniform(-0.3, 0.3, 3)), tuple(rng.uniform(-0.01, 0.01, 3)))
            Ts.append(c)
            for k in range(3):
                r = np.zeros(3)
                r[k] = rot_deg
                t = np.zeros(3)
                t[k] = trans
                Ts.append(S.perturb(c, tuple(r), tuple(t)))
        lists[name] = np.stack(Ts)
    return lists


def worker(args):
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
    out = {"config": args.config, "points": n, "library": V.library_path()}

    def run(fn):
        cost.set_profiling(True)
        cost.reset_profile()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        p = cost.profile()
        cost.set_profiling(False)
        plain_pp = (p["poses_total"] - p["delta_poses"]) * n
        return {"us_per_pass": 1e3 * p["kernel_ms_total"] / max(1, p["passes"]), "passes": p["passes"], "poses": p["poses_total"], "delta_passes": p["delta_passes"],
                "wall_ms": 1e3 * wall, "deferred_plain": p["deferred_plain"], "deferred_delta": p["deferred_delta"],
                "deferred_share_plain_passes": p["deferred_plain"] / plain_pp if plain_pp else None,
                "deferred_share_delta_passes": p["deferred_delta"] / (p["delta_poses"] * n) if p["delta_poses"] else None}

    starts = bag["starts"][: cfg["solves_per_step"]]

    def solves():
        for T0 in starts:
            VC.estimate_pose_on_costs([cost], T0, params)

    solves()  # warm-up
    out["solves"] = run(solves)
    cost.set_poses_per_pass(4)
    for name, Ts in fixed_lists(bag, args.batches).items():
        cost.calculate_batch(Ts[:8])
        out[name] = run(lambda: [cost.calculate_batch(Ts) for _ in range(args.list_reps)])
    cost.set_poses_per_pass(8)
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3", choices=["C3"])
    ap.add_argument("--libs", default="", help="comma-separated libraries to compare (VLCAL_LIB); empty: the in-tree build only")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=64, help="4-pose batches per fixed pose list")
    ap.add_argument("--list-reps", type=int, default=4)
    ap.add_argument("--worker", action="store_true")
    args = ap.parse_args()
    if args.worker:
        worker(args)
        return
    libs = [l for l in args.libs.split(",") if l] or [""]
    runs = {l: [] for l in libs}
    for r in range(args.rounds):
        for lib in libs:
            env = dict(os.environ)
            if lib:
                env["VLCAL_LIB"] = os.path.abspath(lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--config", args.config, "--batches", str(args.batches), "--list-reps", str(args.list_reps)]
            res = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True)
            line = res.stdout.strip().splitlines()[-1]
            print(line, flush=True)
            runs[lib].append(json.loads(line))
    summary = {}
    for w in ("solves", "delta", "plain"):
        med = {lib: float(np.median([o[w]["us_per_pass"] for o in runs[lib]])) for lib in libs}
        base = med[libs[0]]
        summary[w] = {os.path.basename(lib) or "in-tree": {"us_per_pass_median": med[lib], "spread": [min(o[w]["us_per_pass"] for o in runs[lib]), max(o[w]["us_per_pass"] for o in runs[lib])],
                                                           "saving_vs_first": 1.0 - med[lib] / base,
                                                           "deferred_share_plain_passes": runs[lib][-1][w]["deferred_share_plain_passes"],
                                                           "deferred_share_delta_passes": runs[lib][-1][w]["deferred_share_delta_passes"]} for lib in libs}
    print(json.dumps({"summary": summary}), flush=True)


if __name__ == "__main__":
    main()
