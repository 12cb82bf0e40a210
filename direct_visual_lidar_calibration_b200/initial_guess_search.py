"""`initial_guess_search`: an initial guess without 2D-3D matches, from a coarse-to-fine NID search over SE(3).

    python -m direct_visual_lidar_calibration_b200.initial_guess_search <data_path> [--prior x y z qx qy qz qw]
        [--rot_range_deg 180] [--rot_step_deg 3] [--trans_range 0.3] [--keep 64] [--nid_bins 16] [--first_n_bags N]
        [--seed 0] [--device D]

Reads calib.json and each bag's <bag>.png / <bag>.ply (from preprocess).  Level 0 scores a near-uniform cover of SO(3)
(or of the rotations within --rot_range_deg of --prior) on the image at 1/8 and 16 384 points per bag; the best --keep
poses after non-maximum suppression are refined level by level -- half the step, a 3x3x3 rotation grid x a translation
grid around every candidate, the next finer image and four times the points -- down to a step of <= 0.25 deg on the
full-resolution image.  Every score is the sum over the bags of CostCalculatorNID::calculate, computed by the pose sweep
kernel (vlcal_nid_sweep_search_set).  Writes results.init_T_lidar_camera_auto into calib.json (the key `calibrate` reads;
other keys stay as they are) and a report to <data_path>/initial_guess_search.json.  No viewer."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

from . import initial_guess as ig
from . import io as vio

LEVEL0_SCALE = 8          # image scale of level 0; halves per level down to 1
LEVEL0_POINTS = 16384     # points per bag at level 0; x4 per level, capped at the cloud
FINAL_STEP_DEG = 0.25     # the search stops at the first full-resolution level whose step is <= this
NMS_FACTOR = 1.5          # no two kept poses within NMS_FACTOR x step of each other
BASIN_FACTOR = 3.0        # a pose farther than BASIN_FACTOR x level-0 step from the winner belongs to another basin
MARGIN_WARN = 0.005       # warn below this NID margin between the winner and the best other basin
MIN_KEEP = 8
# A pose that sees next to nothing has a near-empty joint histogram and an NID near 0 -- below any real alignment.  Poses
# that count fewer points than this share of the level's best-covered pose are set aside (scored NaN: they rank last).
MIN_OVERLAP = 0.25


def level_schedule(rot_step_deg: float, trans_range: float, keep: int) -> list:
    """Per level: image scale, points per bag, rotation step, translation grid, candidates kept afterwards."""
    levels = [{"index": 0, "scale": LEVEL0_SCALE, "points": LEVEL0_POINTS, "step_deg": float(rot_step_deg), "trans_spacing": 0.0, "trans_half_steps": 0, "keep": keep}]
    while True:
        prev = levels[-1]
        i = prev["index"] + 1
        # level 1 covers the whole +-trans_range box at half-range spacing (5x5x5); later levels only the 3x3x3
        # neighbourhood of each candidate at half the previous spacing, so the pose count does not grow with depth
        spacing, half = (trans_range / 2.0, 2) if i == 1 else (prev["trans_spacing"] / 2.0, 1)
        lv = {"index": i, "scale": max(1, LEVEL0_SCALE >> i), "points": LEVEL0_POINTS * 4**i, "step_deg": prev["step_deg"] / 2.0, "trans_spacing": spacing,
              "trans_half_steps": half, "keep": max(MIN_KEEP, keep >> i)}
        levels.append(lv)
        if lv["scale"] == 1 and lv["step_deg"] <= FINAL_STEP_DEG:
            return levels


def run_search(score, rot_step_deg: float = 3.0, prior_T_lidar_camera=None, rot_range_deg: float = 180.0, trans_range: float = 0.3, keep: int = 64, log=print) -> dict:
    """The coarse-to-fine search.  score(level, search_set) -> (scores[n_poses], inliers[n_poses], kernel_ms) scores one level's poses (the
    GPU sweep in the tool; tests inject a callable).  Returns the report: levels, the candidates kept per level, the final
    top 5, the margin to the best other basin and the winner as T_camera_lidar."""
    levels = level_schedule(rot_step_deg, trans_range, keep)
    report = {"levels": [], "candidates": []}
    candidates = None
    basin_deg = BASIN_FACTOR * rot_step_deg
    level0 = None
    for lv in levels:
        if lv["index"] == 0:
            sset = ig.rotation_set(lv["step_deg"], prior_T_lidar_camera, rot_range_deg)
        else:
            sset = ig.local_set(candidates, lv["step_deg"], lv["trans_spacing"], lv["trans_half_steps"])
        t0 = time.perf_counter()
        scores, inliers, kernel_ms = score(lv, sset)
        wall_ms = (time.perf_counter() - t0) * 1e3
        scores, inliers = np.asarray(scores, dtype=np.float64), np.asarray(inliers, dtype=np.int64)
        if scores.shape != (sset.n_poses,) or inliers.shape != (sset.n_poses,):
            raise ValueError("the scorer must return one score and one inlier count per pose")
        # ranked at a resolution of 1e-12: histograms that are permutations of each other have the same NID up to the
        # order of the sums, and such ties are to break by list order, not by the last bits of whoever did the scoring
        scores = np.round(np.where(inliers < MIN_OVERLAP * inliers.max(), np.nan, scores), 12)
        kept = ig.nms_top_k(sset.poses, scores, lv["keep"], NMS_FACTOR * lv["step_deg"])
        if kept.size == 0 or np.isnan(scores[kept[0]]):
            raise RuntimeError(f"level {lv['index']}: no pose of the search set sees any point of the cloud")
        kept = kept[~np.isnan(scores[kept])]
        candidates = sset.poses(kept)
        cand_scores = scores[kept]
        if level0 is None:
            level0 = (sset, scores)
        report["levels"].append({"level": lv["index"], "scale": lv["scale"], "points_per_bag": lv["points"], "step_deg": lv["step_deg"], "trans_spacing": lv["trans_spacing"],
                                 "poses": int(sset.n_poses), "kernel_ms": float(kernel_ms), "wall_ms": wall_ms, "kept": int(kept.size),
                                 "best_nid": [float(v) for v in cand_scores[:5]]})
        report["candidates"].append({"poses": candidates, "nid": cand_scores})
        log(f"level {lv['index']}: 1/{lv['scale']} image, step {lv['step_deg']:g} deg, {sset.n_poses} poses, kernel {kernel_ms:.1f} ms, best NID {cand_scores[0]:.6f}")
    report["T_camera_lidar"] = candidates[0]
    report["top"] = [{"T_lidar_camera": vio.T_to_tum(vio.invert_isometry(T)), "nid": float(s)} for T, s in zip(candidates[:5], cand_scores[:5])]
    # margin: on the coarsest level, where every basin was scored, the best pose of another basin (farther than basin_deg
    # from the winner) against the best pose of the winner's own
    sset, scores = level0
    own, other = np.inf, np.inf
    for s0 in range(0, sset.n_poses, 1 << 16):
        which = np.arange(s0, min(sset.n_poses, s0 + (1 << 16)))
        sc = np.where(np.isnan(scores[which]), np.inf, scores[which])
        away = ig.rotation_angle_deg(sset.poses(which)[:, :3, :3], candidates[0, :3, :3]) > basin_deg
        own, other = min(own, sc[~away].min(initial=np.inf)), min(other, sc[away].min(initial=np.inf))
    report["margin"] = float(other - own) if np.isfinite(own) and np.isfinite(other) else None
    return report


class SweepScorer:
    """score(level, search_set) on the GPU: one CostCalculatorNID per (bag, level) over the level's image, camera and
    cloud subset, built on first use, and the pose sweep over all bags."""

    def __init__(self, camera_model: str, intrinsics, distortion, dataset, nid_bins: int = 16, seed: int = 0, device: int = -1):
        self.camera_model, self.intrinsics, self.distortion = camera_model, list(intrinsics), list(distortion)
        self.dataset, self.bins, self.seed, self.device = dataset, nid_bins, seed, device
        self._costs = {}

    def costs(self, level: dict) -> list:
        from . import CostCalculatorNID, NIDCostParams, VisualLiDARData, create_camera

        key = (level["scale"], level["points"])
        if key not in self._costs:
            proj = create_camera(self.camera_model, ig.pyramid_intrinsics(self.camera_model, self.intrinsics, level["scale"]), self.distortion)
            costs = []
            for b, data in enumerate(self.dataset):
                sub = np.sort(ig.cloud_subset(data.size(), level["points"], self.seed + b))
                image = ig.pyramid_image(data.image, level["scale"])
                costs.append(CostCalculatorNID(proj, VisualLiDARData(image, data.points[sub], data.intensities[sub]), NIDCostParams(self.bins), device=self.device))
            self._costs[key] = costs
        return self._costs[key]

    def __call__(self, level: dict, sset: ig.SearchSet):
        return ig.sweep_search_set(self.costs(level), sset)

    def close(self):
        for costs in self._costs.values():
            for c in costs:
                c.close()
        self._costs = {}


def write_results(data_path: str, config: dict, report: dict) -> None:
    config.setdefault("results", {})["init_T_lidar_camera_auto"] = vio.T_to_tum(vio.invert_isometry(report["T_camera_lidar"]))
    vio.save_calib_json(data_path, config)
    out = {"levels": report["levels"], "top": report["top"], "margin": report["margin"]}
    with open(os.path.join(data_path, "initial_guess_search.json"), "w") as f:
        f.write(json.dumps(out, indent=2) + "\n")


def main(argv=None, score=None) -> int:
    """score: a replacement for the GPU scorer (tests); see run_search."""
    ap = argparse.ArgumentParser(prog="initial_guess_search")
    ap.add_argument("data_path", help="directory that contains preprocessed data")
    ap.add_argument("--prior", type=float, nargs=7, default=None, metavar=("x", "y", "z", "qx", "qy", "qz", "qw"), help="rough T_lidar_camera (TUM order)")
    ap.add_argument("--rot_range_deg", type=float, default=180.0, help="search only rotations within this angle of the prior")
    ap.add_argument("--rot_step_deg", type=float, default=3.0, help="rotation step of the coarsest level [deg]")
    ap.add_argument("--trans_range", type=float, default=0.3, help="half-width of the searched box of camera positions [m]")
    ap.add_argument("--keep", type=int, default=64, help="candidates kept after the coarsest level")
    ap.add_argument("--nid_bins", type=int, default=16, help="Number of histogram bins for NID")
    ap.add_argument("--first_n_bags", type=int, default=None, help="use only the first N bags")
    ap.add_argument("--seed", type=int, default=0, help="seed of the cloud subsets")
    ap.add_argument("--device", type=int, default=-1, help="CUDA device (-1: the current one)")
    args = ap.parse_args(argv)

    def refuse(msg: str) -> int:
        print(f"error: {msg}", file=sys.stderr)
        return 1

    if not os.path.exists(os.path.join(args.data_path, "calib.json")):
        return refuse(f"failed to open {args.data_path}/calib.json")
    if not (args.rot_step_deg > 0.0 and args.rot_range_deg > 0.0 and args.trans_range > 0.0):
        return refuse("--rot_step_deg, --rot_range_deg and --trans_range must be positive")
    if args.rot_step_deg > 10.0:
        return refuse("--rot_step_deg above 10 deg leaves gaps no NID basin covers")
    if args.keep < 1 or args.nid_bins < 2 or (args.first_n_bags is not None and args.first_n_bags < 1):
        return refuse("--keep and --first_n_bags must be at least 1, --nid_bins at least 2")
    prior = None
    if args.prior is not None:
        qn = float(np.linalg.norm(args.prior[3:]))
        if not np.all(np.isfinite(args.prior)) or abs(qn - 1.0) > 1e-3:
            return refuse(f"--prior: the quaternion is not of unit length (norm {qn:g})")
        prior = vio.tum_to_T(args.prior)
    elif args.rot_range_deg < 180.0:
        return refuse("--rot_range_deg needs --prior")

    config = vio.load_calib_json(args.data_path)
    cam = config["camera"]
    from . import create_camera

    if create_camera(cam["camera_model"], cam["intrinsics"], cam["distortion_coeffs"]) is None:
        return 1
    bag_names = list(config["meta"]["bag_names"])
    if args.first_n_bags is not None:
        bag_names = bag_names[: args.first_n_bags]
        print(f"use only the first {args.first_n_bags} bags")
    scorer = None
    if score is None:
        dataset = []
        for name in bag_names:
            print(f"loading {args.data_path}/{name}.(png|ply)")
            dataset.append(vio.load_visual_lidar_data(args.data_path, name))
        scorer = score = SweepScorer(cam["camera_model"], cam["intrinsics"], cam["distortion_coeffs"], dataset, args.nid_bins, args.seed, args.device)
    try:
        report = run_search(score, args.rot_step_deg, prior, args.rot_range_deg, args.trans_range, args.keep)
    finally:
        if scorer is not None:
            scorer.close()
    if report["margin"] is None:
        print("margin: the coarsest level scored no pose outside the winner's basin")
    else:
        print(f"margin to the best other basin on the coarsest level: {report['margin']:.6f}")
        if report["margin"] < MARGIN_WARN:
            print("warning: another basin scores almost as well as the winner -- the scene may be ambiguous (symmetric room, too little texture); pass --prior", file=sys.stderr)
    T_lidar_camera = vio.invert_isometry(report["T_camera_lidar"])
    print("--- T_lidar_camera ---")
    print(np.array2string(T_lidar_camera, precision=6, suppress_small=True))
    write_results(args.data_path, config, report)
    print(f"saved to {args.data_path}/calib.json")
    return 0


if __name__ == "__main__":
    sys.exit(main())
