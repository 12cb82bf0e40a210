"""`assess`: how well is a calibration constrained?  The NID objective around the calibrated pose, on the GPU.

    python -m direct_visual_lidar_calibration_b200.assess <data_path> [--dst_path DIR] [--transformation auto|manual|result]
           [--first_n_bags N] [--nid_bins 16] [--starts 16] [--start_rot_deg 1.0] [--start_trans 0.05] [--profile_steps 41]
           [--disable_culling] [--seed 0] [--device -1]

Reads <data_path>/calib.json (+ <bag>.png / <bag>.ply) as `viewer` does and selects the transformation the same way (the
last one found unless --transformation names another).  Every bag is view-culled once at that pose T, as `calibrate`
culls at the start of an outer iteration; everything below runs on those culled points.  Writes assessment.json and
<bag>_agreement.png to DIR (default <data_path>; nothing else is changed):

  local     per bag and summed over the bags: 1-D profiles of NID along each tangent axis (T * Exp(s e_k), the
            parameterisation of calibrate's Nelder-Mead solve: rotations +-2 deg, translations +-10 cm), the 6x6
            central-difference Hessian at a step of 0.05 deg / 2.5 mm and at twice that step, its eigen-decomposition, and
            per axis the curvature and the width over which NID stays within RISE of its value at T.  All poses of a bag
            are scored in one persistent-kernel launch.
  solves    --starts Nelder-Mead solves from T perturbed by seeded random rotations of --start_rot_deg and translations
            of --start_trans, plus one leave-one-bag-out solve per bag (two bags or more), all in ONE launch of the
            persistent kernel's solve axis (vlcal_estimate_poses_nelder_mead_ctx); each solve is the solve `calibrate`'s
            inner loop would run from its start over its bags.
  warnings  axes whose curvature is below WEAK_RATIO of the largest of their kind (rotations are compared with
            rotations, translations with translations: the two are in different units), axes whose two Hessian steps
            disagree by more than 2x (NID counts whole pixels, so it is piecewise constant in the pose and a finite
            difference below the quantisation means nothing), starts that found a lower NID away from T (a better
            optimum the calibration missed), and outlier bags (three bags or more: leaving the bag out moves the
            optimum more than OUTLIER_FACTOR x the median over the bags, and beyond the solve tolerance).
  <bag>_agreement.png
            per bag, the pointwise mutual information log(p(a,b) / (p(a) p(b))) of every culled point's joint bin in
            the NID histogram at T, drawn through K5's z-buffer over the camera image (turbo: red where the bin pair is
            more frequent than chance, blue where it is rarer; agreement_map, csrc/agreement.cu)."""
from __future__ import annotations

import argparse
import copy
import json
import math
import os
import sys

import numpy as np

from . import io as vio
from .calibration import VisualCameraCalibrationParams, estimate_poses_on_costs, se3_expmap
from .camera import create_camera
from .cost import CostCalculatorNID, NIDCostParams, VisualLiDARData, score_poses
from .culling import ViewCulling, ViewCullingParams
from .points_color_updater import agreement_map
from .viewer import TRANSFORMATIONS, find_transformations

AXES = ["rx", "ry", "rz", "tx", "ty", "tz"]  # tangent coordinates (omega, v) of gtsam's Pose3::Expmap
PROFILE_HALF = np.array([math.radians(2.0)] * 3 + [0.10] * 3)  # profile half-ranges: +-2 deg, +-10 cm
HESSIAN_STEP = np.array([math.radians(0.05)] * 3 + [0.0025] * 3)  # central-difference step: 0.05 deg, 2.5 mm
RISE = 1e-3  # NID rise that bounds an axis' width
WEAK_RATIO = 0.1  # an axis is weak below this fraction of the largest curvature of its kind
STEP_DISAGREEMENT = 2.0  # the curvatures at step h and 2h differ by more than this factor
AWAY_ROT_DEG, AWAY_TRANS = 0.1, 0.005  # a solve "ended away from T" beyond either
OUTLIER_FACTOR = 3.0
MAX_SOLVES = 64  # the persistent kernel's solve axis


def tangent_poses(T: np.ndarray, xs) -> np.ndarray:
    """T * Exp(x) for every row x = (omega, v): the poses calibrate's Nelder-Mead solve visits from init T (init_T * Expmap(x))."""
    xs = np.asarray(xs, dtype=np.float64).reshape(-1, 6)
    return np.stack([T @ se3_expmap(x) for x in xs]) if len(xs) else np.empty((0, 4, 4))


def profile_offsets(steps: int) -> np.ndarray:
    """(6, steps, 6) tangent offsets: row k holds s * e_k for s evenly spaced over +-PROFILE_HALF[k] (steps odd: s = 0 included)."""
    s = np.linspace(-1.0, 1.0, steps)
    out = np.zeros((6, steps, 6))
    for k in range(6):
        out[k, :, k] = s * PROFILE_HALF[k]
    return out


def hessian_stencil(h) -> np.ndarray:
    """(73, 6) offsets of the central-difference stencil for a full 6x6 Hessian with per-axis steps h: the centre, +-h_i e_i
    (12), and (+-h_i e_i) + (+-h_j e_j) for i < j (4 x 15), in that order."""
    h = np.asarray(h, dtype=np.float64)
    rows = [np.zeros(6)]
    for i in range(6):
        for sgn in (1.0, -1.0):
            x = np.zeros(6)
            x[i] = sgn * h[i]
            rows.append(x)
    for i in range(6):
        for j in range(i + 1, 6):
            for si, sj in ((1.0, 1.0), (1.0, -1.0), (-1.0, 1.0), (-1.0, -1.0)):
                x = np.zeros(6)
                x[i], x[j] = si * h[i], sj * h[j]
                rows.append(x)
    return np.stack(rows)


def hessian_from_stencil(f, h) -> np.ndarray:
    """The 6x6 central-difference Hessian from the values f of hessian_stencil(h)."""
    f = np.asarray(f, dtype=np.float64)
    h = np.asarray(h, dtype=np.float64)
    H = np.zeros((6, 6))
    f0 = f[0]
    for i in range(6):
        H[i, i] = (f[1 + 2 * i] - 2.0 * f0 + f[2 + 2 * i]) / (h[i] * h[i])
    k = 13
    for i in range(6):
        for j in range(i + 1, 6):
            fpp, fpm, fmp, fmm = f[k : k + 4]
            H[i, j] = H[j, i] = (fpp - fpm - fmp + fmm) / (4.0 * h[i] * h[j])
            k += 4
    return H


def profile_width(s: np.ndarray, f: np.ndarray, f0: float, rise: float = RISE):
    """Width of the interval around s = 0 over which f stays below f0 + rise: the distance between the first offsets on
    either side where it reaches it; None when a side never does within the profile (the axis is flat there)."""
    c = int(np.argmin(np.abs(s)))
    right = next((s[i] for i in range(c, len(s)) if f[i] >= f0 + rise), None)
    left = next((s[i] for i in range(c, -1, -1) if f[i] >= f0 + rise), None)
    if right is None or left is None:
        return None
    return float(right - left)


def weak_axes(curvature) -> list[int]:
    """Axes whose curvature is below WEAK_RATIO of the largest curvature of their kind (rotations, translations)."""
    c = np.asarray(curvature, dtype=np.float64)
    weak = []
    for group in (range(0, 3), range(3, 6)):
        top = max(c[k] for k in group)
        weak += [k for k in group if not (top > 0.0 and c[k] >= WEAK_RATIO * top)]
    return weak


def disagreeing_axes(curv_h, curv_2h) -> list[int]:
    """Axes whose curvatures at the two steps differ by more than STEP_DISAGREEMENT x (or in sign)."""
    out = []
    for k, (a, b) in enumerate(zip(curv_h, curv_2h)):
        if a <= 0.0 or b <= 0.0 or max(a, b) > STEP_DISAGREEMENT * min(a, b):
            out.append(k)
    return out


def pose_distance(T: np.ndarray, U: np.ndarray):
    """(translation distance, rotation angle in degrees) of T^-1 U."""
    D = np.linalg.inv(T) @ U
    R = D[:3, :3]
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    angle = math.atan2(0.5 * float(np.linalg.norm(v)), 0.5 * (float(np.trace(R)) - 1.0))
    return float(np.linalg.norm(D[:3, 3])), math.degrees(angle)


def random_starts(T: np.ndarray, n: int, rot_deg: float, trans: float, seed: int) -> np.ndarray:
    """n starts T * Exp(x): rotation of rot_deg about a random axis, translation of length trans in a random direction."""
    rng = np.random.default_rng(seed)
    xs = np.zeros((n, 6))
    for i in range(n):
        a, b = rng.normal(size=3), rng.normal(size=3)
        xs[i, :3] = a / np.linalg.norm(a) * math.radians(rot_deg)
        xs[i, 3:] = b / np.linalg.norm(b) * trans
    return tangent_poses(T, xs)


def local_shape(f_profiles: np.ndarray, f_h: np.ndarray, f_2h: np.ndarray, steps: int) -> dict:
    """Report of one objective (one bag, or the sum over bags) from its scores: profiles (6, steps), stencils (73,) at h and 2h."""
    s = np.linspace(-1.0, 1.0, steps)
    H = hessian_from_stencil(f_h, HESSIAN_STEP)
    H2 = hessian_from_stencil(f_2h, 2.0 * HESSIAN_STEP)
    w, V = np.linalg.eigh(H)
    f0 = float(f_h[0])
    curv, curv2 = np.diag(H), np.diag(H2)
    return {
        "nid_at_T": _num(f0),
        "profiles": [{"axis": AXES[k], "offset": [float(v) for v in s * PROFILE_HALF[k]], "nid": [_num(v) for v in f_profiles[k]]} for k in range(6)],
        "hessian": _mat(H),
        "hessian_2h": _mat(H2),
        "eigenvalues": [_num(v) for v in w],
        "eigenvectors": _mat(V.T),  # row i: the eigenvector of eigenvalue i
        "curvature": [_num(v) for v in curv],
        "curvature_2h": [_num(v) for v in curv2],
        "width": [profile_width(s * PROFILE_HALF[k], f_profiles[k], f0) for k in range(6)],
        "weak_axes": [AXES[k] for k in weak_axes(curv)],
        "step_disagreement_axes": [AXES[k] for k in disagreeing_axes(curv, curv2)],
    }


def summarize_solves(T: np.ndarray, nid_T: float, starts, ends, ys, iterations, bag_names, loo_ends) -> tuple[dict, list, list[str]]:
    """(summary, per-solve records, warnings) of the multi-start solves (starts / ends / ys / iterations) and the
    leave-one-bag-out end poses (loo_ends[b]: the optimum without bag b; empty below three bags)."""
    warnings = []
    records = []
    dists = []
    away = better = 0
    for i, (S, E, y, it) in enumerate(zip(starts, ends, ys, iterations)):
        dt, dr = pose_distance(T, E)
        is_away = dt > AWAY_TRANS or dr > AWAY_ROT_DEG
        is_lower = y < nid_T
        away += is_away
        better += is_lower
        if is_away and is_lower:
            warnings.append(f"multi-start solve {i} ended {dt * 1000:.1f} mm / {dr:.3f} deg from T with a lower NID ({y:.6f} < {nid_T:.6f}): a better optimum the calibration missed")
        dists.append((dt, dr))
        records.append({"kind": "multi_start", "start": vio.T_to_tum(np.linalg.inv(S)), "end": vio.T_to_tum(np.linalg.inv(E)), "distance_trans": dt, "distance_rot_deg": dr, "nid": _num(y), "iterations": int(it)})
    d = np.array(dists).reshape(-1, 2)
    summary = {
        "starts": len(starts),
        "max_trans": float(d[:, 0].max()) if len(d) else None,
        "rms_trans": float(np.sqrt(np.mean(d[:, 0] ** 2))) if len(d) else None,
        "max_rot_deg": float(d[:, 1].max()) if len(d) else None,
        "rms_rot_deg": float(np.sqrt(np.mean(d[:, 1] ** 2))) if len(d) else None,
        "ended_away": int(away),
        "lower_nid": int(better),
        "away_threshold": {"trans": AWAY_TRANS, "rot_deg": AWAY_ROT_DEG},
    }
    loo = []
    for b, E in enumerate(loo_ends):
        dt, dr = pose_distance(T, E)
        loo.append({"bag": bag_names[b], "distance_trans": dt, "distance_rot_deg": dr, "distance_normalised": max(dt / AWAY_TRANS, dr / AWAY_ROT_DEG)})
    if len(loo) >= 3:  # the median of two distances cannot single one out
        med = float(np.median([r["distance_normalised"] for r in loo]))
        for r in loo:
            if r["distance_normalised"] > 1.0 and r["distance_normalised"] > OUTLIER_FACTOR * med:
                warnings.append(f"bag {r['bag']} is an outlier: leaving it out moves the optimum {r['distance_trans'] * 1000:.1f} mm / {r['distance_rot_deg']:.3f} deg, more than {OUTLIER_FACTOR:g}x the median over the bags")
    summary["leave_one_out"] = loo
    return summary, records, warnings


def _num(v):
    v = float(v)
    return None if math.isnan(v) else v  # NaN: no point in view at that pose


def _mat(M):
    return [[_num(v) for v in row] for row in np.asarray(M)]


def assess(proj, dataset, bag_names, T_camera_lidar, nid_bins=16, starts=16, start_rot_deg=1.0, start_trans=0.05, profile_steps=41, disable_culling=False, seed=0, device=-1, params=None,
           dst_path=None):
    """The assessment report (dict) of T_camera_lidar on the dataset; with dst_path, also one <bag>_agreement.png per bag there."""
    if profile_steps < 3 or profile_steps % 2 == 0:
        raise ValueError("profile_steps must be odd and at least 3 (the profile passes through T)")
    first = dataset[0]
    culling = ViewCulling(proj, (first.image.shape[1], first.image.shape[0]), ViewCullingParams(not disable_culling), device=device)
    costs, culled = [], []
    try:
        for d in dataset:
            pts, ins = culling.cull(d.points, d.intensities, T_camera_lidar)
            culled.append(int(len(pts)))
            if dst_path is not None:  # the agreement map of the culled points (one launch sequence per bag, no host loop over points)
                import cv2

                _, _, bgr, _ = agreement_map(proj, d.image, T_camera_lidar, pts, ins, nid_bins, device=device)
                if not cv2.imwrite(os.path.join(dst_path, f"{bag_names[len(culled) - 1]}_agreement.png"), bgr):
                    raise OSError(f"failed to write {bag_names[len(culled) - 1]}_agreement.png")
            costs.append(CostCalculatorNID(proj, VisualLiDARData(d.image, pts, ins), NIDCostParams(nid_bins), device=device))
        # ---- local shape: one pose list per bag, one launch each ----
        prof = profile_offsets(profile_steps).reshape(-1, 6)
        st_h, st_2h = hessian_stencil(HESSIAN_STEP), hessian_stencil(2.0 * HESSIAN_STEP)
        poses = tangent_poses(T_camera_lidar, np.concatenate([prof, st_h, st_2h]))
        per_bag = np.stack([score_poses([c], poses) for c in costs])
        total = np.zeros(per_bag.shape[1])
        for row in per_bag:  # the objective's sum over bags, in bag order
            total = total + row
        n_prof = prof.shape[0]

        def shape_of(f):
            return local_shape(f[:n_prof].reshape(6, profile_steps), f[n_prof : n_prof + 73], f[n_prof + 73 :], profile_steps)

        local = {"per_bag": [dict(bag=n, **shape_of(f)) for n, f in zip(bag_names, per_bag)], "sum": shape_of(total)}
        # ---- solves: multi-start and leave-one-bag-out, one launch ----
        n_loo = len(costs) if len(costs) >= 2 else 0
        if starts + n_loo > MAX_SOLVES:
            raise ValueError(f"--starts {starts} and {n_loo} leave-one-out solves exceed the {MAX_SOLVES} solves of one launch")
        start_T = random_starts(T_camera_lidar, starts, start_rot_deg, start_trans, seed)
        init = np.concatenate([start_T, np.repeat(T_camera_lidar[None], n_loo, axis=0)])
        mask = np.ones((len(init), len(costs)), dtype=bool)
        for b in range(n_loo):
            mask[starts + b, b] = False
        params = copy.copy(params) if params is not None else VisualCameraCalibrationParams()
        params.nid_bins = nid_bins
        ends, res = estimate_poses_on_costs(costs, init, mask, params) if len(init) else (np.empty((0, 4, 4)), [])
    finally:
        for c in costs:
            c.close()
    nid_T = float(total[n_prof])
    summary, records, warnings = summarize_solves(T_camera_lidar, nid_T, start_T, ends[:starts], [r["y"] for r in res[:starts]], [r["num_iterations"] for r in res[:starts]], bag_names, ends[starts:])
    for b in range(n_loo):
        r = res[starts + b]
        records.append({"kind": "leave_one_out", "bag": bag_names[b], "start": vio.T_to_tum(np.linalg.inv(T_camera_lidar)), "end": vio.T_to_tum(np.linalg.inv(ends[starts + b])),
                        "distance_trans": summary["leave_one_out"][b]["distance_trans"], "distance_rot_deg": summary["leave_one_out"][b]["distance_rot_deg"], "nid": _num(r["y"]), "iterations": r["num_iterations"]})
    warnings = [f"axis {a} is weakly constrained: its curvature is below {WEAK_RATIO:g} of the largest of its kind" for a in local["sum"]["weak_axes"]] + \
               [f"axis {a}: the curvatures at the two Hessian steps disagree by more than {STEP_DISAGREEMENT:g}x" for a in local["sum"]["step_disagreement_axes"]] + warnings
    return {
        "axes": AXES,
        "nid_bins": nid_bins,
        "rise": RISE,
        "weak_ratio": WEAK_RATIO,
        "profile_half_range": {"rot_deg": 2.0, "trans": 0.10, "steps": profile_steps},
        "hessian_step": {"rot_deg": 0.05, "trans": 0.0025},
        "bag_names": list(bag_names),
        "culled_points": culled,
        "local": local,
        "solves": records,
        "summary": summary,
        "warnings": warnings,
    }


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="assess")
    ap.add_argument("data_path", help="directory that contains preprocessed data")
    ap.add_argument("--dst_path", default=None, help="directory assessment.json is written to (default: data_path)")
    ap.add_argument("--transformation", choices=[t[2] for t in TRANSFORMATIONS], default=None, help="the transformation to assess (default: the last one found)")
    ap.add_argument("--first_n_bags", type=int, default=None, help="use only the first N bags")
    ap.add_argument("--nid_bins", type=int, default=16)
    ap.add_argument("--starts", type=int, default=16, help="multi-start Nelder-Mead solves")
    ap.add_argument("--start_rot_deg", type=float, default=1.0, help="rotation of every start from T, degrees")
    ap.add_argument("--start_trans", type=float, default=0.05, help="translation of every start from T, metres")
    ap.add_argument("--profile_steps", type=int, default=41, help="poses per 1-D profile (odd)")
    ap.add_argument("--disable_culling", action="store_true", help="disable depth buffer-based hidden points removal")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=-1)
    args = ap.parse_args(argv)

    try:
        config = vio.load_calib_json(args.data_path)
    except OSError:
        print(f"error: failed to open {args.data_path}/calib.json", file=sys.stderr)
        return 1
    try:
        labels, T_lidar_camera, selected = find_transformations(config, args.transformation)
    except ValueError as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    if args.starts < 0 or args.profile_steps < 3 or args.profile_steps % 2 == 0:
        print("error: --starts must be >= 0 and --profile_steps odd and >= 3", file=sys.stderr)
        return 1
    cam = config["camera"]
    proj = create_camera(cam["camera_model"], cam["intrinsics"], cam["distortion_coeffs"])
    if proj is None:
        return 1
    bag_names = list(config["meta"]["bag_names"])
    if args.first_n_bags is not None:
        bag_names = bag_names[: args.first_n_bags]
    dataset = [vio.load_visual_lidar_data(args.data_path, name) for name in bag_names]
    print(f"assessing transformation: {labels[selected]}")
    dst = args.dst_path or args.data_path
    os.makedirs(dst, exist_ok=True)
    T_camera_lidar = vio.invert_isometry(T_lidar_camera[selected])
    try:
        report = assess(proj, dataset, bag_names, T_camera_lidar, args.nid_bins, args.starts, args.start_rot_deg, args.start_trans, args.profile_steps, args.disable_culling, args.seed, args.device,
                        dst_path=dst)
    except ValueError as e:
        print(f"error: {e}", file=sys.stderr)
        return 1
    report = {"transformation": labels[selected], "T_lidar_camera": vio.T_to_tum(T_lidar_camera[selected]), **report}
    with open(os.path.join(dst, "assessment.json"), "w") as f:
        f.write(json.dumps(report, indent=2) + "\n")
    s = report["local"]["sum"]
    print("axis  curvature       width")
    for k, a in enumerate(AXES):
        w = s["width"][k]
        print(f"{a:4s}  {s['curvature'][k]!s:14.14s}  {'flat' if w is None else f'{w:.6g}'}")
    sm = report["summary"]
    if sm["starts"]:
        print(f"multi-start: {sm['starts']} solves, max {sm['max_trans'] * 1000:.2f} mm / {sm['max_rot_deg']:.4f} deg from T, {sm['ended_away']} ended away")
    for w in report["warnings"]:
        print(f"warning: {w}")
    print(f"saved to {dst}/(assessment.json|<bag>_agreement.png)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
