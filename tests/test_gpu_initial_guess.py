"""GPU checks of initial_guess_auto: the RANSAC scoring launch against the CPU checker (tests/cpp/pose_oracle.c) for all six
camera models, the tiling at large M, determinism, the error paths, and the CLI end to end on a written dataset followed
by `calibrate`."""
import json
import os

import numpy as np
import pytest

import pose_oracle
import util
from direct_visual_lidar_calibration_b200 import io as vio
from direct_visual_lidar_calibration_b200 import pose_estimation as PE
from direct_visual_lidar_calibration_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _problem(model, m, seed, outliers=0.3, noise=1.0):
    """Projections of random points under the ground truth with pixel noise; a share of the keypoints replaced by random pixels."""
    intr, dist, (W, H) = util.CAMERAS[model]
    rng = np.random.default_rng(seed)
    T = S.gt_T_camera_lidar()
    pts = S.lidar_directions("sphere" if model == "equirectangular" else "avia", m, rng) * rng.uniform(1.0, 30.0, (m, 1))
    pts = pts.astype(np.float32).astype(np.float64)
    pc = pts @ T[:3, :3].T + T[:3, 3]
    from oracle import oracle as O

    ocam = O.create_camera(model, intr, dist)
    kp = np.array([O.project(ocam, p) for p in pc]) + rng.normal(0.0, noise, (m, 2))
    out = rng.random(m) < outliers
    kp[out] = rng.uniform([0, 0], [W, H], (int(out.sum()), 2))
    pts[5] = pts[4] * 2.0  # parallel LiDAR bearings: a degenerate hypothesis wherever 4 and 5 are drawn together
    return intr, dist, kp, pts, ocam


def _pairs(m, h, seed):
    pairs = PE.sample_pairs(m, h).copy()
    rng = np.random.default_rng(seed)
    k = rng.choice(h, 24, replace=False)
    pairs[k[:12], 1] = pairs[k[:12], 0]  # the same index twice
    pairs[k[12:]] = [4, 5]
    return pairs


def _check_counts(counts, degenerate, ref_counts, ref_degenerate, ref_near):
    assert np.array_equal(degenerate, ref_degenerate)
    diff = np.abs(counts.astype(np.int64) - ref_counts)
    assert np.all(diff <= ref_near), f"{int((diff > ref_near).sum())} hypotheses differ beyond the near-threshold correspondences"
    assert np.all(counts[degenerate] == 0)


@pytest.mark.parametrize("model", util.MODELS)
def test_counts_match_the_oracle(gpu, model):
    intr, dist, kp, pts, ocam = _problem(model, 2000, seed=11)
    pairs = _pairs(kp.shape[0], 8192, seed=1)
    cam = gpu.create_camera(model, intr, dist)
    counts, degenerate = PE.score_pairs(cam, kp, pts, pairs, 5.0)
    ref_counts, ref_degenerate, ref_near = pose_oracle.score(ocam, kp, pts, pairs, 5.0)
    _check_counts(counts, degenerate, ref_counts, ref_degenerate, ref_near)
    assert ref_degenerate.sum() >= 24
    assert counts.max() > 100  # the ground-truth rotation is among the hypotheses' neighbours
    # the winner rule: largest count, ties to the lowest index
    assert int(np.argmax(counts)) == int(np.argmax(ref_counts))


def test_tiling_at_large_m(gpu):
    model = "plumb_bob"
    intr, dist, kp, pts, ocam = _problem(model, 100_003, seed=12)
    pairs = _pairs(kp.shape[0], 320, seed=2)
    counts, degenerate = PE.score_pairs(gpu.create_camera(model, intr, dist), kp, pts, pairs, 5.0)
    ref_counts, ref_degenerate, ref_near = pose_oracle.score(ocam, kp, pts, pairs, 5.0)
    _check_counts(counts, degenerate, ref_counts, ref_degenerate, ref_near)
    assert counts.max() > 10_000


def test_estimate_is_deterministic_and_reports_its_winner(gpu):
    model = "fisheye"
    intr, dist, kp, pts, ocam = _problem(model, 3000, seed=13)
    cam = gpu.create_camera(model, intr, dist)
    runs = []
    for _ in range(2):
        est = PE.PoseEstimation()
        T, inliers = est.estimate(cam, kp, pts)
        runs.append((T, inliers, est.stats))
    assert runs[0][0].tobytes() == runs[1][0].tobytes()
    assert np.array_equal(runs[0][1], runs[1][1]) and runs[0][2] == runs[1][2]
    T, inliers, st = runs[0]
    pairs = PE.sample_pairs(kp.shape[0], 8192)
    ref_counts, ref_degenerate, ref_near = pose_oracle.score(ocam, kp, pts, pairs, 5.0)
    assert st["hypotheses"] == 8192 and st["degenerate"] == int(ref_degenerate.sum())
    assert st["best_index"] == int(np.argmax(ref_counts)) and abs(st["best_inliers"] - ref_counts.max()) <= ref_near[st["best_index"]]
    assert int(inliers.sum()) == st["best_inliers"]
    assert np.degrees(np.arccos(np.clip((np.trace(T[:3, :3].T @ S.gt_T_camera_lidar()[:3, :3]) - 1) / 2, -1, 1))) < 0.2


def test_no_inliers_is_an_error(gpu):
    intr, dist, kp, pts, _ = _problem("plumb_bob", 500, seed=14, outliers=1.0)
    cam = gpu.create_camera("plumb_bob", intr, dist)
    with pytest.raises(gpu.VlcalError, match="no hypothesis with an inlier"):
        PE.PoseEstimation(PE.PoseEstimationParams(ransac_iterations=64, ransac_error_thresh=1e-6)).estimate(cam, kp, pts)
    with pytest.raises(gpu.VlcalError, match="at least 2 correspondences"):
        PE.PoseEstimation().estimate(cam, kp[:1], pts[:1])


def _angle_deg(A, B):
    c = (np.trace(A[:3, :3].T @ B[:3, :3]) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))


def test_cli_writes_a_guess_calibrate_starts_from(gpu, oracle, tmp_path, capsys):
    from direct_visual_lidar_calibration_b200 import calibrate as calib_cli
    from direct_visual_lidar_calibration_b200 import initial_guess_auto as cli

    bags = S.write_initial_guess_dataset(str(tmp_path), n_bags=2, outlier_fraction=0.25, seed=5)
    assert cli.main([str(tmp_path)]) == 0
    out = capsys.readouterr().out
    assert "num_inliers: " in out and "--- T_lidar_camera ---" in out
    cfg = vio.load_calib_json(str(tmp_path))
    assert set(cfg) == {"camera", "meta", "results"} and list(cfg["results"]) == ["init_T_lidar_camera_auto"]
    T_gt = bags[0]["T_gt"]
    T_auto = vio.invert_isometry(vio.tum_to_T(cfg["results"]["init_T_lidar_camera_auto"]))
    assert _angle_deg(T_auto, T_gt) < 0.5
    assert np.linalg.norm(T_auto[:3, 3] - T_gt[:3, 3]) < 0.03

    # calibrate from that file, checked against the oracle's calibration from the same guess (as the existing CLI test)
    assert calib_cli.main([str(tmp_path), "--registration_type", "nid_nelder_mead"]) == 0
    cfg = vio.load_calib_json(str(tmp_path))
    T = vio.invert_isometry(vio.tum_to_T(cfg["results"]["T_lidar_camera"]))
    ocam = oracle.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    ref = oracle.calibrate(ocam, [(b["image"], b["points"], b["intensities"]) for b in bags], T_auto)
    assert np.abs(T - ref["T"]).max() < 1e-9
    with open(os.path.join(tmp_path, "bag0_matches.json")) as f:
        assert len(json.load(f)["matches"]) > 300
