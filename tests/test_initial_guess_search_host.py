"""Host side of initial_guess_search: the rotation set, the search sets' host generator, the image / camera / cloud
pyramids, non-maximum suppression and the whole driver with an injected scorer (no GPU needed)."""
import json
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import util
from direct_visual_lidar_calibration_b200 import create_camera
from direct_visual_lidar_calibration_b200 import initial_guess as ig
from direct_visual_lidar_calibration_b200 import initial_guess_search as igs
from direct_visual_lidar_calibration_b200 import io as vio
from direct_visual_lidar_calibration_b200 import synthetic as S


def _all_rotations(s):
    ib, il, _ = s.split()
    return s.rotations(ib, il)


# ---- rotation set -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("step", [3.0, 7.5, 20.0])
def test_rotation_set_counts_and_orthonormality(step):
    d = math.radians(step)
    assert ig.rotation_set_counts(step) == (math.ceil(4 * math.pi / d**2), math.ceil(2 * math.pi / d))
    s = ig.rotation_set(step)
    assert s.n_poses == np.prod(ig.rotation_set_counts(step)) and s.indices is None
    R = _all_rotations(s)[:: max(1, s.n_poses // 20000)]
    assert np.abs(np.einsum("nij,nkj->nik", R, R) - np.eye(3)).max() < 1e-15
    assert np.abs(np.linalg.det(R) - 1.0).max() < 1e-15
    T = s.poses(np.arange(0, s.n_poses, max(1, s.n_poses // 50)))
    assert np.array_equal(T[:, :3, 3], np.zeros((len(T), 3))) and np.array_equal(T[:, 3], np.tile([0.0, 0.0, 0.0, 1.0], (len(T), 1)))


def test_rotation_set_covers_so3():
    step = 6.0
    R = _all_rotations(ig.rotation_set(step)).reshape(-1, 9)
    Q = Rotation.random(2000, random_state=3).as_matrix().reshape(-1, 9)
    tr = np.concatenate([(Q[i : i + 250] @ R.T).max(axis=1) for i in range(0, 2000, 250)])
    nearest = np.degrees(np.arccos(np.clip((tr - 1.0) / 2.0, -1.0, 1.0)))
    assert nearest.max() < 0.8 * step


def test_rotation_set_with_a_prior_keeps_exactly_the_members_in_range():
    prior = np.eye(4)
    prior[:3, :3] = Rotation.from_rotvec([0.4, -0.9, 0.2]).as_matrix()
    prior[:3, 3] = [0.3, -0.1, 0.2]
    full, part = ig.rotation_set(8.0), ig.rotation_set(8.0, prior, 30.0)
    ang = ig.rotation_angle_deg(_all_rotations(full), prior[:3, :3].T)
    assert np.array_equal(part.indices, np.nonzero(ang <= 30.0)[0]) and 0 < part.n_poses < full.n_poses
    again = ig.rotation_set(8.0, prior, 30.0)
    assert again.poses().tobytes() == part.poses().tobytes()
    # the camera position of every pose is the prior's
    T = part.poses()
    pos = -np.einsum("nji,nj->ni", T[:, :3, :3], T[:, :3, 3])
    assert np.abs(pos - prior[:3, 3]).max() < 1e-15
    assert ig.rotation_set(8.0, prior, 180.0).n_poses == full.n_poses


def test_local_set_layout():
    cands = np.stack([S.gt_T_camera_lidar(), S.perturb(S.gt_T_camera_lidar(), (20, -30, 40), (0.5, 0.1, -0.2))])
    s = ig.local_set(cands, 1.5, 0.15, 2)
    assert s.n_poses == 2 * 27 * 125
    T = s.poses()
    centre = (13 * 125) + 62  # the zero rotation and the zero offset
    for b in range(2):
        assert np.abs(T[b * 27 * 125 + centre] - cands[b]).max() < 1e-15
    ang = ig.rotation_angle_deg(T[: 27 * 125 : 125, :3, :3], cands[0, :3, :3])
    assert ang.min() == 0.0 and abs(ang.max() - 1.5 * math.sqrt(3.0)) < 1e-9
    pos = -np.einsum("nji,nj->ni", T[:125, :3, :3], T[:125, :3, 3]) - (-cands[0, :3, :3].T @ cands[0, :3, 3])
    assert np.abs(np.abs(pos).max(axis=0) - 0.3).max() < 1e-12 and np.unique(np.round(pos, 9)).size == 5
    with pytest.raises(ValueError, match="index out of range"):
        ig.SearchSet(s.left, s.base, s.center, s.offset, indices=[s.n_poses])


# ---- pyramids -----------------------------------------------------------------------------------------------------------

def test_box_halve_and_crop():
    img = np.arange(7 * 9, dtype=np.uint8).reshape(7, 9) * 3
    half = ig.box_halve(img)
    assert half.shape == (3, 4)
    ref = np.floor(img[:6, :8].astype(np.float64).reshape(3, 2, 4, 2).mean(axis=(1, 3)) + 0.5)
    assert np.array_equal(half, ref.astype(np.uint8))
    rng = np.random.default_rng(0)
    big = rng.integers(0, 256, (101, 203), dtype=np.uint8)
    assert ig.pyramid_image(big, 8).shape == (12, 25) and ig.pyramid_image(big, 1) is not None
    assert np.array_equal(ig.pyramid_image(big, 1), big)
    assert ig.pyramid_image(big, 4).tobytes() == ig.pyramid_image(big.copy(), 4).tobytes()
    assert ig.pyramid_image(big, 4).max() == 255  # re-equalised
    with pytest.raises(ValueError):
        ig.pyramid_image(big, 3)


@pytest.mark.parametrize("model", util.MODELS)
def test_level_camera_projects_to_the_full_resolution_pixel_divided_by_the_scale(model):
    intr, dist, (W, H) = util.CAMERAS[model]
    rng = np.random.default_rng(5)
    pts = S.lidar_directions("frustum", 400, rng) @ S.R_CAMERA_LIDAR.T * rng.uniform(1.0, 20.0, (400, 1))
    uv = create_camera(model, intr, dist).project(pts)
    for s in (2, 4, 8):
        uvs = create_camera(model, ig.pyramid_intrinsics(model, intr, s), dist).project(pts)
        ok = np.isfinite(uv).all(axis=1) & (uv > 0).all(axis=1) & (uv[:, 0] < W) & (uv[:, 1] < H) & (np.abs(uv - np.round(uv)).min(axis=1) > 1e-6)
        assert ok.sum() > 100
        assert np.array_equal(np.trunc(uvs[ok]).astype(int), np.trunc(uv[ok]).astype(int) // s)
    assert ig.pyramid_intrinsics("omnidir", util.CAMERAS["omnidir"][0], 4)[4] == util.CAMERAS["omnidir"][0][4]


def test_cloud_subsets_are_nested_and_seeded():
    a, b = ig.cloud_subset(100_000, 16384, seed=4), ig.cloud_subset(100_000, 65536, seed=4)
    assert np.array_equal(a, b[:16384]) and np.unique(b).size == 65536
    assert ig.cloud_subset(1000, 16384, seed=4).size == 1000
    assert ig.cloud_subset(100_000, 16384, seed=4).tobytes() == a.tobytes() and not np.array_equal(a, ig.cloud_subset(100_000, 16384, seed=5))


# ---- non-maximum suppression ----------------------------------------------------------------------------------------------

def test_nms_top_k_with_nans_and_ties():
    def rz(deg):
        T = np.eye(4)
        T[:3, :3] = Rotation.from_euler("z", deg, degrees=True).as_matrix()
        return T

    poses = np.stack([rz(a) for a in (0.0, 1.0, 10.0, 10.5, 20.0, 30.0, 40.0)])
    scores = np.array([0.5, 0.4, 0.4, 0.3, np.nan, 0.4, 0.9])
    kept = ig.nms_top_k(lambda w: poses[w], scores, keep=10, min_sep_deg=2.0)
    # 10.5 deg wins and suppresses 10 deg; 1 deg before 30 deg (tie, list order) and suppresses 0 deg; NaN last
    assert kept.tolist() == [3, 1, 5, 6, 4]
    assert ig.nms_top_k(lambda w: poses[w], scores, keep=2, min_sep_deg=2.0).tolist() == [3, 1]
    assert ig.nms_top_k(lambda w: poses[w], scores, keep=3, min_sep_deg=0.0).tolist() == [3, 1, 2]


# ---- the driver with an injected scorer -----------------------------------------------------------------------------------

def _synthetic_scorer(T_gt, calls):
    pg = -T_gt[:3, :3].T @ T_gt[:3, 3]

    def score(level, sset):
        T = sset.poses()
        ang = ig.rotation_angle_deg(T[:, :3, :3], T_gt[:3, :3])
        pos = -np.einsum("nji,nj->ni", T[:, :3, :3], T[:, :3, 3])
        nid = 1.0 - 0.3 * np.exp(-((ang / 20.0) ** 2) - (np.linalg.norm(pos - pg, axis=1) / 0.5) ** 2)
        inliers = np.full(len(T), 1000, dtype=np.int64)
        inliers[ang > 170.0] = 3  # poses that see next to nothing ...
        nid[ang > 170.0] = 0.0    # ... and score spuriously well
        calls.append((dict(level), sset.n_poses))
        return nid, inliers, 1.25
    return score


def test_level_schedule():
    lv = igs.level_schedule(3.0, 0.3, 64)
    assert [l["scale"] for l in lv] == [8, 4, 2, 1, 1] and [l["step_deg"] for l in lv] == [3.0, 1.5, 0.75, 0.375, 0.1875]
    assert [l["points"] for l in lv] == [16384 * 4**i for i in range(5)] and [l["keep"] for l in lv] == [64, 32, 16, 8, 8]
    assert [(l["trans_spacing"], l["trans_half_steps"]) for l in lv[1:]] == [(0.15, 2), (0.075, 1), (0.0375, 1), (0.01875, 1)]
    assert len(igs.level_schedule(0.2, 0.3, 4)) == 4 and igs.level_schedule(0.2, 0.3, 4)[-1]["scale"] == 1


def test_driver_finds_the_minimum_and_sets_aside_empty_views():
    T_gt = S.perturb(S.gt_T_camera_lidar(), (25.0, -12.0, 31.0), (0.12, -0.2, 0.07))
    calls = []
    rep = igs.run_search(_synthetic_scorer(T_gt, calls), rot_step_deg=6.0, keep=16, log=lambda *_: None)
    assert [c[1] for c in calls] == [np.prod(ig.rotation_set_counts(6.0)), 16 * 27 * 125, 8 * 27 * 27, 8 * 27 * 27, 8 * 27 * 27, 8 * 27 * 27]
    assert [l["poses"] for l in rep["levels"]] == [c[1] for c in calls] and all(l["kernel_ms"] == 1.25 for l in rep["levels"])
    T = rep["T_camera_lidar"]
    assert ig.rotation_angle_deg(T[:3, :3], T_gt[:3, :3]) < 0.2
    assert np.linalg.norm(vio.invert_isometry(T)[:3, 3] - vio.invert_isometry(T_gt)[:3, 3]) < 0.02
    assert len(rep["top"]) == 5 and rep["top"][0]["nid"] == rep["levels"][-1]["best_nid"][0] > 0.69
    assert 0.0 < rep["margin"] < 0.3
    for c in rep["candidates"]:
        assert np.all(np.diff(c["nid"]) >= 0)


def _dataset(tmp_path):
    cfg = {"camera": {"camera_model": "plumb_bob", "intrinsics": [400.0, 400.0, 320.0, 240.0], "distortion_coeffs": [0.0] * 5},
           "meta": {"bag_names": ["bag0", "bag1"], "data_path": "somewhere"}, "results": {"T_lidar_camera": [0, 0, 0, 0, 0, 0, 1]}}
    vio.save_calib_json(str(tmp_path), cfg)
    return cfg


def test_cli_writes_the_key_calibrate_reads_and_the_report(tmp_path, capsys):
    cfg = _dataset(tmp_path)
    T_gt = S.perturb(S.gt_T_camera_lidar(), (5.0, 8.0, -6.0), (0.1, 0.05, -0.1))
    prior = vio.T_to_tum(vio.invert_isometry(S.gt_T_camera_lidar()))
    calls = []
    argv = [str(tmp_path), "--prior", *map(str, prior), "--rot_range_deg", "25", "--rot_step_deg", "5", "--keep", "8"]
    assert igs.main(argv, score=_synthetic_scorer(T_gt, calls)) == 0
    out = capsys.readouterr().out
    assert "level 0: 1/8 image, step 5 deg" in out and "--- T_lidar_camera ---" in out and "margin" in out
    assert calls[0][1] < 0.05 * np.prod(ig.rotation_set_counts(5.0))
    new = vio.load_calib_json(str(tmp_path))
    assert new["camera"] == cfg["camera"] and new["meta"] == cfg["meta"] and new["results"]["T_lidar_camera"] == cfg["results"]["T_lidar_camera"]
    assert list(new["results"]) == ["T_lidar_camera", "init_T_lidar_camera_auto"]
    T = vio.invert_isometry(vio.tum_to_T(new["results"]["init_T_lidar_camera_auto"]))
    assert ig.rotation_angle_deg(T[:3, :3], T_gt[:3, :3]) < 0.3
    with open(tmp_path / "initial_guess_search.json") as f:
        rep = json.load(f)
    assert set(rep) == {"levels", "top", "margin"} and len(rep["top"]) == 5 and set(rep["top"][0]) == {"T_lidar_camera", "nid"}
    assert set(rep["levels"][0]) == {"level", "scale", "points_per_bag", "step_deg", "trans_spacing", "poses", "kernel_ms", "wall_ms", "kept", "best_nid"}


@pytest.mark.parametrize("extra, message", [
    (["--rot_step_deg", "0"], "must be positive"),
    (["--rot_step_deg", "-3"], "must be positive"),
    (["--trans_range", "0"], "must be positive"),
    (["--rot_range_deg", "-1"], "must be positive"),
    (["--rot_step_deg", "15"], "leaves gaps"),
    (["--keep", "0"], "at least 1"),
    (["--first_n_bags", "0"], "at least 1"),
    (["--prior", "0", "0", "0", "0", "0", "0", "2"], "not of unit length"),
    (["--prior", "0", "0", "0", "0", "0", "0", "0"], "not of unit length"),
    (["--rot_range_deg", "40"], "needs --prior"),
])
def test_cli_refuses(tmp_path, capsys, extra, message):
    _dataset(tmp_path)
    before = (tmp_path / "calib.json").read_bytes()
    assert igs.main([str(tmp_path)] + extra, score=lambda *_: pytest.fail("must not score")) == 1
    assert message in capsys.readouterr().err
    assert (tmp_path / "calib.json").read_bytes() == before


def test_cli_refuses_a_missing_dataset_and_an_unknown_camera(tmp_path, capsys):
    assert igs.main([str(tmp_path / "nowhere")], score=lambda *_: None) == 1
    assert "failed to open" in capsys.readouterr().err
    cfg = _dataset(tmp_path)
    cfg["camera"]["camera_model"] = "pinhole9"
    vio.save_calib_json(str(tmp_path), cfg)
    assert igs.main([str(tmp_path)], score=lambda *_: None) == 1
    assert "unknown camera model" in capsys.readouterr().err
