"""Host-side checks of initial_guess_auto: the lidar-index PNG, the correspondence rules, the RANSAC's hypothesis
sampling, the bearings and the Levenberg-Marquardt refinement (no GPU needed)."""
import json

import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

import pose_oracle
import util
from direct_visual_lidar_calibration_b200 import io as vio
from direct_visual_lidar_calibration_b200 import pose_estimation as PE
from direct_visual_lidar_calibration_b200 import synthetic as S


def test_lidar_indices_png_roundtrips_int32_exactly(tmp_path):
    rng = np.random.default_rng(0)
    idx = rng.integers(-1, 5_000_000, (37, 53), dtype=np.int64).astype(np.int32)
    idx[0, :4] = [-1, 0, 2**31 - 1, -(2**31)]
    idx[5:9, 7:20] = -1
    path = str(tmp_path / "bag_lidar_indices.png")
    vio.save_lidar_indices(path, idx)
    back = vio.load_lidar_indices(path)
    assert back.dtype == np.int32 and np.array_equal(back, idx)


def _fixture(tmp_path):
    """6 x 5 index image; keypoints exercise truncation, -1 matches, a blank pixel with a point next to it and one without."""
    idx = -np.ones((5, 6), dtype=np.int32)
    idx[1, 1], idx[1, 2], idx[3, 4], idx[4, 0] = 7, 3, 0, 9
    #                  kpts1 pixel       ->  point
    kpts1 = [1.99, 1.2,   # 0: (1, 1)  -> 7
             2.0, 1.999,  # 1: (2, 1)  -> 3
             3.5, 2.5,    # 2: (3, 2)  blank, neighbour (4, 3) has a point -> skipped without a warning
             5.5, 0.2,    # 3: (5, 0)  blank, no neighbour with a point -> skipped with the warning
             4.0, 3.0,    # 4: (4, 3)  -> 0
             0.3, 4.9]    # 5: (0, 4)  -> 9
    kpts0 = [10.9, 20.1,  -0.7, 5.5,  3.0, 4.0,  7.2, 8.8,  100.99, 200.5,  1.5, 2.5,  9.9, 9.9]
    matches = [0, 1, -1, 2, 3, 4, 5]
    data = {"kpts0": kpts0, "kpts1": kpts1, "matches": matches, "confidence": [0.5] * 7}
    with open(tmp_path / "b_matches.json", "w") as f:
        json.dump(data, f)
    vio.save_lidar_indices(str(tmp_path / "b_lidar_indices.png"), idx)
    points = np.arange(30, dtype=np.float64).reshape(10, 3) + 1.0
    return idx, data, points


def test_correspondence_rules_match_the_fixture_and_the_oracle(tmp_path, capsys):
    idx, data, points = _fixture(tmp_path)
    kp0, pts = vio.read_correspondences(str(tmp_path), "b", points)
    # kpts0 entries 0, 1, 5, 6 survive; their keypoints are truncated toward zero like static_cast<int>
    assert kp0.tolist() == [[10.0, 20.0], [0.0, 5.0], [1.0, 2.0], [9.0, 9.0]]
    assert np.array_equal(pts, points[[7, 3, 0, 9]])
    assert capsys.readouterr().out.count("warning: ignore keypoint in a blank region!!") == 1
    used, point_index, warnings = pose_oracle.correspondences(idx, data["kpts0"], data["kpts1"], data["matches"], points.shape[0])
    assert used.tolist() == [0, 1, 5, 6] and point_index.tolist() == [7, 3, 0, 9] and warnings == 1


@pytest.mark.parametrize("edit, message", [
    (lambda d: d["kpts1"].__setitem__(0, 6.0), "outside"),   # x = 6 in a 6-wide image
    (lambda d: d["kpts1"].__setitem__(1, -1.5), "outside"),  # y = -1
    (lambda d: d["matches"].__setitem__(0, 6), "past the 6 kpts1"),
])
def test_correspondence_loader_rejects_out_of_range_input(tmp_path, edit, message):
    idx, data, points = _fixture(tmp_path)
    edit(data)
    with open(tmp_path / "b_matches.json", "w") as f:
        json.dump(data, f)
    with pytest.raises(ValueError, match=message):
        vio.read_correspondences(str(tmp_path), "b", points)
    with pytest.raises(ValueError):
        pose_oracle.correspondences(idx, data["kpts0"], data["kpts1"], data["matches"], points.shape[0])


def test_correspondence_loader_rejects_point_index_past_the_cloud(tmp_path):
    idx, data, points = _fixture(tmp_path)
    with pytest.raises(ValueError, match="past the 9 points"):
        vio.read_correspondences(str(tmp_path), "b", points[:9])


def test_ransac_samples_what_a_one_thread_reference_run_samples():
    # std::mt19937 mt; mts[0] = std::mt19937(mt() + 8192 * 0); two uniform_int_distribution<>(0, M-1) draws per iteration
    assert PE.sample_pairs(37, 16).tolist() == [
        [20, 26], [12, 33], [0, 21], [32, 19], [35, 36], [6, 24], [11, 19], [25, 29], [9, 2], [21, 12], [12, 21], [8, 1], [6, 34], [35, 0], [24, 28], [17, 12]]
    assert PE.sample_pairs(1000, 16).tolist() == [
        [561, 726], [348, 915], [6, 594], [872, 515], [959, 975], [169, 661], [316, 528], [701, 788], [255, 74], [574, 329], [338, 583], [238, 30],
        [172, 928], [966, 19], [653, 779], [477, 336]]
    assert np.array_equal(PE.sample_pairs(1000, 8192)[:16], PE.sample_pairs(1000, 16))


@pytest.mark.parametrize("model", util.MODELS)
def test_bearings_bit_identical_to_the_oracle(vlcal, oracle, model):
    intr, dist, (W, H) = util.CAMERAS[model]
    rng = np.random.default_rng(3)
    px = np.floor(rng.uniform([0, 0], [W, H], (200, 2)))
    got = PE.estimate_directions(vlcal.create_camera(model, intr, dist), px)
    dc, _ = pose_oracle.bearings(oracle.create_camera(model, intr, dist), px, np.ones((200, 3)))
    assert np.array_equal(got, dc)


def _exact_problem(vlcal, model, n=400, seed=0):
    intr, dist, (W, H) = util.CAMERAS[model]
    cam = vlcal.create_camera(model, intr, dist)
    rng = np.random.default_rng(seed)
    T = S.gt_T_camera_lidar()
    pts = S.lidar_directions("sphere" if model == "equirectangular" else "avia", n, rng) * rng.uniform(2.0, 20.0, (n, 1))
    pts = pts.astype(np.float32).astype(np.float64)
    kp = cam.project(pts @ T[:3, :3].T + T[:3, 3])
    T0 = np.eye(4)
    T0[:3, :3] = S.perturb(T, (1.0, -1.0, 1.5), (0, 0, 0))[:3, :3]  # a RANSAC-like start: rotation off by ~2 deg, t = 0
    return cam, T, pts, kp, T0


@pytest.mark.parametrize("model", util.MODELS)
def test_refinement_recovers_the_exact_pose(vlcal, model):
    cam, T, pts, kp, T0 = _exact_problem(vlcal, model)
    T_est, iterations, cost = PE.refine(cam, kp, pts, T0, 10.0)
    assert np.abs(T_est - T).max() < 1e-9, (iterations, cost)


def _plumb_bob_np(intr, dist, pc):
    x, y = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
    k1, k2, p1, p2, k3 = dist
    r2 = x * x + y * y
    rc = 1 + k1 * r2 + k2 * r2**2 + k3 * r2**3
    xd = rc * x + p1 * 2 * x * y + p2 * (r2 + 2 * x * x)
    yd = rc * y + p1 * (r2 + 2 * y * y) + p2 * 2 * x * y
    return np.stack([intr[0] * xd + intr[2], intr[1] * yd + intr[3]], axis=1)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_refinement_with_outliers_is_a_minimum(vlcal, seed):
    intr, dist, (W, H) = util.CAMERAS["plumb_bob"]
    cam, T, pts, kp, T0 = _exact_problem(vlcal, "plumb_bob", n=500, seed=seed)
    rng = np.random.default_rng(100 + seed)
    kp = kp + rng.normal(0.0, 0.5, kp.shape)
    out = rng.choice(kp.shape[0], kp.shape[0] * 3 // 10, replace=False)
    kp[out] = rng.uniform([0, 0], [W, H], (out.size, 2))
    T_est, _, cost = PE.refine(cam, kp, pts, T0, 10.0)

    # the same objective, 1/2 sum b log(1 + |r_i|^2 / b), minimised independently by scipy (numpy projection, rotation vector)
    def residual_norms(x, Tb):
        R = Rotation.from_rotvec(x[:3]).as_matrix()
        return np.linalg.norm(_plumb_bob_np(intr, dist, pts @ (R @ Tb[:3, :3]).T + (R @ Tb[:3, 3] + x[3:])) - kp, axis=1)

    tight = dict(loss="cauchy", f_scale=10.0, ftol=1e-15, xtol=1e-15, gtol=1e-15)
    ref = least_squares(residual_norms, np.zeros(6), args=(T0,), **tight)
    assert cost <= ref.cost * (1 + 1e-9)
    assert abs(0.5 * np.sum(100.0 * np.log1p(residual_norms(np.zeros(6), T_est) ** 2 / 100.0)) - cost) <= 1e-9 * cost
    # stationary: per tangent direction, the decrease a Newton step on the robust cost would still make (g^2 / 2h, central
    # differences) is negligible
    def F(x):
        return 0.5 * np.sum(100.0 * np.log1p(residual_norms(x, T_est) ** 2 / 100.0))

    for k in range(6):
        e = np.zeros(6)
        e[k] = 1e-5
        fp, f0, fm = F(e), F(np.zeros(6)), F(-e)
        g, h = (fp - fm) / 2e-5, (fp - 2 * f0 + fm) / 1e-10
        assert h > 0 and g * g / (2 * h) <= 1e-10 * cost, (k, g, h)


def test_fewer_than_two_correspondences_is_an_error(vlcal):
    cam = vlcal.create_camera("plumb_bob", *util.CAMERAS["plumb_bob"][:2])
    with pytest.raises(vlcal.VlcalError, match="at least 2 correspondences"):
        PE.PoseEstimation().estimate(cam, np.zeros((1, 2)), np.ones((1, 3)))
    with pytest.raises(vlcal.VlcalError, match="at least 2 correspondences"):
        PE.PoseEstimation().estimate(cam, np.zeros((0, 2)), np.ones((0, 3)))
