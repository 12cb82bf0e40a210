"""GPU checks of the equirectangular delta step of the persistent kernel (csrc/lean_filter.cuh, classify_lean_delta):
poses 1..P-1 of a batch of nearby poses are classified as first-order updates from pose 0.  Every verdict it keeps must
be the exact path's, and the histograms of a batch that takes it must equal the oracle's."""
import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import synthetic as _S

pytestmark = pytest.mark.gpu


def _cost(V, pr, bins=16):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    data = V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])
    return V.CostCalculatorNID(cam, data, V.NIDCostParams(bins))


def _line_batch(T, rng, steps):
    """Pose 0 = T, then poses along one random direction through it (as Nelder-Mead's xr, xe, xc lie on a line through xo)."""
    rot = rng.normal(size=3)
    tr = rng.normal(size=3)
    rot *= np.degrees(1.0) / np.linalg.norm(rot)  # one radian per unit step
    tr /= np.linalg.norm(tr)
    return [T] + [_S.perturb(T, s * rot, s * tr) for s in steps]


def _c3_like_problem(n, seed):
    """C3-like geometry: equirectangular 3840x1920, points all around, some far, some close, some near the poles and the seam."""
    rng = np.random.default_rng(seed)
    pr = util.random_problem("equirectangular", n, seed=seed, size=(3840, 1920))
    pr["intrinsics"] = [3840.0, 1920.0]
    pts = pr["points"][:, :3].copy()
    k = n // 8
    pts[:k] *= rng.uniform(5.0, 40.0, (k, 1))                                          # far
    pts[k : 2 * k] = _S.lidar_directions("sphere", k, rng) * rng.uniform(0.05, 0.5, (k, 1))  # close to the sensor
    cam_dirs = _S.lidar_directions("sphere", 2 * k, rng) * rng.uniform(0.5, 25.0, (2 * k, 1))
    R, t = pr["T"][:3, :3], pr["T"][:3, 3]
    cam_dirs[:k, 0] *= 1e-3   # camera frame x ~ 0: near the poles (|y| ~ |p|) when z is small too, near the seam when z < 0
    cam_dirs[:k, 2] *= rng.choice([1e-3, 1.0], k)
    pts[2 * k : 4 * k] = (cam_dirs - t) @ R  # lidar frame
    pr["points"][:, :3] = pts.astype(np.float32).astype(np.float64)
    return pr


def test_delta_step_bound_is_sound_on_c3_like_geometry(gpu):
    """Delta mode of the verify kernel: 0 contradictions and error / bound < 1 over >= 1e7 point-poses."""
    total = 0
    deferred_total = 0
    for seed in (61, 62, 63):
        pr = _c3_like_problem(400000, seed)
        cost = _cost(gpu, pr)
        rng = np.random.default_rng(seed)
        Ts = []
        for _ in range(4):  # four 8-pose batches: anchor + 7 poses at 1e-6 .. 5e-3 rad / m along a line
            anchor = _S.perturb(pr["T"], rng.uniform(-2, 2, 3), rng.uniform(-0.1, 0.1, 3))
            Ts += _line_batch(anchor, rng, np.geomspace(1e-6, 5e-3, 7) * rng.choice([-1.0, 1.0], 7))
        n_pp, deferred, mismatches, ratio = cost.debug_filter_check(np.stack(Ts), delta=True)
        assert n_pp == 400000 * 32
        assert mismatches == 0
        assert ratio < 1.0, ratio
        total += n_pp
        deferred_total += deferred
    assert total >= 1e7
    print(f"delta step: {deferred_total / total:.4%} of {total} point-poses deferred")
    assert deferred_total / total < 0.2


def test_clustered_pose_list_takes_the_delta_step_and_matches_the_oracle(gpu, oracle):
    pr = util.random_problem("equirectangular", n=120000, seed=71)
    cost = _cost(gpu, pr)
    rng = np.random.default_rng(72)
    Ts = np.stack(_line_batch(pr["T"], rng, [1e-3, 2e-3, -1e-3, 5e-4, 1.5e-3, 2.5e-4, 1e-5]))  # one chunk of 8
    cost.reset_profile()
    nid, hist = cost.calculate_batch(Ts, return_hist=True)
    prof = cost.profile()
    assert prof["passes"] == 1 and prof["delta_passes"] == 1, prof
    cam = oracle.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = oracle.estimate_camera_fov(cam, pr["W"], pr["H"])
    ref = [oracle.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], 16, fov, T) for T in Ts]
    assert np.array_equal(hist, np.stack([r[1] for r in ref]))
    assert hist.sum() > 100000
    assert np.all(np.abs(nid - np.array([r[0] for r in ref])) < 1e-12)
    # a widely spread list takes the plain classifier
    cost.reset_profile()
    cost.calculate_batch(util.random_poses(pr["T"], 8, seed=3, rot_deg=5.0, trans=0.5))
    assert cost.profile()["delta_passes"] == 0
