"""GPU checks of the anchor of the equirectangular delta step (csrc/lean_filter.cuh: lean_delta_anchor): the most
central pose of a batch is classified first, through the plain classifier, and the others as first-order updates from
it.  With the anchor at a non-zero index every kept verdict must still be the exact path's, and every pose's counts must
land in its own histogram."""
import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import synthetic as _S

pytestmark = pytest.mark.gpu


def _cost(V, pr, bins=16):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    data = V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])
    return V.CostCalculatorNID(cam, data, V.NIDCostParams(bins))


def _line(T, rng, steps, size):
    """poses T * Exp(s * diff) for s in steps, diff a random direction of `size` rad and metres"""
    w, v = rng.normal(size=3), rng.normal(size=3)
    w *= size / np.linalg.norm(w)
    v *= size / np.linalg.norm(v)
    return [_S.perturb(T, tuple(np.degrees(s * w)), tuple(s * v)) for s in steps]


def _c3_like_problem(n, seed):
    """equirectangular 3840x1920, points all around: far, close to the sensor, near the poles and the seam"""
    rng = np.random.default_rng(seed)
    pr = util.random_problem("equirectangular", n, seed=seed, size=(3840, 1920))
    pr["intrinsics"] = [3840.0, 1920.0]
    pts = pr["points"][:, :3].copy()
    k = n // 8
    pts[:k] *= rng.uniform(5.0, 40.0, (k, 1))
    pts[k : 2 * k] = _S.lidar_directions("sphere", k, rng) * rng.uniform(0.05, 0.5, (k, 1))
    cam_dirs = _S.lidar_directions("sphere", 2 * k, rng) * rng.uniform(0.5, 25.0, (2 * k, 1))
    R, t = pr["T"][:3, :3], pr["T"][:3, 3]
    cam_dirs[:k, 0] *= 1e-3
    cam_dirs[:k, 2] *= rng.choice([1e-3, 1.0], k)
    pts[2 * k : 4 * k] = (cam_dirs - t) @ R
    pr["points"][:, :3] = pts.astype(np.float32).astype(np.float64)
    return pr


# Nelder-Mead iteration {xo, xr, xe, xc} (anchor: xr, index 1), twice per group of 8, and an 8-pose line whose central
# pose (s = 0) sits at index 3
ITERATION = (0.0, 1.0, 2.0, 0.5)
CENTRAL_AT_3 = (-3.0, -2.0, -1.0, 0.0, 1.0, 2.0, 3.0, 0.5)


def test_delta_step_with_a_central_anchor_is_sound_on_c3_like_geometry(gpu):
    """Verify kernel, delta mode, anchor at index 1 or 3: 0 contradictions and error / bound < 1."""
    total = 0
    for seed in (81, 82):
        pr = _c3_like_problem(300000, seed)
        cost = _cost(gpu, pr)
        rng = np.random.default_rng(seed)
        Ts = []
        for size in (1e-4, 1e-3, 2e-3):
            anchor = _S.perturb(pr["T"], rng.uniform(-2, 2, 3), rng.uniform(-0.1, 0.1, 3))
            Ts += _line(anchor, rng, ITERATION, size) + _line(anchor, rng, ITERATION, size / 2)
            Ts += _line(anchor, rng, CENTRAL_AT_3, size)
        n_pp, deferred, mismatches, ratio = cost.debug_filter_check(np.stack(Ts), delta=True)
        assert n_pp == 300000 * len(Ts)
        assert mismatches == 0
        assert ratio < 1.0, ratio
        assert deferred / n_pp < 0.2
        total += n_pp
    assert total >= 1e7


def test_pose_list_with_the_central_pose_not_first_matches_the_plain_instance(gpu, oracle):
    """One chunk of 8 inside the gate only around its central pose (index 3): it takes the delta step, and every pose's
    histogram equals the plain instance's (one-pose chunks) and the oracle's."""
    pr = _c3_like_problem(150000, 91)
    cost = _cost(gpu, pr)
    rng = np.random.default_rng(92)
    # s = -3 .. 3 at 1.2e-3 rad: poses 0 and 6 are 7.2e-3 rad apart, > 4e-3 in the rotation's largest axis component (>= 1/sqrt3
    # of it) -- outside the gate from pose 0; from index 3 every pose is within 3.6e-3 rad
    Ts = np.stack(_line(pr["T"], rng, CENTRAL_AT_3, 1.2e-3))
    cost.reset_profile()
    _, hist = cost.calculate_batch(Ts, return_hist=True)
    prof = cost.profile()
    assert prof["passes"] == 1 and prof["delta_passes"] == 1, prof
    assert hist.sum() > 100000
    plain = [cost.calculate_batch(T[None], return_hist=True) for T in Ts]
    assert cost.profile()["delta_passes"] == 1  # the one-pose chunks took the plain instance
    assert np.array_equal(hist, np.concatenate([h for _, h in plain]))
    cam = oracle.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = oracle.estimate_camera_fov(cam, pr["W"], pr["H"])
    ref = [oracle.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], 16, fov, T) for T in Ts]
    assert np.array_equal(hist, np.stack([r[1] for r in ref]))
