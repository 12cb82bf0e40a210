"""The RANSAC hypothesis rotation (CPU, no GPU): the closed form the scoring kernel and its checker (tests/cpp/pose_oracle.c)
share, R = a^ p^T + b^ q^T + (a^ x b^)(p^ x q^)^T with a = c1 + c2, b = c1 - c2, p = l1 + l2, q = l1 - l2, held to the
reference's own find_rotation (estimate_pose.cpp:55-83) restated with numpy.linalg.svd:

    AB = sum_k c_k l_k^T,   AB = U D V^T,   S = diag(1, 1, sign(det U det V)),   R = U S V^T.

AB has rank 2 with singular values sigma_1 >= sigma_2 = min(|a||p|, |b||q|) / 2 (and 0).  Both constructions recover
its singular vectors to about eps / sigma_2 (the SVD's perturbation bound; in the closed form the rounding of
c1 - c2 and l1 - l2 divided by |b| and |q|), so

    ||R_closed - R_svd||_F <= 16 eps / sigma_2.

Measured over these cases the ratio stays below 6.  Where sigma_2 >= 1/4, R^T R = I and det R = 1 hold to 16 eps
(3.6e-15; the closed form reaches 7 eps, and U S V^T from numpy's SVD itself 10 eps in the same measure, so 1e-15 is
below what evaluating R^T R in double resolves).  Nearer parallel the closed form's a^ and b^ are orthogonal only to the
unit-norm rounding of the bearings over |b|, so there the eps / sigma_2 bound above applies to them.  The GPU suite
(test_gpu_ransac_edges.py) holds the kernel bit for bit to the checker, so these bounds are statements about the
kernel's rotation too."""
import numpy as np
import pytest

import pose_oracle

EPS = np.finfo(np.float64).eps
K = 16.0


def _unit(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])  # Eigen normalized(), as the LiDAR bearings


def _svd_rotation(c1, c2, l1, l2):
    AB = np.outer(c1, l1) + np.outer(c2, l2)
    U, s, Vt = np.linalg.svd(AB)
    S = np.diag([1.0, 1.0, -1.0 if np.linalg.det(U) * np.linalg.det(Vt) < 0.0 else 1.0])
    return U @ S @ Vt, s


def _at_angle(v, angle, rng):
    """A unit vector at `angle` rad from unit v, in a random direction."""
    w = np.cross(v, rng.normal(size=3))
    w /= np.linalg.norm(w)
    return _unit(np.cos(angle) * v + np.sin(angle) * w)


def _check(c1, c2, l1, l2):
    R = pose_oracle.rotation(c1, c2, l1, l2)
    assert R is not None
    Rs, s = _svd_rotation(c1, c2, l1, l2)
    bound = K * EPS / s[1]
    err = np.linalg.norm(R - Rs)
    assert err <= bound, (err, bound, s)
    ortho = 16.0 * EPS if s[1] >= 0.25 else max(16.0 * EPS, bound)
    assert np.abs(R.T @ R - np.eye(3)).max() <= ortho, (np.abs(R.T @ R - np.eye(3)).max(), s)
    assert abs(np.linalg.det(R) - 1.0) <= ortho
    # the pair in the other order: the same bits (IEEE subtraction is sign-symmetric, the two sign flips cancel)
    assert pose_oracle.rotation(c2, c1, l2, l1).tobytes() == R.tobytes()
    return R, Rs, s


def test_random_pairs_with_unequal_angles():
    """Noisy bearings: the camera and LiDAR angles differ, AB's singular values are distinct."""
    rng = np.random.default_rng(1)
    for _ in range(2000):
        l1, l2 = _unit(rng.normal(size=3)), _unit(rng.normal(size=3))
        Rt = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        Rt *= np.sign(np.linalg.det(Rt))
        c1, c2 = _unit(Rt @ l1 + rng.normal(0, 0.05, 3)), _unit(Rt @ l2 + rng.normal(0, 0.05, 3))
        R, Rs, s = _check(c1, c2, l1, l2)
        assert s[0] > s[1] * (1.0 + 1e-6)


def test_noise_free_pairs_recover_the_rotation():
    rng = np.random.default_rng(2)
    for _ in range(200):
        Rt = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        Rt *= np.sign(np.linalg.det(Rt))
        l1, l2 = _unit(rng.normal(size=3)), _unit(rng.normal(size=3))
        R, _, s = _check(Rt @ l1, Rt @ l2, l1, l2)
        assert np.abs(R - Rt).max() <= K * EPS / s[1]


def test_perpendicular_pairs():
    """90 degree pairs on both sides: |a| = |b| = |p| = |q| = sqrt(2), so sigma_1 = sigma_2 = 1."""
    rng = np.random.default_rng(3)
    for _ in range(500):
        c1, l1 = _unit(rng.normal(size=3)), _unit(rng.normal(size=3))
        c2, l2 = _at_angle(c1, np.pi / 2, rng), _at_angle(l1, np.pi / 2, rng)
        _, _, s = _check(c1, c2, l1, l2)
        assert abs(s[0] - s[1]) < 1e-14
    # axes: e0 -> e1, e1 -> e2
    e = np.eye(3)
    R, _, _ = _check(e[1], e[2], e[0], e[1])
    assert np.abs(R - np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])).max() <= 4 * EPS


@pytest.mark.parametrize("side", ["camera", "lidar", "both"])
@pytest.mark.parametrize("anti", [False, True], ids=["parallel", "antiparallel"])
def test_pairs_1e_8_rad_from_parallel(side, anti):
    """One (or both) pairs 1e-8 rad from parallel or antiparallel: |b| or |a| ~ 1e-8, still above the 1e-9 rad degenerate
    rule; the other side at a random angle.  sigma_2 ~ 1e-8 (1e-16 with both), the bound scales with it."""
    rng = np.random.default_rng(4 + 2 * ["camera", "lidar", "both"].index(side) + anti)
    angle = np.pi - 1e-8 if anti else 1e-8
    for _ in range(300):
        c1, l1 = _unit(rng.normal(size=3)), _unit(rng.normal(size=3))
        c2 = _at_angle(c1, angle, rng) if side in ("camera", "both") else _unit(rng.normal(size=3))
        l2 = _at_angle(l1, angle, rng) if side in ("lidar", "both") else _unit(rng.normal(size=3))
        _, _, s = _check(c1, c2, l1, l2)
        assert s[1] < (1e-15 if side == "both" else 1e-7)


def test_equal_singular_values():
    """|a||p| = |b||q| (the LiDAR angle the supplement of the camera angle): the SVD is not unique, U S V^T is."""
    rng = np.random.default_rng(5)
    for _ in range(500):
        theta = rng.uniform(0.1, np.pi - 0.1)
        c1, l1 = _unit(rng.normal(size=3)), _unit(rng.normal(size=3))
        c2, l2 = _at_angle(c1, theta, rng), _at_angle(l1, np.pi - theta, rng)
        _, _, s = _check(c1, c2, l1, l2)
        assert abs(s[0] - s[1]) < 1e-12


def test_degenerate_pairs_have_no_rotation():
    e = np.eye(3)
    assert pose_oracle.rotation(e[0], e[0], e[0], e[1]) is None  # b = 0
    assert pose_oracle.rotation(e[0], -e[0], e[0], e[1]) is None  # a = 0
    assert pose_oracle.rotation(e[0], e[1], e[2], e[2]) is None  # q = 0
    assert pose_oracle.rotation(e[0], e[1], e[2], -e[2]) is None  # p = 0
    assert pose_oracle.rotation(e[0], [np.nan, 0, 0], e[0], e[1]) is None
