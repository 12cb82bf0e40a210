"""Host-side checks of `assess`: the pose stencils and the finite differences built on them, the warning logic on
synthetic inputs, the report's JSON shape, and the exported C-ABI entry point of the solve axis.  No GPU needed."""
import ctypes
import json
import math

import numpy as np
import pytest

from direct_visual_lidar_calibration_b200 import assess as A
from direct_visual_lidar_calibration_b200 import load_library
from direct_visual_lidar_calibration_b200.calibration import se3_expmap


def _quadratic(Hq, g):
    return lambda x: 0.5 * x @ Hq @ x + g @ x + 0.25


def test_stencil_shape_and_order():
    h = A.HESSIAN_STEP
    st = A.hessian_stencil(h)
    assert st.shape == (73, 6)
    assert np.all(st[0] == 0.0)
    for i in range(6):
        assert st[1 + 2 * i][i] == h[i] and st[2 + 2 * i][i] == -h[i]
        assert np.count_nonzero(st[1 + 2 * i]) == 1
    assert all(np.count_nonzero(r) == 2 for r in st[13:])
    assert len({tuple(r) for r in st}) == 73


@pytest.mark.parametrize("scale", [1.0, 2.0])
def test_finite_difference_hessian_of_a_quadratic_is_exact(scale):
    rng = np.random.default_rng(3)
    M = rng.normal(size=(6, 6))
    Hq = M @ M.T + np.diag([1e3, 2e3, 3e3, 4e2, 5e2, 6e2])
    f = _quadratic(Hq, rng.normal(size=6))
    h = scale * A.HESSIAN_STEP
    H = A.hessian_from_stencil([f(x) for x in A.hessian_stencil(h)], h)
    np.testing.assert_allclose(H, Hq, rtol=1e-6, atol=1e-6 * np.abs(Hq).max())


def test_profiles_span_the_stated_ranges():
    off = A.profile_offsets(41)
    assert off.shape == (6, 41, 6)
    for k in range(6):
        assert off[k, 0, k] == -A.PROFILE_HALF[k] and off[k, -1, k] == A.PROFILE_HALF[k] and off[k, 20, k] == 0.0
        assert np.count_nonzero(np.delete(off[k], k, axis=1)) == 0
    assert math.isclose(A.PROFILE_HALF[0], math.radians(2.0)) and A.PROFILE_HALF[3] == 0.10


def test_tangent_poses_follow_calibrates_parameterisation():
    rng = np.random.default_rng(1)
    T = se3_expmap(rng.normal(size=6) * 0.3)
    xs = rng.normal(size=(5, 6)) * 0.01
    P = A.tangent_poses(T, xs)
    for x, U in zip(xs, P):
        np.testing.assert_array_equal(U, T @ se3_expmap(x))  # init_T * Expmap(x), as the Nelder-Mead objective forms it
    # the first three coordinates rotate, the last three translate along the rotated axes
    U = A.tangent_poses(T, [[0, 0, 0, 0.01, 0, 0]])[0]
    dt, dr = A.pose_distance(T, U)
    assert math.isclose(dt, 0.01, rel_tol=1e-12) and dr < 1e-9
    U = A.tangent_poses(T, [[0, 0, math.radians(0.5), 0, 0, 0]])[0]
    dt, dr = A.pose_distance(T, U)
    assert dt < 1e-12 and math.isclose(dr, 0.5, rel_tol=1e-9)


def test_profile_width():
    s = np.linspace(-1, 1, 21)
    f = 0.5 + 0.01 * s**2
    w = A.profile_width(s, f, 0.5, rise=1e-3)
    assert math.isclose(w, 0.8)  # 0.01 s^2 >= 1e-3 first at |s| = 0.4 on either side
    assert A.profile_width(s, np.full(21, 0.5), 0.5) is None


def test_weak_axes_compare_within_a_kind():
    assert A.weak_axes([100, 90, 95, 1e4, 2e4, 1.5e4]) == []  # translations far above rotations: not weak
    assert A.weak_axes([100, 5, 95, 1e4, 2e4, 1.5e3]) == [1, 5]
    assert A.weak_axes([100, 90, -1, 1e4, 2e4, 1.5e4]) == [2]


def test_step_disagreement():
    assert A.disagreeing_axes([1, 1, 1, 1, 1, 1], [1.5, 0.6, 1, 1, 1, 1]) == []
    assert A.disagreeing_axes([1, 1, 1, 1, 1, 1], [2.5, 1, 1, 1, 0.4, -1]) == [0, 4, 5]


def test_solve_summary_warnings():
    T = np.eye(4)
    starts = A.random_starts(T, 4, 1.0, 0.05, seed=0)
    for S in starts:
        dt, dr = A.pose_distance(T, S)
        # Exp couples the translation with the rotation (its V matrix): the length is 0.05 to first order
        assert math.isclose(dt, 0.05, rel_tol=1e-4) and math.isclose(dr, 1.0, rel_tol=1e-9)
    near = A.tangent_poses(T, [[0, 0, 0, 0.001, 0, 0]] * 3 + [[0, 0, 0, 0, 0.02, 0]])
    ys = [0.5, 0.49, 0.5, 0.45]
    names = ["a", "b", "c", "d", "e"]
    loo = A.tangent_poses(T, [[0, 0, 0, 0.001, 0, 0], [0, 0, 0, 0, 0.0012, 0], [0, 0, 0, 0.03, 0, 0], [0, 0, 0, 0, 0, 0.0009], [0.0001, 0, 0, 0, 0, 0]])
    summary, records, warnings = A.summarize_solves(T, 0.5, starts, near, ys, [10, 11, 12, 13], names, loo)
    assert summary["ended_away"] == 1 and summary["lower_nid"] == 2
    assert math.isclose(summary["max_trans"], 0.02)
    assert len(records) == 4 and records[3]["iterations"] == 13
    # start 1: lower NID but within tolerance of T (the same optimum); start 3: lower and away -> a missed optimum
    assert len([w for w in warnings if "better optimum" in w]) == 1 and "solve 3" in warnings[0]
    outl = [w for w in warnings if "outlier" in w]
    assert len(outl) == 1 and "bag c" in outl[0]
    # every bag a little off, none beyond the tolerance: no outlier however uneven
    loo_small = A.tangent_poses(T, [[0, 0, 0, 1e-5, 0, 0], [0, 0, 0, 1e-5, 0, 0], [0, 0, 0, 4e-3, 0, 0]])
    _, _, w2 = A.summarize_solves(T, 0.5, [], [], [], [], names[:3], loo_small)
    assert w2 == []


def test_local_shape_report_is_json():
    steps = 11
    Hq = np.diag([4e3, 3e3, 2e1, 3e3, 2e3, 2.5e3])
    f = _quadratic(Hq, np.zeros(6))
    prof = np.array([[f(x) for x in row] for row in A.profile_offsets(steps)])
    fh = np.array([f(x) for x in A.hessian_stencil(A.HESSIAN_STEP)])
    f2h = np.array([f(x) for x in A.hessian_stencil(2 * A.HESSIAN_STEP)])
    r = A.local_shape(prof, fh, f2h, steps)
    json.loads(json.dumps(r))
    assert r["weak_axes"] == ["rz"] and r["step_disagreement_axes"] == []
    np.testing.assert_allclose(r["curvature"], np.diag(Hq), rtol=1e-6)
    assert len(r["eigenvalues"]) == 6 and len(r["profiles"]) == 6 and len(r["profiles"][0]["nid"]) == steps


def test_solve_axis_symbol_is_exported():
    L = load_library()
    assert isinstance(L.vlcal_estimate_poses_nelder_mead_ctx, ctypes._CFuncPtr)
    with open(__file__.replace("tests/test_assess_host.py", "include/vlcal_nid.h")) as fh:
        assert "int vlcal_estimate_poses_nelder_mead_ctx(" in fh.read()


def test_oracle_histogram_pmi_weighted_by_counts_is_the_mutual_information():
    """The agreement map's PMI per joint bin, log(c_ab N / (c_a c_b)), weighted by the counts, sums to the mutual information
    of the oracle's histogram; and NID = (H_ab - MI) / H_ab reproduces the oracle's NID up to the reference's 1e-6 inside
    its logarithms."""
    import util
    from oracle import oracle as O

    pr = util.random_problem("plumb_bob", n=20000, seed=9)
    cam = O.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    nid, hist = O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], 16, O.estimate_camera_fov(cam, pr["W"], pr["H"]), pr["T"])
    h = np.asarray(hist, dtype=np.float64)
    N = h.sum()
    ca, cb = h.sum(axis=1), h.sum(axis=0)
    nz = h > 0
    pmi = np.log((h * N) / np.outer(ca, cb), where=nz, out=np.zeros_like(h))
    mi_from_pmi = (h[nz] * pmi[nz]).sum() / N
    p, pa, pb = h[nz] / N, ca[ca > 0] / N, cb[cb > 0] / N
    H_ab, H_a, H_b = -(p * np.log(p)).sum(), -(pa * np.log(pa)).sum(), -(pb * np.log(pb)).sum()
    assert abs(mi_from_pmi - (H_a + H_b - H_ab)) < 1e-12
    assert abs((H_ab - mi_from_pmi) / H_ab - nid) < 1e-4
