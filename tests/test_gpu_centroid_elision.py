"""GPU checks of the centroid elision of the Nelder-Mead inner solve (csrc/nm_machine.cuh, run_inner_solve in
csrc/calibration.cu): without an observer of the objective's side effects -- no best-cost callback, no recorded solve
trace, no all-reduce -- every iteration batch scores {xr, xe, xc} instead of {xo, xr, xe, xc}.  The solve must not change:
same pose, simplex result, iterations, reference evaluations and batches as with the centroid scored, one pose fewer per
iteration batch, the host loop (solver mode 1) and the persistent kernel (mode 3) identical batch for batch, and any
observer brings the centroid back with the reference's callback sequence."""
import math

import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import calibration as _VC
from direct_visual_lidar_calibration_b200 import synthetic as _S

pytestmark = pytest.mark.gpu
NID_TOL = 1e-12
ITERS = 40


@pytest.fixture(scope="module", params=["equirectangular", "plumb_bob"])
def problem(request, gpu, oracle):
    """A small bag, culled at the start pose as the solve culls it, its cost object and the oracle's solve from there."""
    V, O = gpu, oracle
    model = request.param
    pr = util.random_problem(model, n=12_000, seed=830)
    cam_args = (pr["model"], pr["intrinsics"], pr["distortion"])
    T0 = _S.perturb(pr["T"], (0.3, -0.2, 0.3), (0.01, 0.0, -0.01))
    ocam = O.create_camera(*cam_args)
    idx = O.view_cull(ocam, pr["W"], pr["H"], O.estimate_camera_fov(ocam, pr["W"], pr["H"]), True, pr["points"], T0)
    cam = V.create_camera(*cam_args)
    cost = V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"][idx], pr["intensities"][idx]), V.NIDCostParams(16))
    op = O.default_calib_params()
    op.max_inner_iterations = ITERS
    ref = O.estimate_pose_nelder_mead(ocam, [(pr["image"], pr["points"], pr["intensities"])], T0, op)
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = ITERS
    yield V, cost, T0, params, ref
    cost.close()


def _solve(V, cost, T0, params, mode, record=False, **kw):
    """One solve in solver mode `mode`; returns (T, result, poses the cost object scored, recorded trace or None)."""
    try:
        V.set_solver_mode(mode)
        if record:
            _VC.record_solve_trace(True)
        cost.reset_profile()
        T, r = _VC.estimate_pose_on_costs([cost], T0, params, **kw)
        poses = cost.profile()["poses_total"]
        trace = _VC.last_solve_trace() if record else None
    finally:
        V.set_solver_mode(0)
        _VC.record_solve_trace(False)
    return T, r, poses, trace


def _iteration_batches(r):
    """Iteration batches of a solve that scored the centroid: 7 poses for the initial simplex, 4 per iteration and 6 per
    shrink, in num_batches = 1 + iterations + shrinks batches."""
    twice = 6 * (r["num_batches"] - 1) + 7 - r["num_evaluations_computed"]
    assert twice >= 0 and twice % 2 == 0, r
    return twice // 2


def _assert_same_trajectory(a, b):
    (Ta, ra), (Tb, rb) = a, b
    assert np.array_equal(Ta, Tb) and np.array_equal(ra["x"], rb["x"])
    assert ra["y"] == rb["y"] or (math.isnan(ra["y"]) and math.isnan(rb["y"]))
    for k in ("converged", "num_iterations", "num_evaluations", "num_batches"):
        assert ra[k] == rb[k], (k, ra[k], rb[k])


def _prefix_minima(costs):
    out, best = [], math.inf
    for c in costs:
        if c < best:
            best = c
            out.append(c)
    return out


@pytest.mark.parametrize("mode", [1, 3])
def test_elided_solve_follows_the_scored_one(problem, mode):
    V, cost, T0, params, ref = problem
    T_s, r_s, poses_s, trace = _solve(V, cost, T0, params, mode, record=True)
    T_e, r_e, poses_e, _ = _solve(V, cost, T0, params, mode)
    _assert_same_trajectory((T_s, r_s), (T_e, r_e))
    iteration_batches = _iteration_batches(r_s)
    assert iteration_batches > 5, r_s
    assert r_s["num_evaluations_computed"] - r_e["num_evaluations_computed"] == iteration_batches
    assert poses_s == r_s["num_evaluations_computed"] and poses_e == r_e["num_evaluations_computed"]
    # both follow the oracle; the recorded trace (centroids included) is the oracle's evaluation sequence
    assert np.array_equal(r_e["x"], ref["x"]) and r_e["num_evaluations"] == ref["num_evaluations"] and np.abs(T_e - ref["T"]).max() == 0.0
    assert trace.shape == ref["trace"].shape and np.array_equal(trace[:, :6], ref["trace"][:, :6])


def test_host_loop_and_persistent_kernel_agree_with_the_centroid_elided(problem):
    V, cost, T0, params, _ = problem
    T1, r1, poses1, _ = _solve(V, cost, T0, params, 1)
    T3, r3, poses3, _ = _solve(V, cost, T0, params, 3)
    _assert_same_trajectory((T1, r1), (T3, r3))
    assert r1["num_evaluations_computed"] == r3["num_evaluations_computed"] == poses1 == poses3


# a host all-reduce runs on the host loop only (the persistent kernel sums over ranks through a peer exchange)
@pytest.mark.parametrize("observer,mode", [("callback", 1), ("callback", 3), ("allreduce", 1)])
def test_an_observer_brings_the_centroid_back(problem, observer, mode):
    V, cost, T0, params, ref = problem
    T_s, r_s, _, _ = _solve(V, cost, T0, params, mode, record=True)
    seen, reduced = [], [0]

    def callback(T, c):
        seen.append(c)

    def allreduce(vals):  # a world of one rank: the sum over ranks is the value itself
        reduced[0] += 1

    kw = {"callback": callback} if observer == "callback" else {"allreduce": allreduce}
    T, r, poses, _ = _solve(V, cost, T0, params, mode, **kw)
    _assert_same_trajectory((T_s, r_s), (T, r))
    assert r["num_evaluations_computed"] == r_s["num_evaluations_computed"] == poses
    if observer == "callback":
        want = _prefix_minima(ref["trace"][:, 6])
        assert len(seen) == len(want) and np.all(np.abs(np.asarray(seen) - np.asarray(want)) < NID_TOL), (seen, want)
    else:
        assert reduced[0] == r["num_batches"]
