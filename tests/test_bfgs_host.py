"""Host-side BFGS on SE(3) (csrc/bfgs.cu) with Python objectives -- no GPU needed.  The reference's solver for this branch
is Ceres (absent here), so these are properties of OUR solver: it minimises, respects the reference's trust region around
the start pose (visual_camera_calibration.cpp:152-156), pulls gradients back to the tangent space correctly."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import direct_visual_lidar_calibration_b200 as V
from direct_visual_lidar_calibration_b200 import bfgs
from direct_visual_lidar_calibration_b200.calibration import outer_step_delta


def make_T(rotvec, t):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(rotvec).as_matrix()
    T[:3, 3] = t
    return T


def quadratic_objective(T_target, weight_t=1.0):
    """0.5 |q - q*|^2 (sign-aligned) + 0.5 w |t - t*|^2 in ambient coordinates: smooth, minimum at T_target."""
    q_t = Rotation.from_matrix(T_target[:3, :3]).as_quat()
    t_t = T_target[:3, 3]
    calls = []

    def f(x):
        q, t = x[:4], x[4:]
        qt = q_t if np.dot(q, q_t) >= 0 else -q_t
        cost = 0.5 * np.sum((q - qt) ** 2) + 0.5 * weight_t * np.sum((t - t_t) ** 2)
        grad = np.concatenate([q - qt, weight_t * (t - t_t)])
        calls.append(cost)
        return True, cost, grad

    return f, calls


def pose_error(A, B):
    d = np.linalg.inv(A) @ B
    return np.linalg.norm(d[:3, 3]), np.linalg.norm(Rotation.from_matrix(d[:3, :3]).as_rotvec())


def test_converges_to_the_minimiser():
    T0 = make_T([0.3, -0.2, 0.5], [1.0, 2.0, -0.5])
    T_star = T0 @ make_T([0.01, -0.015, 0.02], [0.03, -0.05, 0.04])
    f, calls = quadratic_objective(T_star, weight_t=3.0)
    seen = []
    T, r = bfgs.minimize_se3(f, T0, callback=lambda Tk, c: seen.append(c))
    dt, dr = pose_error(T, T_star)
    assert dt < 1e-5 and dr < 1e-5, (dt, dr, r)
    assert r["final_cost"] < 1e-10 and r["final_cost"] <= r["initial_cost"]
    assert r["iterations"] == len(seen) and r["evaluations"] >= len(calls)  # trial poses outside the trust region are not evaluated
    assert all(b <= a + 1e-15 for a, b in zip(seen, seen[1:]))  # accepted iterates never increase the cost
    assert r["termination"] in ("function_tolerance", "gradient_tolerance", "parameter_tolerance")
    # a handful of iterations: quasi-Newton, not gradient descent
    assert r["iterations"] <= 25


def test_respects_the_trust_region_around_the_start_pose():
    """MultiNIDCost returns false beyond 0.2 m / 2 deg from the start pose: the solver must stay inside."""
    T0 = make_T([0.1, 0.2, -0.1], [0.5, 0.5, 0.5])
    T_star = T0 @ make_T([0.2, 0.0, 0.0], [1.0, 0.0, 0.0])  # far outside
    f, _ = quadratic_objective(T_star)
    T, r = bfgs.minimize_se3(f, T0)
    dt, dr = pose_error(T0, T)
    assert dt <= 0.2 + 1e-12 and dr <= np.deg2rad(2.0) + 1e-12
    assert r["final_cost"] < r["initial_cost"]
    p = bfgs.default_bfgs_params()
    p.max_translation_from_init, p.max_rotation_from_init = 0.01, np.deg2rad(0.1)
    T, r = bfgs.minimize_se3(f, T0, p)
    dt, dr = pose_error(T0, T)
    assert dt <= 0.01 + 1e-12 and dr <= np.deg2rad(0.1) + 1e-12


def test_invalid_start_is_reported_not_hidden():
    T0 = make_T([0, 0, 0], [0, 0, 0])
    T, r = bfgs.minimize_se3(lambda x: (False, 0.0, np.zeros(7)), T0)
    assert r["termination"] == "failure" and np.allclose(T, T0)
    assert r["evaluations"] == 1 and r["iterations"] == 0  # the start pose was evaluated once


def test_objective_invalid_in_a_region():
    """Invalid evaluations inside the line search (a bag's functor returning false) only shorten the step."""
    T0 = make_T([0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
    T_star = T0 @ make_T([0.0, 0.01, 0.0], [0.1, 0.0, 0.0])
    base, _ = quadratic_objective(T_star)

    def f(x):
        ok, c, g = base(x)
        return (x[4] < 0.05), c, g  # a wall at tx = 0.05, before the minimiser at 0.1

    T, r = bfgs.minimize_se3(f, T0)
    assert T[0, 3] < 0.05 and T[0, 3] > 0.02 and r["final_cost"] < r["initial_cost"]


def test_tangent_pull_back_matches_finite_differences():
    """One steepest-descent step is along -J^T g: with max_num_iterations = 1 and a tiny fixed step the decrease must match
    the directional derivative predicted by the ambient gradient."""
    rng = np.random.default_rng(3)
    T0 = make_T(rng.normal(size=3) * 0.4, rng.normal(size=3))
    A = rng.normal(size=(7, 7))
    A = A @ A.T + np.eye(7)
    x_ref = np.concatenate([Rotation.from_matrix(T0[:3, :3]).as_quat(), T0[:3, 3]]) + 0.05 * rng.normal(size=7)

    def f(x):
        if np.dot(x[:4], x_ref[:4]) < 0:
            x = np.concatenate([-x[:4], x[4:]])
        e = x - x_ref
        return True, 0.5 * e @ A @ e, A @ e

    p = bfgs.default_bfgs_params()
    p.max_num_iterations = 1
    T, r = bfgs.minimize_se3(f, T0, p)
    assert r["iterations"] == 1 and r["final_cost"] < r["initial_cost"]
    # the accepted step satisfies the Armijo condition with the solver's own slope: check it against a numerical slope
    x0 = np.concatenate([Rotation.from_matrix(T0[:3, :3]).as_quat(), T0[:3, 3]])
    x1 = np.concatenate([Rotation.from_matrix(T[:3, :3]).as_quat(), T[:3, 3]])
    if np.dot(x0[:4], x1[:4]) < 0:
        x1[:4] = -x1[:4]
    _, c0, g0 = f(x0)
    lin = g0 @ (x1 - x0)
    assert lin < 0  # moved downhill to first order in ambient coordinates too


def test_registration_type_enum_and_params():
    p = V.VisualCameraCalibrationParams()
    assert p.registration_type == V.RegistrationType.NID_NELDER_MEAD and p.bfgs_params is None
    d = bfgs.default_bfgs_params()
    assert d.max_num_iterations == 50 and d.function_tolerance == 1e-6 and d.gradient_tolerance == 1e-10 and d.parameter_tolerance == 1e-8
    assert d.max_translation_from_init == 0.2 and abs(d.max_rotation_from_init - np.deg2rad(2.0)) < 1e-15


def _steps_at_the_threshold(O, T0, w, v, component, thresh, ulps=4):
    """Outer-loop results new_T(s) = T0 * Expmap(s w, s v) whose oracle step (delta_t if component == 0, delta_r if 1)
    straddles `thresh`: bisection over s down to adjacent doubles, then the first s that reaches the threshold and
    `ulps` doubles either side of it."""
    def new_T(s):
        return O.isometry_mul(T0, O.se3_expmap(np.concatenate([s * np.asarray(w), s * np.asarray(v)])))

    lo, hi = 0.0, 1.0
    assert O.outer_step_delta(T0, new_T(lo))[component] < thresh <= O.outer_step_delta(T0, new_T(hi))[component]
    while np.nextafter(lo, hi) != hi:
        mid = 0.5 * (lo + hi)
        if mid in (lo, hi):
            mid = np.nextafter(lo, hi)
        if O.outer_step_delta(T0, new_T(mid))[component] < thresh:
            lo = mid
        else:
            hi = mid
    ss = [hi]
    for _ in range(ulps):
        ss = [np.nextafter(ss[0], -np.inf)] + ss + [np.nextafter(ss[-1], np.inf)]
    return [new_T(s) for s in ss]


@pytest.mark.parametrize("component", ["translation", "rotation"])
def test_bfgs_outer_loop_stops_on_the_reference_rule(oracle, component):
    """The NID_BFGS outer loop (visual_camera_calibration.cpp:35-68) stops when delta = new_T^-1 * T, as isometries, has
    |translation| < delta_trans_thresh and AngleAxisd angle < delta_rot_thresh.  The inner solve is replaced by a stub
    returning chosen poses placed at each threshold to the ulp, so the decision and the outer-iteration count must be
    the oracle rule's bit for bit: a general 4x4 inverse, np.linalg.norm or arccos of the trace would stop on a
    different outer iteration for some of these poses."""
    params = V.VisualCameraCalibrationParams()
    params.registration_type = V.RegistrationType.NID_BFGS
    T0 = make_T([0.3, -0.2, 0.5], [1.0, 2.0, -0.5])
    if component == "translation":  # rotation of the step well inside its threshold, translation at 0.1 m
        w, v, k, thresh = [0.01, -0.02, 0.015], [0.6, -0.5, 0.7], 0, params.delta_trans_thresh
    else:  # translation well inside, rotation at 0.5 deg
        w, v, k, thresh = [0.6, -0.5, 0.7], [0.8, 0.5, -0.6], 1, params.delta_rot_thresh
    decisions, general_rule_differs = [], False
    for new_T in _steps_at_the_threshold(oracle, T0, w, v, k, thresh):
        dt, dr = oracle.outer_step_delta(T0, new_T)
        assert outer_step_delta(T0, new_T) == (dt, dr)
        stop = dt < params.delta_trans_thresh and dr < params.delta_rot_thresh
        decisions.append(stop)
        # the general-matrix rule this loop must not use: it decides at least one of these poses differently
        d = np.linalg.inv(new_T) @ T0
        g_dt, g_dr = np.linalg.norm(d[:3, 3]), np.arccos(np.clip(0.5 * (np.trace(d[:3, :3]) - 1.0), -1.0, 1.0))
        general_rule_differs |= (g_dt < params.delta_trans_thresh and g_dr < params.delta_rot_thresh) != stop
        # the stub's second solve returns its start pose: delta 0, the loop stops there at the latest
        calls = []

        def stub(T, _new_T=new_T):
            calls.append(np.array(T))
            return (_new_T if len(calls) == 1 else np.array(T)), {"evaluations": 1}

        calib = V.VisualCameraCalibration(None, [], params)
        calib.estimate_pose_bfgs = stub
        T = calib.calibrate(T0)
        assert calib.stats["outer_iterations"] == (1 if stop else 2), (component, dt, dr)
        assert np.array_equal(T, new_T) and np.array_equal(calls[0], T0)
    assert True in decisions and False in decisions  # the poses straddle the threshold
    assert general_rule_differs  # so the stub loop above fails on the old rule for this component


BFGS_WORKER = r"""
import os, sys, numpy as np, torch, torch.distributed as dist
from scipy.spatial.transform import Rotation
sys.path.insert(0, sys.argv[1])
import direct_visual_lidar_calibration_b200 as V
from direct_visual_lidar_calibration_b200 import bfgs
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dist.init_process_group("gloo", rank=rank, world_size=world)
# bag-sharded BFGS: each rank owns one term of the objective; value, the 7 partials and the failure count are summed over
# the ranks at every evaluation (the 9-double all-reduce of vlcal_estimate_pose_bfgs_ctx), so all ranks take the same steps.
def make_T(rv, t):
    T = np.eye(4); T[:3, :3] = Rotation.from_rotvec(rv).as_matrix(); T[:3, 3] = t; return T
T0 = make_T([0.2, -0.1, 0.3], [0.5, -0.2, 1.0])
targets = [T0 @ make_T([0.01, 0.0, -0.01], [0.02, 0.01, 0.0]), T0 @ make_T([-0.005, 0.01, 0.0], [0.0, -0.02, 0.03])]
def term(r, x):
    qt = Rotation.from_matrix(targets[r][:3, :3]).as_quat(); tt = targets[r][:3, 3]
    if np.dot(x[:4], qt) < 0: qt = -qt
    e = np.concatenate([x[:4] - qt, (r + 1.0) * (x[4:] - tt)])
    return 0.5 * float(e @ e), np.concatenate([x[:4] - qt, (r + 1.0) ** 2 * (x[4:] - tt)])
def sharded(x):
    c, g = term(rank, x)
    t = torch.from_numpy(np.concatenate([[c], g, [0.0]]))
    dist.all_reduce(t)
    v = t.numpy()
    return v[8] == 0.0, v[0], v[1:8]
T, r = bfgs.minimize_se3(sharded, T0)
out = torch.from_numpy(np.concatenate([T.reshape(-1), [r["final_cost"], r["iterations"], r["evaluations"]]]))
gathered = [torch.zeros_like(out) for _ in range(world)]
dist.all_gather(gathered, out)
if rank == 0:
    assert all(torch.equal(g, gathered[0]) for g in gathered), "ranks diverged"
    def joint(x):
        cs = [term(k, x) for k in range(world)]
        return True, sum(c for c, _ in cs), sum(g for _, g in cs)
    T1, r1 = bfgs.minimize_se3(joint, T0)
    assert np.allclose(T1, T, atol=1e-12) and r1["iterations"] == r["iterations"] and r["final_cost"] < r["initial_cost"]
    print("GLOO_BFGS_OK", r["iterations"], r["final_cost"])
dist.destroy_process_group()
"""


def test_bag_sharded_bfgs_over_gloo_world_size_2(tmp_path):
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "bfgs_worker.py"
    script.write_text(BFGS_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29537", WORLD_SIZE="2", OMP_NUM_THREADS="1")
    procs = [subprocess.Popen([sys.executable, str(script), root], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=240)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert "GLOO_BFGS_OK" in outs[0]


def test_bfgs_on_the_oracle_mode_b_objective():
    """The whole NID_BFGS branch on the CPU: our solver driving the ORACLE's NIDCost<Jet> (value + 7 partials), on a small
    synthetic bag.  Checks the interplay the GPU path relies on: ambient gradient -> tangent pull-back -> descent."""
    import util as U
    from direct_visual_lidar_calibration_b200 import synthetic as S
    from oracle import oracle as O

    bag = S.make_bag("pinhole_640x480", "frustum", 6000, config_index=12, scale=0.5)
    cam = O.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    T0 = S.perturb(bag["T_gt"], (0.25, -0.2, 0.2), (0.008, -0.006, 0.005))
    fov = O.estimate_camera_fov(cam, bag["width"], bag["height"])
    idx = O.view_cull(cam, bag["width"], bag["height"], fov, True, bag["points"], T0)  # :196 cull at the start pose
    pts, ins = bag["points"][idx], bag["intensities"][idx]
    evals = []

    def f(x):
        ok, nid, grad = O.nid_cost_bspline_grad(cam, bag["image"], pts, ins, 16, x)
        evals.append(nid)
        return ok, nid, grad

    p = bfgs.default_bfgs_params()
    p.max_num_iterations = 12
    seen = []
    T, r = bfgs.minimize_se3(f, T0, p, callback=lambda Tk, c: seen.append(c))
    assert r["iterations"] >= 2 and r["final_cost"] < r["initial_cost"] - 1e-4, r
    assert seen == sorted(seen, reverse=True) and abs(seen[-1] - r["final_cost"]) < 1e-15
    # the reported costs are the functor's values at the reported poses
    q = np.concatenate([Rotation.from_matrix(T[:3, :3]).as_quat(), T[:3, 3]])
    ok, c1, _ = O.nid_cost_bspline_grad(cam, bag["image"], pts, ins, 16, q)
    assert ok and (abs(c1 - r["final_cost"]) < 1e-9)
    dt, dr = pose_error(T0, T)
    assert dt <= 0.2 and dr <= np.deg2rad(2.0)
