"""The NID_BFGS solve on the GPU (vlcal_estimate_pose_bfgs_ctx: K3 per bag, summed in bag order, csrc/bfgs.cu) against
the same C solver driven by the oracle's functor.

The host reference is bfgs.minimize_se3 over a Python objective that culls every bag with oracle.view_cull at the start
pose, sums oracle.nid_cost_bspline_grad (NIDCost::operator()<Jet>) over the bags in bag order and is ok only if every bag
is ok -- ctx_objective with the oracle in place of K3.  Only the objective differs, so the two runs must take the same
decisions: the same iterations, evaluations and termination, every evaluated and every accepted pose within 1e-9, and
every cost within the sum of the bags' certified NID bounds (mode_b_reference.nid_bound) of the exact-sum NID."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import mode_b_reference as R
from direct_visual_lidar_calibration_b200 import bfgs
from direct_visual_lidar_calibration_b200 import synthetic as S

pytestmark = pytest.mark.gpu
ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED = -1, -6
POSE_TOL = 1e-9


def _bags(counts, double_layout=(), seed=12):
    """Bags of one 320x240 pinhole camera; bag b has counts[b] points, in the 32-byte double layout if b in double_layout."""
    out = []
    for b, n in enumerate(counts):
        bag = S.make_bag("pinhole_640x480", "frustum", n, config_index=seed, bag_index=b, scale=0.5)
        if b in double_layout:  # not float32-representable: K3 reads the double layout
            bag["points"] = bag["points"].copy()
            bag["points"][:, :3] *= 1.0 + 2.0**-40
        out.append(bag)
    return out


def _start(bags, rot=(0.3, -0.2, 0.25), trans=(0.01, -0.008, 0.006)):
    return S.perturb(bags[0]["T_gt"], rot, trans)


def _x7(T):
    return np.concatenate([Rotation.from_matrix(T[:3, :3]).as_quat(), T[:3, 3]])


def _same_pose(A, B, tol=POSE_TOL):
    d = np.linalg.inv(A) @ B
    return np.linalg.norm(d[:3, 3]) <= tol and np.linalg.norm(Rotation.from_matrix(d[:3, :3]).as_rotvec()) <= tol


def _same_x7(x, y, tol=POSE_TOL):
    if np.dot(x[:4], y[:4]) < 0:
        y = np.concatenate([-y[:4], y[4:]])
    return np.abs(x - y).max() <= tol


class OracleObjective:
    """ctx_objective on the oracle: cull each bag at T0, sum the Jet functor over the bags in bag order."""

    def __init__(self, O, bags, T0):
        b0 = bags[0]
        self.O = O
        self.cam = O.create_camera(b0["camera_model"], b0["intrinsics"], b0["distortion"])
        fov = O.estimate_camera_fov(self.cam, b0["width"], b0["height"])
        self.clouds = []
        for bag in bags:
            idx = O.view_cull(self.cam, b0["width"], b0["height"], fov, True, bag["points"], T0)  # :196
            self.clouds.append((bag["image"], bag["points"][idx], bag["intensities"][idx]))
        self.calls = []  # (x7, ok, cost)

    def __call__(self, x):
        total, g, ok = 0.0, np.zeros(7), True
        for image, pts, ins in self.clouds:
            okb, nid, gb = self.O.nid_cost_bspline_grad(self.cam, image, pts, ins, 16, x)
            ok = ok and okb
            total += nid
            g = g + gb
        self.calls.append((np.array(x), ok, total))
        return ok, total, g

    def exact(self, x):
        """(sum over the bags of the exact-sum NID at x, sum of the certified bounds on K3's NID there)."""
        nid, bound = 0.0, 0.0
        for image, pts, ins in self.clouds:
            ex = R.Exact(self.O, self.cam, image, pts, ins, 16, x)
            nid += float(ex.nid)
            bound += R.nid_bound(ex, R.fixed_bits(pts.shape[0]), R.PROJ_TOL["plumb_bob"])
        return nid, bound


class GpuObjective:
    """The same objective over the GPU NIDCost objects of the culled clouds, every evaluation recorded."""

    def __init__(self, V, bags, T0):
        b0 = bags[0]
        cam = V.create_camera(b0["camera_model"], b0["intrinsics"], b0["distortion"])
        culling = V.ViewCulling(cam, (b0["width"], b0["height"]))
        self.costs = []
        for bag in bags:
            pts, ins = culling.cull(bag["points"], bag["intensities"], T0)
            self.costs.append(V.NIDCost(cam, V.VisualLiDARData(bag["image"], pts, ins), 16))
        self.calls = []

    def __call__(self, x):
        total, g, ok = 0.0, np.zeros(7), True
        for c in self.costs:
            okb, nid, gb = c.evaluate_with_gradient(x)
            ok = ok and bool(okb[0])
            total += float(nid[0])
            g = g + gb[0]
        self.calls.append((np.array(x), ok, total))
        return ok, total, g


def _calibration(V, bags, bfgs_params=None):
    b0 = bags[0]
    cam = V.create_camera(b0["camera_model"], b0["intrinsics"], b0["distortion"])
    params = V.VisualCameraCalibrationParams()
    params.registration_type = V.RegistrationType.NID_BFGS
    params.bfgs_params = bfgs_params
    data = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    return V.VisualCameraCalibration(cam, data, params)


def _solve_three_ways(V, O, bags, T0, p=None):
    """(ctx run, GPU-objective run, oracle run), each (T, result, callback poses[, objective])."""
    calib = _calibration(V, bags, p)
    T_ctx, r_ctx = calib.estimate_pose_bfgs(T0)
    cb_ctx = [T for T, _ in calib.trace]
    gobj = GpuObjective(V, bags, T0)
    cb_gpu = []
    T_gpu, r_gpu = bfgs.minimize_se3(gobj, T0, p, callback=lambda T, c: cb_gpu.append(T))
    oobj = OracleObjective(O, bags, T0)
    cb_o = []
    T_o, r_o = bfgs.minimize_se3(oobj, T0, p, callback=lambda T, c: cb_o.append(T))
    return (T_ctx, r_ctx, cb_ctx), (T_gpu, r_gpu, cb_gpu, gobj), (T_o, r_o, cb_o, oobj)


def _check_same_solve(runs):
    (T_ctx, r_ctx, cb_ctx), (T_gpu, r_gpu, cb_gpu, gobj), (T_o, r_o, cb_o, oobj) = runs
    for r in (r_ctx, r_gpu):
        assert (r["iterations"], r["evaluations"], r["termination"]) == (r_o["iterations"], r_o["evaluations"], r_o["termination"]), (r, r_o)
    assert len(gobj.calls) == len(oobj.calls)
    for (xg, okg, cg), (xo, oko, co) in zip(gobj.calls, oobj.calls):
        assert _same_x7(xg, xo) and okg == oko
    for cb in (cb_ctx, cb_gpu):
        assert len(cb) == len(cb_o) == r_o["iterations"]
        assert all(_same_pose(a, b) for a, b in zip(cb, cb_o))
    assert _same_pose(T_ctx, T_o) and _same_pose(T_gpu, T_o)
    # every GPU cost within the certified bound of the exact-sum NID at its pose (invalid ones are not finite)
    worst = 0.0
    for k, (x, ok, c) in enumerate(gobj.calls):
        if not ok:
            continue
        exact, b = oobj.exact(x)
        assert abs(c - exact) <= b, (k, c, exact, b)
        worst = max(worst, b)
    assert abs(r_ctx["final_cost"] - r_o["final_cost"]) <= 2 * worst
    print(f"iterations {r_o['iterations']}  evaluations {r_o['evaluations']}  objective calls {len(oobj.calls)}  termination {r_o['termination']}  "
          f"largest cost bound {worst:.3g}")


def _params(max_iterations):
    p = bfgs.default_bfgs_params()
    p.max_num_iterations = max_iterations
    return p


@pytest.mark.parametrize("counts", [(40000,), (40000, 40000), (40000, 40000, 300)], ids=["1bag", "2bags", "3bags"])
def test_bfgs_solve_matches_the_oracle_driven_solve(gpu, oracle, counts):
    """1, 2 and 3 bags in bag order: the second in the double layout, the third a few hundred points."""
    bags = _bags(counts, double_layout=(1,))
    T0 = _start(bags)
    runs = _solve_three_ways(gpu, oracle, bags, T0, _params(12))
    _check_same_solve(runs)
    r_o = runs[2][1]
    assert r_o["iterations"] >= 2 and r_o["final_cost"] < r_o["initial_cost"]


def test_first_trial_step_leaves_the_trust_region(gpu, oracle):
    """A start whose first trial step leaves the 0.2 m / 2 deg region: the solver counts an evaluation it never passes to
    the objective, and the line search falls back inside the region the same way on both objectives."""
    bags = _bags((40000,), seed=13)
    T0 = _start(bags, rot=(0.6, -0.5, 0.4), trans=(0.05, -0.04, 0.03))
    runs = _solve_three_ways(gpu, oracle, bags, T0, _params(6))
    _check_same_solve(runs)
    r_o, oobj = runs[2][1], runs[2][3]
    assert r_o["evaluations"] > len(oobj.calls)


def _edge_bag(O, bag, n, seed=5):
    """n points of `bag`'s camera that project within 1.5 px of the right image edge at T_gt, with random intensities.
    Culling at T_gt keeps some of them; a solve from T_gt moves them out of the image at some trial poses."""
    rng = np.random.default_rng(seed)
    cam = O.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    W, H = bag["width"], bag["height"]
    targets = np.c_[W - rng.uniform(0.2, 1.5, n), rng.uniform(0.4 * H, 0.6 * H, n)]
    pts, _ = R.place_points(O, cam, R.sophus_params(bag["T_gt"]), targets, rng.uniform(4.0, 8.0, n))
    small = dict(bag)
    small["points"] = np.c_[pts, np.ones(n)]
    small["intensities"] = rng.uniform(0.0, 1.0, n)
    return small


def test_a_bag_leaving_the_image_mid_line_search(gpu, oracle):
    """A 5-point bag at the right image edge empties (NID not finite, functor false) at some trial poses of the first two
    line searches: those trials are invalid for the whole sum, on the GPU as on the oracle.

    Why two iterations and not more: at some trial poses this bag keeps one inlier whose 16 taps share one image bin.
    Then Hip = ln(1 + 1e-6) ~ 1e-6 and its NID is a difference of entropies of that size divided by Hip, so its certified
    bound (nid_bound) is 3.2e-4; K3 and the oracle differ there by up to 9.1e-7, inside it.  The line search interpolates
    those costs, so from the third iteration on the trial poses of the two runs drift apart by up to 4e-8.  That is the
    solver, not K3: a relative change of 1e-12 in the oracle's own cost and gradient moves them as far.  Over the first two
    iterations, relative changes of up to 1e-8 move no pose by more than 2.4e-10, so the 1e-9 pose tolerance holds."""
    base = _bags((40000,), seed=12)
    bags = base + [_edge_bag(oracle, base[0], 12)]
    runs = _solve_three_ways(gpu, oracle, bags, base[0]["T_gt"], _params(2))
    _check_same_solve(runs)
    oobj = runs[2][3]
    assert [c[1].shape[0] for c in oobj.clouds][1] == 5
    # ok = false mid-solve, between valid calls, inside a line search
    oks = [ok for _, ok, _ in oobj.calls]
    assert oks[0] and not all(oks) and any(not a and b for a, b in zip(oks, oks[1:])), oks


def test_invalid_start_is_a_failure(gpu, oracle):
    """No inlier in any bag at the start pose (every point projects far right of the image, so every NID is NaN):
    termination failure, T_out the start, no callback -- on the GPU ctx path as on the oracle."""
    bags = _bags((2000, 2000), seed=14)
    T0 = _start(bags)
    rng = np.random.default_rng(14)
    for b in bags:
        pc = np.c_[rng.uniform(50.0, 60.0, 2000), rng.uniform(-1.0, 1.0, 2000), rng.uniform(1.0, 2.0, 2000), np.ones(2000)]
        b["points"] = pc @ np.linalg.inv(T0).T  # camera points (x / z >= 25) in the LiDAR frame
    cam = gpu.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    costs = [gpu.NIDCost(cam, gpu.VisualLiDARData(b["image"], b["points"], b["intensities"]), 16) for b in bags]
    seen = []
    T, r = bfgs.estimate_pose_bfgs_on_costs(costs, T0, callback=lambda Tk, c: seen.append(Tk))
    assert r["termination"] == "failure" and np.array_equal(T, T0) and not seen and r["evaluations"] == 1
    ocam = oracle.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])

    def f(x):
        res = [oracle.nid_cost_bspline_grad(ocam, b["image"], b["points"], b["intensities"], 16, x) for b in bags]
        return all(o for o, _, _ in res), sum(c for _, c, _ in res), sum(g for _, _, g in res)

    seen_o = []
    T_o, r_o = bfgs.minimize_se3(f, T0, callback=lambda Tk, c: seen_o.append(Tk))
    assert (r_o["termination"], r_o["evaluations"], r_o["iterations"]) == (r["termination"], r["evaluations"], r["iterations"])
    assert np.array_equal(T_o, T0) and not seen_o


def _pull_back(x, g7):
    """g6 = J^T g7, J = d(x * exp(delta)) / d delta at 0 (bfgs.cu pull_back_gradient)."""
    qx, qy, qz, qw = x[:4]
    Rm = Rotation.from_quat(x[:4]).as_matrix()
    return np.concatenate([Rm.T @ g7[4:], 0.5 * np.array([qw * g7[0] + qz * g7[1] - qy * g7[2] - qx * g7[3],
                                                          -qz * g7[0] + qw * g7[1] + qx * g7[2] - qy * g7[3],
                                                          qy * g7[0] - qx * g7[1] + qw * g7[2] - qz * g7[3]])])


def test_zero_iterations_report_the_pulled_back_k3_gradient(gpu, oracle):
    bags = _bags((40000, 40000), double_layout=(1,))
    T0 = _start(bags)
    calib = _calibration(gpu, bags, _params(0))
    T, r = calib.estimate_pose_bfgs(T0)
    assert r["iterations"] == 0 and r["evaluations"] == 1 and r["termination"] == "no_convergence" and _same_pose(T, T0, 1e-14)
    gobj = GpuObjective(gpu, bags, T0)
    x = _x7(T0)
    ok, _, g7 = gobj(x)
    assert ok
    g6 = _pull_back(x, g7)
    assert abs(r["gradient_max_norm"] - np.abs(g6).max()) <= 1e-9 * np.abs(g6).max(), (r["gradient_max_norm"], np.abs(g6).max())
    _, _, go = OracleObjective(oracle, bags, T0)(x)
    assert abs(r["gradient_max_norm"] - np.abs(_pull_back(x, go)).max()) <= 1e-8 * max(1.0, np.abs(g6).max())


def test_unusable_contexts_raise_and_return_no_pose(gpu):
    """A 57-bin context among 16-bin ones (K3 refuses it: ERR_UNSUPPORTED, propagated out of the solve) and a mode-A
    context (ERR_INVALID_ARGUMENT): the solve raises, no callback runs."""
    bags = _bags((2000, 2000), seed=15)
    T0 = _start(bags)
    b0 = bags[0]
    cam = gpu.create_camera(b0["camera_model"], b0["intrinsics"], b0["distortion"])
    data = [gpu.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    seen = []
    for costs, code in (
        ([gpu.NIDCost(cam, data[0], 16), gpu.NIDCost(cam, data[1], 57), gpu.NIDCost(cam, data[0], 16)], ERR_UNSUPPORTED),
        ([gpu.NIDCost(cam, data[0], 16), gpu.CostCalculatorNID(cam, data[1])], ERR_INVALID_ARGUMENT),
    ):
        with pytest.raises(gpu.VlcalError) as e:
            bfgs.estimate_pose_bfgs_on_costs(costs, T0, callback=lambda Tk, c: seen.append(Tk))
        assert e.value.code == code
    assert not seen


def test_calibrate_matches_the_oracle_pipeline(gpu, oracle):
    """calibrate() with NID_BFGS on two bags against the oracle pipeline: per outer iteration cull at the current pose,
    minimise the oracle objective, stop on the reference's rule (orc_rotation_angle of the isometry delta).  The same
    number of outer iterations, the same pose after each within 1e-9."""
    bags = _bags((30000, 30000), seed=16)
    T0 = _start(bags, rot=(0.5, -0.4, 0.3), trans=(0.04, -0.03, 0.02))
    p = _params(8)
    calib = _calibration(gpu, bags, p)
    calib.params.max_outer_iterations = 4
    outer = []
    inner = calib.estimate_pose_bfgs

    def record(T):
        Tn, r = inner(T)
        outer.append(Tn)
        return Tn, r

    calib.estimate_pose_bfgs = record
    T_gpu = calib.calibrate(T0)
    T, ref = T0, []
    for _ in range(calib.params.max_outer_iterations):
        T_new, _ = bfgs.minimize_se3(OracleObjective(oracle, bags, T), T, p)
        ref.append(T_new)
        dt, dr = oracle.outer_step_delta(T, T_new)
        T = T_new
        if dt < calib.params.delta_trans_thresh and dr < calib.params.delta_rot_thresh:
            break
    assert calib.stats["outer_iterations"] == len(ref) == len(outer)
    assert all(_same_pose(a, b) for a, b in zip(outer, ref))
    assert _same_pose(T_gpu, T)
    print(f"outer iterations {len(ref)}")
