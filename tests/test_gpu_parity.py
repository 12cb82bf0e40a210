"""GPU suite (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle and the committed golden
fixtures.  Bar: integer histograms bit-exact (0 differing counts); NID within 1e-12 of the oracle (the required
tolerance of BASELINE.json's north_star is 1e-6) -- the only non-identical arithmetic is log() in the entropy tail
(CUDA libdevice vs glibc, <= 1 ulp each) and the fixed-tree summation order."""
import math
import os

import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import synthetic as _S

util.S = _S

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NID_TOL = 1e-12


def _cost(V, pr, bins=16, **kw):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    data = V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])
    return V.CostCalculatorNID(cam, data, V.NIDCostParams(bins), **kw)


def _oracle_eval(O, pr, Ts, bins=16):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(cam, pr["W"], pr["H"])
    out = [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], bins, fov, T) for T in Ts]
    return np.array([o[0] for o in out]), np.stack([o[1] for o in out])


def _assert_close_nid(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    m = ~np.isnan(a)
    assert np.all(np.abs(a[m] - b[m]) < NID_TOL), np.abs(a[m] - b[m]).max()


@pytest.mark.parametrize("model", util.MODELS)
def test_golden_fixtures(gpu, model):
    V = gpu
    g = np.load(os.path.join(GOLDEN, f"mode_a_{model}.npz"))
    cam = V.create_camera(model, g["intrinsics"], g["distortion"])
    data = V.VisualLiDARData(g["image"], np.concatenate([g["points"][:, :3].astype(np.float64), np.ones((g["points"].shape[0], 1))], axis=1), g["intensities"].astype(np.float64))
    cost = V.CostCalculatorNID(cam, data)
    assert cost.max_fov == float(g["max_fov"])
    nid, hist = cost.calculate_batch(g["poses"], return_hist=True)
    assert np.array_equal(hist, g["hist"])
    _assert_close_nid(nid, g["nid"])
    idx = V.ViewCulling(cam, (g["image"].shape[1], g["image"].shape[0])).cull_indices(data.points, g["poses"][0])
    assert np.array_equal(idx, g["cull_indices"])


@pytest.mark.parametrize("model", util.MODELS)
def test_histograms_bit_exact_vs_oracle(gpu, oracle, model):
    pr = util.random_problem(model, n=60000, seed=21)
    Ts = util.random_poses(pr["T"], 5, seed=4)
    cost = _cost(gpu, pr)
    assert cost.points_are_f32
    nid, hist = cost.calculate_batch(Ts, return_hist=True)
    ref_nid, ref_hist = _oracle_eval(oracle, pr, Ts)
    assert int(np.abs(hist - ref_hist).sum()) == 0
    assert hist.sum() > 10000
    _assert_close_nid(nid, ref_nid)
    # reference surface: calculate(T) == batch entry, bit for bit
    assert cost.calculate(Ts[2]) == nid[2]


def test_batch_equals_singles_and_chunking(gpu, oracle):
    pr = util.random_problem("plumb_bob", n=30000, seed=5)
    Ts = util.random_poses(pr["T"], 21, seed=8)  # three passes of the persistent kernel (the round-1 chunking: test_gpu_round1_edges.py)
    cost = _cost(gpu, pr)
    nid, hist = cost.calculate_batch(Ts, return_hist=True)
    for p in (0, 7, 8, 20):
        n1, h1 = cost.calculate_batch(Ts[p : p + 1], return_hist=True)
        assert n1[0] == nid[p] and np.array_equal(h1[0], hist[p])
    ref_nid, ref_hist = _oracle_eval(oracle, pr, Ts)
    assert np.array_equal(hist, ref_hist)
    _assert_close_nid(nid, ref_nid)
    # repeated evaluation is deterministic and the self-cleaning accumulators leave no residue
    nid2, hist2 = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(nid, nid2) and np.array_equal(hist, hist2)


@pytest.mark.parametrize("bins", [1, 4, 32, 64, 128])
def test_other_bin_counts(gpu, oracle, bins):
    pr = util.random_problem("plumb_bob", n=20000, seed=6)
    Ts = util.random_poses(pr["T"], 3, seed=1)
    nid, hist = _cost(gpu, pr, bins).calculate_batch(Ts, return_hist=True)
    ref_nid, ref_hist = _oracle_eval(oracle, pr, Ts, bins)
    assert np.array_equal(hist, ref_hist)
    _assert_close_nid(nid, ref_nid)


def test_unsupported_bins_is_an_error_not_a_fallback(gpu):
    pr = util.random_problem("plumb_bob", n=100, seed=6)
    with pytest.raises(gpu.VlcalError) as e:
        _cost(gpu, pr, 256)
    assert e.value.code == -6


def test_double_layout_when_points_are_not_float32(gpu, oracle):
    pr = util.random_problem("rational_polynomial", n=20000, seed=7, f32=False)
    Ts = util.random_poses(pr["T"], 4, seed=2)
    cost = _cost(gpu, pr)
    assert not cost.points_are_f32
    nid, hist = cost.calculate_batch(Ts, return_hist=True)
    ref_nid, ref_hist = _oracle_eval(oracle, pr, Ts)
    assert np.array_equal(hist, ref_hist)
    _assert_close_nid(nid, ref_nid)


def test_edge_cases(gpu, oracle):
    V = gpu
    cam = V.create_camera("plumb_bob", [100.0, 100.0, 2.0, 2.0], [])
    img = (np.arange(16, dtype=np.uint8).reshape(4, 4) * 16).copy()
    T = np.eye(4)

    def inliers(x, y, z=1.0):
        data = V.VisualLiDARData(img, np.array([[x, y, z, 1.0]]), np.array([0.5]))
        c = V.CostCalculatorNID(cam, data, max_fov=1.4)
        return int(c.calculate_batch(T[None], return_hist=True)[1].sum())

    assert inliers(-0.025, 0.0) == 1  # u = -0.5 truncates to column 0 and is accepted
    assert inliers(-0.0301, 0.0) == 0 and inliers(0.0199, 0.0) == 1 and inliers(0.02, 0.0) == 0
    assert inliers(0.0, -0.025) == 1 and inliers(0.0, 0.0201) == 0
    assert inliers(0.0, 0.0, -1.0) == 0  # behind the camera
    assert inliers(float("nan"), 0.0) == 0
    # no inliers -> NaN, as the reference (no guard, cost_calculator_nid.cpp:54-64)
    data = V.VisualLiDARData(img, np.array([[0.0, 0.0, -1.0, 1.0]]), np.array([0.5]))
    assert math.isnan(V.CostCalculatorNID(cam, data, max_fov=1.4).calculate(T))
    # empty cloud -> NaN
    data = V.VisualLiDARData(img, np.zeros((0, 4)), np.zeros(0))
    assert math.isnan(V.CostCalculatorNID(cam, data, max_fov=1.4).calculate(T))
    # padded image rows (row_stride > width)
    big = np.random.default_rng(0).integers(0, 256, (48, 80), dtype=np.uint8)
    view = big[:, :64]
    pr = util.random_problem("plumb_bob", n=5000, seed=3, size=(64, 48))
    cam2 = V.create_camera("plumb_bob", [40.0, 41.0, 32.0, 24.0], pr["distortion"])
    ocam = oracle.create_camera("plumb_bob", [40.0, 41.0, 32.0, 24.0], pr["distortion"])

    class _D:  # VisualLiDARData would make the view contiguous; build the strided case by hand
        image, points, intensities = view, pr["points"], pr["intensities"]

        @staticmethod
        def size():
            return pr["points"].shape[0]

    c = V.CostCalculatorNID(cam2, _D)
    _, h = c.calculate_batch(pr["T"][None], return_hist=True)
    fov = oracle.estimate_camera_fov(ocam, 64, 48)
    _, href = oracle.nid_calculate(ocam, np.ascontiguousarray(view), pr["points"], pr["intensities"], 16, fov, pr["T"])
    assert np.array_equal(h[0], href)
    # w != 1 is rejected loudly
    bad = V.VisualLiDARData(img, np.array([[0.0, 0.0, 1.0, 2.0]]), np.array([0.5]))
    with pytest.raises(V.VlcalError):
        V.CostCalculatorNID(cam, bad)


def test_reorder_for_pose_changes_nothing_but_the_order(gpu, oracle):
    pr = util.random_problem("plumb_bob", n=50000, seed=13)
    Ts = util.random_poses(pr["T"], 6, seed=2)
    cost = _cost(gpu, pr)
    nid0, hist0 = cost.calculate_batch(Ts, return_hist=True)
    cost.reorder_for_pose(Ts[0])
    nid1, hist1 = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(hist0, hist1) and np.array_equal(nid0, nid1, equal_nan=True)
    assert np.array_equal(hist1, _oracle_eval(oracle, pr, Ts)[1])


def test_permutation_invariance(gpu):
    pr = util.random_problem("fisheye", n=40000, seed=12)
    perm = np.random.default_rng(1).permutation(40000)
    a = _cost(gpu, pr).calculate_batch(pr["T"][None], return_hist=True)
    pr2 = dict(pr, points=pr["points"][perm], intensities=pr["intensities"][perm])
    b = _cost(gpu, pr2).calculate_batch(pr["T"][None], return_hist=True)
    assert np.array_equal(a[1], b[1]) and a[0][0] == b[0][0]


@pytest.mark.parametrize("model", util.MODELS)
@pytest.mark.parametrize("depth", [True, False])
def test_view_culling_indices_identical(gpu, oracle, model, depth):
    pr = util.random_problem(model, n=80000, seed=31)
    cam = gpu.create_camera(model, pr["intrinsics"], pr["distortion"])
    ocam = oracle.create_camera(model, pr["intrinsics"], pr["distortion"])
    fov = oracle.estimate_camera_fov(ocam, pr["W"], pr["H"])
    ref = oracle.view_cull(ocam, pr["W"], pr["H"], fov, depth, pr["points"], pr["T"])
    idx = gpu.ViewCulling(cam, (pr["W"], pr["H"]), gpu.ViewCullingParams(depth)).cull_indices(pr["points"], pr["T"])
    assert np.array_equal(idx, ref) and len(ref) > 1000


def _synthetic_bag(n, cfg=3, scale=0.5):
    from direct_visual_lidar_calibration_b200 import synthetic as S

    bag = S.make_bag("pinhole_640x480", "frustum", n, config_index=cfg, scale=scale)
    bag["T_init"] = S.perturb(bag["T_gt"], (0.3, -0.3, 0.3), (0.01, -0.01, 0.01))
    return bag


def test_inner_solve_follows_oracle_evaluation_by_evaluation(gpu, oracle):
    V = gpu
    bag = _synthetic_bag(40000)
    cam = V.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    ocam = oracle.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    data = V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 80
    calib = V.VisualCameraCalibration(cam, [data], params)
    T, r = calib.estimate_pose_nelder_mead(bag["T_init"])
    op = oracle.default_calib_params()
    op.max_inner_iterations = 80
    ref = oracle.estimate_pose_nelder_mead(ocam, [(bag["image"], bag["points"], bag["intensities"])], bag["T_init"], op)
    assert r["num_iterations"] == ref["num_iterations"] and r["converged"] == ref["converged"]
    assert r["num_evaluations"] == ref["num_evaluations"]
    assert np.array_equal(r["x"], ref["x"])  # identical decisions -> identical simplex arithmetic
    assert abs(r["y"] - ref["y"]) < NID_TOL
    assert np.abs(T - ref["T"]).max() == 0.0
    # best-cost callback sequence == prefix minima of the oracle's evaluation trace
    tr = ref["trace"][:, 6]
    best, expect = float("inf"), []
    for c in tr:
        if c < best:
            best = c
            expect.append(c)
    got = [c for _, c in calib.trace]
    assert len(got) == len(expect) and np.allclose(got, expect, atol=NID_TOL)
    assert calib.stats["total_batches"] < ref["num_evaluations"]  # batched: fewer launches than evaluations


def test_host_loop_equals_persistent_solve_and_oracle(gpu, oracle):
    """The Nelder-Mead state machine advanced inside every block of the persistent cooperative kernel (mode 3, warp-parallel
    step) must walk exactly the trajectory of the host loop (mode 1), and both that of the oracle: same x, y, iterations,
    evaluations, callback sequence."""
    V = gpu
    bag = _synthetic_bag(40000, cfg=6)
    cam = V.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    data = V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 100
    out = {}
    try:
        for mode in (1, 3):
            V.set_solver_mode(mode)
            calib = V.VisualCameraCalibration(cam, [data], params)
            T, r = calib.estimate_pose_nelder_mead(bag["T_init"])
            out[mode] = (T, r, [c for _, c in calib.trace], calib.stats)
    finally:
        V.set_solver_mode(0)
    (Th, rh, trh, sth), (Tp, rp, trp, stp) = out[1], out[3]
    assert np.array_equal(Th, Tp) and np.array_equal(rh["x"], rp["x"]) and rh["y"] == rp["y"]
    assert rh["num_iterations"] == rp["num_iterations"] and rh["num_evaluations"] == rp["num_evaluations"] and rh["converged"] == rp["converged"]
    assert rh["num_batches"] == rp["num_batches"] and rh["num_evaluations_computed"] == rp["num_evaluations_computed"]
    assert trh == trp and len(trh) > 3
    ocam = oracle.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    op = oracle.default_calib_params()
    op.max_inner_iterations = 100
    ref = oracle.estimate_pose_nelder_mead(ocam, [(bag["image"], bag["points"], bag["intensities"])], bag["T_init"], op)
    assert np.array_equal(rh["x"], ref["x"]) and rh["num_iterations"] == ref["num_iterations"] and rh["num_evaluations"] == ref["num_evaluations"]
    assert np.abs(Th - ref["T"]).max() == 0.0 and abs(rh["y"] - ref["y"]) < NID_TOL
    # max_inner_iterations = 0: the loop body never runs, the result is the un-sorted x0 (nelder_mead.hpp:49,99)
    params.max_inner_iterations = 0
    for mode in (1, 3):
        try:
            V.set_solver_mode(mode)
            T0, r0 = V.VisualCameraCalibration(cam, [data], params).estimate_pose_nelder_mead(bag["T_init"])
        finally:
            V.set_solver_mode(0)
        assert r0["num_evaluations"] == 7 and np.array_equal(r0["x"], np.zeros(6)) and np.abs(T0 - bag["T_init"]).max() < 1e-15


def test_persistent_solve_two_bags_one_launch(gpu, oracle):
    """Several bags per GPU: the persistent kernel partitions its grid over the bags and sums their scores in bag order;
    the trajectory must be the host loop's (one launch per bag and batch) and the oracle's."""
    V = gpu
    b1, b2 = _synthetic_bag(30000, cfg=4), _synthetic_bag(9000, cfg=5)
    cam = V.create_camera(b1["camera_model"], b1["intrinsics"], b1["distortion"])
    ds = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in (b1, b2)]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 60
    out = {}
    try:
        for mode in (1, 3):
            V.set_solver_mode(mode)
            calib = V.VisualCameraCalibration(cam, ds, params)
            T, r = calib.estimate_pose_nelder_mead(b1["T_init"])
            out[mode] = (T, r, [c for _, c in calib.trace])
    finally:
        V.set_solver_mode(0)
    (Th, rh, trh), (Tp, rp, trp) = out[1], out[3]
    assert np.array_equal(Th, Tp) and np.array_equal(rh["x"], rp["x"]) and rh["y"] == rp["y"] and trh == trp
    assert rh["num_evaluations"] == rp["num_evaluations"] and rh["num_batches"] == rp["num_batches"]
    ocam = oracle.create_camera(b1["camera_model"], b1["intrinsics"], b1["distortion"])
    op = oracle.default_calib_params()
    op.max_inner_iterations = 60
    ref = oracle.estimate_pose_nelder_mead(ocam, [(b["image"], b["points"], b["intensities"]) for b in (b1, b2)], b1["T_init"], op)
    assert np.array_equal(rp["x"], ref["x"]) and rp["num_evaluations"] == ref["num_evaluations"] and np.abs(Tp - ref["T"]).max() == 0.0


@pytest.mark.parametrize("bins,n_bags", [(8, 1), (10, 2), (32, 2), (16, 4)])
def test_persistent_solve_other_bin_counts_and_finalizer_rounds(gpu, bins, n_bags):
    """The every-block finalizer stages bins^2 + 2 bins entropy terms per (bag, pose) in the dead histogram copies and works
    through the items in rounds of what fits (7 items at 32 bins, 21 at 16): bin counts that are not 16, not a power of two,
    and bag counts that need several rounds must walk the host loop's trajectory, bit for bit."""
    V = gpu
    bags = [_synthetic_bag(20000 + 3000 * k, cfg=4 + (k % 3)) for k in range(n_bags)]
    cam = V.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    ds = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 30
    params.nid_bins = bins
    out = {}
    try:
        for mode in (1, 3):
            V.set_solver_mode(mode)
            calib = V.VisualCameraCalibration(cam, ds, params)
            T, r = calib.estimate_pose_nelder_mead(bags[0]["T_init"])
            out[mode] = (T, r, [c for _, c in calib.trace])
    finally:
        V.set_solver_mode(0)
    (Th, rh, trh), (Tp, rp, trp) = out[1], out[3]
    assert np.array_equal(Th, Tp) and np.array_equal(rh["x"], rp["x"]) and rh["y"] == rp["y"] and trh == trp
    assert rh["num_evaluations"] == rp["num_evaluations"] and rh["num_batches"] == rp["num_batches"]


def test_score_poses_equals_calculate(gpu, oracle):
    """vlcal_nid_score_poses (one persistent launch for a pose list of any length, several bags) == calculate() per pose."""
    V = gpu
    pr1, pr2 = util.random_problem("plumb_bob", n=60000, seed=3), util.random_problem("plumb_bob", n=25000, seed=4)
    pr2["image"], pr2["intrinsics"], pr2["distortion"] = pr1["image"][::-1].copy(), pr1["intrinsics"], pr1["distortion"]
    c1, c2 = _cost(V, pr1), _cost(V, pr2)
    Ts = util.random_poses(pr1["T"], 37, seed=5, rot_deg=2.0, trans=0.1)  # 37: four full chunks of 8 and a partial one
    got = V.score_poses([c1, c2], Ts)
    a, b = c1.calculate_batch(Ts), c2.calculate_batch(Ts)
    assert np.array_equal(got, a + b, equal_nan=True)
    singles = np.array([c1.calculate(T) for T in Ts[:5]])
    assert np.array_equal(singles, a[:5], equal_nan=True)
    assert np.array_equal(V.score_poses([c1], Ts), a, equal_nan=True)
    ref_nid, _ = _oracle_eval(oracle, pr1, Ts[:3])
    _assert_close_nid(a[:3], ref_nid)


def test_full_calibrate_single_bag_host_loop_and_default(gpu, oracle):
    """The whole calibrate() of one bag, in the host loop (mode 1) and in the default mode (0), against the oracle's."""
    V = gpu
    bag = _synthetic_bag(30000, cfg=8)
    cam = V.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    ocam = oracle.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations, params.max_outer_iterations = 50, 3
    params.delta_trans_thresh, params.delta_rot_thresh = 1e-4, 1e-5
    op = oracle.default_calib_params()
    op.max_inner_iterations, op.max_outer_iterations, op.delta_trans_thresh, op.delta_rot_thresh = 50, 3, 1e-4, 1e-5
    ref = oracle.calibrate(ocam, [(bag["image"], bag["points"], bag["intensities"])], bag["T_init"], op)
    for mode in (1, 0):
        calib = V.VisualCameraCalibration(cam, [V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])], params)
        try:
            V.set_solver_mode(mode)
            T = calib.calibrate(bag["T_init"])
        finally:
            V.set_solver_mode(0)
        assert calib.stats["outer_iterations"] == ref["outer_iterations"] and calib.stats["inner_iterations"] == ref["inner_iterations"], mode
        assert calib.stats["total_evaluations"] == ref["total_evaluations"], mode
        assert np.abs(T - ref["T"]).max() < 1e-15, mode


def test_full_calibrate_matches_oracle_two_bags(gpu, oracle):
    V = gpu
    b1, b2 = _synthetic_bag(30000, cfg=4), _synthetic_bag(25000, cfg=5)
    cam = V.create_camera(b1["camera_model"], b1["intrinsics"], b1["distortion"])
    ocam = oracle.create_camera(b1["camera_model"], b1["intrinsics"], b1["distortion"])
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 40
    params.max_outer_iterations = 3
    params.delta_trans_thresh = 1e-4  # force more than one outer iteration
    params.delta_rot_thresh = 1e-5
    ds = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in (b1, b2)]
    calib = V.VisualCameraCalibration(cam, ds, params)
    T = calib.calibrate(b1["T_init"])
    op = oracle.default_calib_params()
    op.max_inner_iterations, op.max_outer_iterations, op.delta_trans_thresh, op.delta_rot_thresh = 40, 3, 1e-4, 1e-5
    ref = oracle.calibrate(ocam, [(b["image"], b["points"], b["intensities"]) for b in (b1, b2)], b1["T_init"], op)
    assert calib.stats["outer_iterations"] == ref["outer_iterations"]
    assert calib.stats["inner_iterations"] == ref["inner_iterations"]
    assert calib.stats["total_evaluations"] == ref["total_evaluations"]
    assert np.abs(T - ref["T"]).max() < 1e-15
    assert np.allclose(calib.stats["inner_final_cost"], ref["inner_final_cost"], atol=2 * NID_TOL)


def test_full_size_properties_c2(gpu):
    """BASELINE.json configs[1] size (1M points, 1920x1080): size-independent properties instead of the oracle."""
    V = gpu
    from direct_visual_lidar_calibration_b200 import synthetic as S

    rng = np.random.default_rng(77)
    n = 1_000_000
    dirs = S.lidar_directions("os1_64", n, rng)
    pts = (dirs * rng.uniform(1.0, 20.0, (n, 1))).astype(np.float32).astype(np.float64)
    inten = rng.integers(0, 256, n) / 256.0
    image = rng.integers(0, 256, (1080, 1920), dtype=np.uint8)
    model, intr, dist, W, H = S.CAMERAS["pinhole_1920x1080"]
    cam = V.create_camera(model, intr, dist)
    xyzw = np.concatenate([pts, np.ones((n, 1))], axis=1)
    T = S.gt_T_camera_lidar()
    Ts = util.random_poses(T, 4, seed=3, rot_deg=0.5, trans=0.02)
    full = V.CostCalculatorNID(cam, V.VisualLiDARData(image, xyzw, inten))
    nid, hist = full.calculate_batch(Ts, return_hist=True)
    # additivity: histogram of the whole cloud == sum of the histograms of its two halves (integer, exact)
    h1 = V.CostCalculatorNID(cam, V.VisualLiDARData(image, xyzw[: n // 2], inten[: n // 2])).calculate_batch(Ts, return_hist=True)[1]
    h2 = V.CostCalculatorNID(cam, V.VisualLiDARData(image, xyzw[n // 2 :], inten[n // 2 :])).calculate_batch(Ts, return_hist=True)[1]
    assert np.array_equal(hist, h1 + h2)
    # lidar marginal of the inliers is bounded by the cloud's own intensity histogram
    lb = np.minimum((inten * 16).astype(int), 15)
    assert np.all(hist.sum(axis=1) <= np.bincount(lb, minlength=16)[None, :])
    assert hist.sum() > 0 and np.all((nid >= 0) & (nid <= 1 + 1e-9))
    # bounds-only culling keeps a subset of the cost's inliers at the same pose: its FoV test divides z by the norm of
    # the homogeneous 4-vector (view_culling.cpp:45), which is stricter than the cost's z/|xyz| (cost_calculator_nid.cpp:32)
    kept = V.ViewCulling(cam, (W, H), V.ViewCullingParams(False)).cull_indices(xyzw, Ts[0])
    assert 0 < len(kept) <= hist[0].sum()
    sub = V.CostCalculatorNID(cam, V.VisualLiDARData(image, xyzw[kept], inten[kept])).calculate_batch(Ts[:1], return_hist=True)[1]
    assert sub[0].sum() == len(kept)  # every culled-in point is an inlier of the cost at that pose


# ---------------------------------------------------------------------------------------------------------------
# fp32 filter + exact recheck (default kernel for pinhole-type cameras on float32-representable clouds)
# ---------------------------------------------------------------------------------------------------------------

FILTER_MODELS = list(util.MODELS)  # every camera model has an fp32 filter with its own error bound


def _adversarial_problem(model, n, seed):
    """Clouds that stress the filter's error bound: far points (|p| large against the depth, large lever arms) and points
    very close to the sensor (tiny depths).  Random points almost never fall inside a decision's uncertain band; the FoV
    cone, the model guards and the pixel edges are targeted in test_gpu_filter_decision_edges.py."""
    rng = np.random.default_rng(seed)
    pr = util.random_problem(model, n=n, seed=seed)
    pts = pr["points"][:, :3].copy()
    k = n // 4
    pts[:k] *= rng.uniform(5.0, 40.0, (k, 1))  # far (up to ~1 km): |p| large vs depth
    pts[k : 2 * k] = util.S.lidar_directions("frustum", k, rng) * rng.uniform(0.05, 0.5, (k, 1))  # very close to the sensor
    pr["points"][:, :3] = pts.astype(np.float32).astype(np.float64)
    return pr


@pytest.mark.parametrize("model", FILTER_MODELS)
def test_filter_kernel_is_bit_identical_to_exact_kernel(gpu, oracle, model):
    pr = _adversarial_problem(model, 200000, seed=41)
    Ts = util.random_poses(pr["T"], 16, seed=9, rot_deg=5.0, trans=0.5)
    cost = _cost(gpu, pr)
    assert cost.filter_enabled
    nid_f, hist_f = cost.calculate_batch(Ts, return_hist=True)
    cost.set_kernel_variant(2)  # filter kernel, 2 points per thread
    nid_2, hist_2 = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(hist_f, hist_2) and np.array_equal(nid_f, nid_2, equal_nan=True)
    cost.set_kernel_variant(3)  # filter kernel, 4 points per thread
    nid_4, hist_4 = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(hist_f, hist_4) and np.array_equal(nid_f, nid_4, equal_nan=True)
    cost.set_kernel_variant(4)  # round-1 filter kernel (one launch per 8 poses)
    nid_r, hist_r = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(hist_f, hist_r) and np.array_equal(nid_f, nid_r, equal_nan=True)
    cost.set_kernel_variant(1)  # exact fp64 kernel
    nid_e, hist_e = cost.calculate_batch(Ts, return_hist=True)
    assert int(np.abs(hist_f - hist_e).sum()) == 0 and hist_f.sum() > 100000
    assert np.array_equal(nid_f, nid_e, equal_nan=True)
    ref_nid, ref_hist = _oracle_eval(oracle, pr, Ts[:3])
    assert np.array_equal(hist_f[:3], ref_hist)
    _assert_close_nid(nid_f[:3], ref_nid)


@pytest.mark.parametrize("model", FILTER_MODELS)
def test_filter_error_bound_is_sound(gpu, model):
    """Every verdict the filter keeps must equal the exact verdict; the measured fp32 error must stay inside the bound."""
    total_pp = 0
    for seed, rot, trans in [(51, 3.0, 0.3), (52, 20.0, 2.0), (53, 0.2, 0.01)]:
        pr = _adversarial_problem(model, 400000, seed=seed)
        Ts = util.random_poses(pr["T"], 24, seed=seed, rot_deg=rot, trans=trans)
        cost = _cost(gpu, pr)
        n_pp, deferred, mismatches, ratio = cost.debug_filter_check(Ts)  # lean classifier (what the default kernel runs)
        assert n_pp == 400000 * 24
        assert mismatches == 0
        assert ratio < 0.6, ratio  # the fp32 error of every accepted verdict uses well under the (x2 safety) bound
        assert deferred / n_pp < 0.2
        cost.set_kernel_variant(4)  # round-1 filter: also reports how much of its bound the fp32 error uses
        n_pp, deferred, mismatches, ratio = cost.debug_filter_check(Ts)
        assert n_pp == 400000 * 24
        assert mismatches == 0
        assert ratio < 0.5, ratio  # observed error uses less than half of the (already x2) bound
        assert deferred / n_pp < 0.15
        total_pp += n_pp
    assert total_pp > 2e7


def test_filter_on_c2_like_geometry_defers_few_points(gpu):
    from direct_visual_lidar_calibration_b200 import synthetic as S

    bag = S.make_bag("pinhole_1920x1080", "os1_64", 300000, config_index=1)
    cam = gpu.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    cost = gpu.CostCalculatorNID(cam, gpu.VisualLiDARData(bag["image"], bag["points"], bag["intensities"]))
    Ts = util.random_poses(bag["T_gt"], 8, seed=1, rot_deg=0.5, trans=0.02)
    n_pp, deferred, mismatches, ratio = cost.debug_filter_check(Ts)
    assert mismatches == 0 and ratio < 0.5
    assert deferred / n_pp < 0.05, deferred / n_pp


def test_filter_disabled_cases_fall_back_to_the_exact_kernel_not_to_cpu(gpu, oracle):
    # non-float32 cloud -> double layout -> exact kernel; pinhole with a ~89 degree half-FoV (z can reach 0) -> exact kernel
    pr = util.random_problem("plumb_bob", n=20000, seed=7, f32=False)
    assert not _cost(gpu, pr).filter_enabled
    pr = util.random_problem("plumb_bob", n=20000, seed=7)
    pr["intrinsics"] = [10.0, 10.0, 320.0, 240.0]
    pr["distortion"] = []
    cost = _cost(gpu, pr)
    assert not cost.filter_enabled
    Ts = util.random_poses(pr["T"], 2, seed=1)
    _, hist = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(hist, _oracle_eval(oracle, pr, Ts)[1]) and hist.sum() > 1000


# ---------------------------------------------------------------------------------------------------------------
# mode B: NIDCost::operator()<double> value (B-spline soft histogram)
# ---------------------------------------------------------------------------------------------------------------


def _sophus_params(T):
    from scipy.spatial.transform import Rotation

    q = Rotation.from_matrix(T[:3, :3]).as_quat()  # x y z w
    return np.concatenate([q, T[:3, 3]])


@pytest.mark.parametrize("model", util.MODELS)
def test_bspline_nid_matches_oracle(gpu, oracle, model):
    pr = util.random_problem(model, n=30000, seed=61)
    Ts = util.random_poses(pr["T"], 11, seed=3)  # > one launch of 8 poses
    tps = np.stack([_sophus_params(T) for T in Ts])
    cam = gpu.create_camera(model, pr["intrinsics"], pr["distortion"])
    cost = gpu.NIDCost(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), 16)
    ok, nid, hist = cost.evaluate(tps, return_hist=True)
    ocam = oracle.create_camera(model, pr["intrinsics"], pr["distortion"])
    for p in range(len(Ts)):
        rok, rnid, rhist = oracle.nid_cost_bspline(ocam, pr["image"], pr["points"], pr["intensities"], 16, tps[p])
        assert bool(ok[p]) == rok
        assert abs(nid[p] - rnid) < 1e-9, abs(nid[p] - rnid)  # 2^-40 fixed-point accumulation vs serial double sum
        assert np.abs(hist[p] - rhist).max() < 1e-6 and abs(hist[p].sum() - rhist.sum()) < 1e-5
        assert hist[p].sum() > 1000
    # deterministic run to run (integer accumulation) and batch == single
    ok2, nid2 = cost.evaluate(tps)
    assert np.array_equal(nid, nid2)
    assert cost(tps[9])[1] == nid[9]


def test_bspline_other_bins_and_failure_flag(gpu, oracle):
    pr = util.random_problem("plumb_bob", n=10000, seed=62)
    tp = _sophus_params(pr["T"])
    cam = gpu.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    ocam = oracle.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    for bins in (8, 32):
        ok, nid = gpu.NIDCost(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), bins).evaluate(tp[None])
        rok, rnid, _ = oracle.nid_cost_bspline(ocam, pr["image"], pr["points"], pr["intensities"], bins, tp)
        assert ok[0] == rok and abs(nid[0] - rnid) < 1e-9
    # every point behind / outside -> no inliers -> NaN -> the functor returns false (nid_cost.hpp:98-102)
    far = np.array([[0.0, 0.0, -5.0, 1.0]] * 10)
    T = np.eye(4)
    ok, nid = gpu.NIDCost(cam, gpu.VisualLiDARData(pr["image"], far * [1, 1, 1, 1] + [1e4, 0, 0, 0], np.full(10, 0.5)), 16).evaluate(_sophus_params(T)[None])
    rok, _, _ = oracle.nid_cost_bspline(ocam, pr["image"], far + [1e4, 0, 0, 0], np.full(10, 0.5), 16, _sophus_params(T))
    assert (not ok[0]) and (not rok)


# ---------------------------------------------------------------------------------------------------------------
# multi-GPU: fused bag all-reduce over NVLink peer memory (needs >= 2 GPUs on the box; skipped otherwise)
# ---------------------------------------------------------------------------------------------------------------


def test_fused_peer_exchange_matches_nccl_and_single_gpu(gpu):
    import subprocess
    import sys

    if gpu.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29541", os.path.join(root, "tools", "dist_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "P2P_CHECK world=2 fused_close_to_nccl=True fused_equals_nccl=True" in out.stdout
    assert "DIST_CHECK world=2 identical=True close=True fused_identical_to_single_gpu=True" in out.stdout
    assert "POSE_SHARD_CHECK world=2" in out.stdout and "identical=True" in out.stdout.split("POSE_SHARD_CHECK")[1]


def test_persistent_exchange_two_ranks_on_one_gpu(gpu):
    """The in-kernel score exchange of the persistent solve (tagged words in cudaIpc-shared mailboxes, summed in (rank, bag)
    order by every block of every rank) with TWO processes on ONE GPU -- so that the single-GPU test box covers it: one
    and two bags per rank and the mixed spinning / non-repetitive dataset of BASELINE config 4; every rank must end with
    the bits of the single-process solve over all bags (one launch) and of the round-1 host loop."""
    import subprocess
    import sys

    env = dict(os.environ, VLCAL_DIST_SINGLE_GPU="1", VLCAL_SYNC_TIMEOUT_MS="30000", OMP_NUM_THREADS="2")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29517", os.path.join(root, "tools", "dist_check_pk.py")],
        capture_output=True, text=True, timeout=900, env=env,
    )
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("PK_DIST_CHECK")]
    assert len(lines) == 3, out.stdout[-3000:]
    for ln in lines:
        assert "ranks_identical=True equals_single_process_one_launch=True equals_host_loop=True" in ln, ln


@pytest.mark.parametrize("model", util.MODELS)
def test_generate_lidar_image_equals_the_oracle(gpu, oracle, model):
    """K5 (generate_lidar_image.cpp:8-41 on the GPU): intensity image and index map identical to the oracle's, incl. ties."""
    for f32 in (True, False):
        pr = util.random_problem(model, n=60000, seed=6, f32=f32)
        pts = np.concatenate([pr["points"], pr["points"][:3000]])
        ins = np.concatenate([pr["intensities"], (pr["intensities"][:3000] + 0.5) % 1.0])
        cam = gpu.create_camera(model, pr["intrinsics"], pr["distortion"])
        inten, index = gpu.generate_lidar_image(cam, (pr["W"], pr["H"]), pr["T"], pts, ins)
        ocam = oracle.create_camera(model, pr["intrinsics"], pr["distortion"])
        ref_inten, ref_index = oracle.generate_lidar_image(ocam, pr["W"], pr["H"], pr["T"], pts, ins)
        assert np.array_equal(index, ref_index) and np.array_equal(inten, ref_inten)
        assert (index >= 0).sum() > 1000 and (index >= 60000).sum() > 10


def test_pose_grid_search_finds_the_basin(gpu, oracle):
    """Config-5 style coarse grid: every score equals the oracle's, and the best grid pose is the one nearest the truth."""
    from direct_visual_lidar_calibration_b200 import initial_guess as IG
    from direct_visual_lidar_calibration_b200 import synthetic as S

    bag = S.make_bag("pinhole_640x480", "frustum", 40000, config_index=12, scale=0.5)
    cam = gpu.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    cost = gpu.CostCalculatorNID(cam, gpu.VisualLiDARData(bag["image"], bag["points"], bag["intensities"]))
    T_rough = S.perturb(bag["T_gt"], (1.0, -1.0, 1.0), (0.02, 0.0, -0.02))
    grid = dict(n_rot=(3, 3, 3), n_trans=(1, 3, 3), rot_half_deg=1.0, trans_half=0.02)
    poses = IG.pose_grid(T_rough, **grid)
    assert poses.shape == (243, 4, 4)
    nid = IG.score_poses(cost, poses)
    ocam = oracle.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    fov = oracle.estimate_camera_fov(ocam, bag["width"], bag["height"])
    for k in (0, 100, 242):
        assert abs(nid[k] - oracle.nid_calculate(ocam, bag["image"], bag["points"], bag["intensities"], 16, fov, poses[k])[0]) < NID_TOL
    best, best_nid = IG.grid_search(cost, T_rough, top_k=3, **grid)
    assert best_nid[0] == np.nanmin(nid) and best_nid[0] <= best_nid[1] <= best_nid[2]
    # the grid contains the ground truth's neighbourhood (perturbation of +-1 deg / +-2 cm): the winner must be closer to it
    # than the rough centre is
    def dist_to_gt(T):
        d = np.linalg.inv(T) @ bag["T_gt"]
        return np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1)) + np.linalg.norm(d[:3, 3])

    assert dist_to_gt(best[0]) < dist_to_gt(T_rough)


# ---------------------------------------------------------------------------------------------------------------
# fuzz: the filter's error bound must hold for arbitrary (plausible and less plausible) camera parameters
# ---------------------------------------------------------------------------------------------------------------


def _random_camera(model, rng):
    W, H = int(rng.integers(320, 2049)), int(rng.integers(240, 1537))
    f = float(rng.uniform(0.25, 1.5) * W)
    intr4 = [f, f * float(rng.uniform(0.9, 1.1)), W / 2 + float(rng.uniform(-40, 40)), H / 2 + float(rng.uniform(-40, 40))]
    if model == "plumb_bob":
        return intr4, list(rng.uniform(-1, 1, 5) * [0.3, 0.2, 5e-3, 5e-3, 0.1]), (W, H)
    if model == "rational_polynomial":
        return intr4, list(rng.uniform(-1, 1, 8) * [0.3, 0.2, 5e-3, 5e-3, 0.1, 0.3, 0.2, 0.1]), (W, H)
    if model == "fisheye":
        return intr4, list(rng.uniform(-1, 1, 4) * [0.1, 0.05, 0.02, 0.01]), (W, H)
    if model == "atan":
        return intr4, [float(rng.choice([0.0, 1e-8, rng.uniform(0.1, 1.2)]))], (W, H)
    if model == "omnidir":
        return intr4 + [float(rng.uniform(0.5, 2.0))], list(rng.uniform(-1, 1, 4) * [0.3, 0.1, 5e-3, 5e-3]), (W, H)
    W2 = int(rng.integers(512, 4097))
    return [float(W2), float(W2 // 2)], [], (W2, W2 // 2)


@pytest.mark.parametrize("model", util.MODELS)
def test_filter_bound_fuzz_over_random_cameras(gpu, model):
    rng = np.random.default_rng(1234 + util.MODELS.index(model))
    checked = 0
    for trial in range(12):
        intr, dist, (W, H) = _random_camera(model, rng)
        pr = _adversarial_problem(model, 60000, seed=int(rng.integers(1 << 30)))
        pr.update(intrinsics=intr, distortion=dist, W=W, H=H, image=rng.integers(0, 256, (H, W), dtype=np.uint8))
        cost = _cost(gpu, pr)
        if not cost.filter_enabled:
            continue  # e.g. a pinhole whose estimated FoV reaches 87 degrees: exact kernel, nothing to check
        Ts = util.random_poses(pr["T"], 8, seed=trial, rot_deg=float(rng.choice([0.3, 5.0, 60.0])), trans=float(rng.choice([0.01, 0.5, 3.0])))
        n_pp, deferred, mismatches, ratio = cost.debug_filter_check(Ts)
        assert mismatches == 0, (model, intr, dist, mismatches)
        assert ratio < 1.0, (model, intr, dist, ratio)
        # and the two kernels agree on the histograms themselves
        h_f = cost.calculate_batch(Ts, return_hist=True)[1]
        cost.set_kernel_variant(1)
        h_e = cost.calculate_batch(Ts, return_hist=True)[1]
        assert np.array_equal(h_f, h_e)
        checked += 1
    assert checked >= 6


@pytest.mark.parametrize("model", util.MODELS)
def test_bspline_gradient_matches_oracle(gpu, oracle, model):
    """K3: NIDCost::operator()<ceres::Jet<double, 7>> -- value and d NID / d (qx qy qz qw tx ty tz) against the oracle
    (which tests/test_reference_pin.py pins bit-exact to the reference functor)."""
    pr = util.random_problem(model, n=20000, seed=81)
    Ts = util.random_poses(pr["T"], 3, seed=4)
    tps = np.stack([_sophus_params(T) for T in Ts])
    cam = gpu.create_camera(model, pr["intrinsics"], pr["distortion"])
    cost = gpu.NIDCost(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), 16)
    ok, nid, grad = cost.evaluate_with_gradient(tps)
    ocam = oracle.create_camera(model, pr["intrinsics"], pr["distortion"])
    for p in range(len(Ts)):
        rok, rnid, rgrad = oracle.nid_cost_bspline_grad(ocam, pr["image"], pr["points"], pr["intensities"], 16, tps[p])
        assert bool(ok[p]) == rok
        assert abs(nid[p] - rnid) < 1e-9, abs(nid[p] - rnid)
        scale = max(1.0, np.abs(rgrad).max())
        assert np.abs(grad[p] - rgrad).max() < 1e-8 * scale, (grad[p], rgrad)
        assert np.abs(rgrad).max() > 1e-4
    # the value half agrees with the value-only kernel (different rounding of the divisions: Jet vs double functor)
    ok2, nid2 = cost.evaluate(tps)
    assert np.abs(nid - nid2).max() < 1e-9
    # run-to-run: the weights are fixed point (bit-stable), the partial sums are double atomics (last bits may move)
    ok3, nid3, grad3 = cost.evaluate_with_gradient(tps)
    assert np.array_equal(nid, nid3) and np.abs(grad - grad3).max() < 1e-10 * max(1.0, np.abs(grad).max())


def test_bspline_gradient_other_bins_and_failure_flag(gpu, oracle):
    pr = util.random_problem("plumb_bob", n=10000, seed=82)
    tp = _sophus_params(pr["T"])
    cam = gpu.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    ocam = oracle.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    for bins in (8, 32):
        ok, nid, grad = gpu.NIDCost(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), bins).evaluate_with_gradient(tp[None])
        rok, rnid, rgrad = oracle.nid_cost_bspline_grad(ocam, pr["image"], pr["points"], pr["intensities"], bins, tp)
        assert ok[0] == rok and abs(nid[0] - rnid) < 1e-9 and np.abs(grad[0] - rgrad).max() < 1e-8 * max(1.0, np.abs(rgrad).max())
    far = np.array([[1.0, 5e3, 0.0, 1.0]] * 10)  # every projection lands outside the image -> NaN -> false (nid_cost.hpp:98-102)
    ok, _, _ = gpu.NIDCost(cam, gpu.VisualLiDARData(pr["image"], far, np.full(10, 0.5)), 16).evaluate_with_gradient(tp[None])
    rok, _, _ = oracle.nid_cost_bspline_grad(ocam, pr["image"], far, np.full(10, 0.5), 16, tp)
    assert not ok[0] and not rok


def test_bspline_gradient_double_layout(gpu, oracle):
    pr = util.random_problem("fisheye", n=8000, seed=83, f32=False)
    tp = _sophus_params(pr["T"])
    cam = gpu.create_camera("fisheye", pr["intrinsics"], pr["distortion"])
    ocam = oracle.create_camera("fisheye", pr["intrinsics"], pr["distortion"])
    ok, nid, grad = gpu.NIDCost(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), 16).evaluate_with_gradient(tp[None])
    rok, rnid, rgrad = oracle.nid_cost_bspline_grad(ocam, pr["image"], pr["points"], pr["intensities"], 16, tp)
    assert ok[0] == rok and abs(nid[0] - rnid) < 1e-9 and np.abs(grad[0] - rgrad).max() < 1e-8 * max(1.0, np.abs(rgrad).max())


def test_bfgs_branch_runs_on_the_gpu_cost(gpu, oracle):
    """NID_BFGS branch (visual_camera_calibration.cpp:187-238) on K3: the solver is ours (Ceres-free), so the checks are
    (i) every cost it reports is the oracle's mode-B NID of the same culled cloud at that pose, (ii) it descends,
    (iii) it stays inside the reference's 0.2 m / 2 deg trust region."""
    from direct_visual_lidar_calibration_b200 import synthetic as S

    bag = S.make_bag("pinhole_640x480", "frustum", 40000, config_index=11, scale=0.5)
    cam = gpu.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    T0 = S.perturb(bag["T_gt"], (0.3, -0.2, 0.25), (0.01, -0.008, 0.006))
    params = gpu.VisualCameraCalibrationParams()
    params.registration_type = gpu.RegistrationType.NID_BFGS
    seen = []
    params.callback = lambda T: seen.append(T.copy())
    calib = gpu.VisualCameraCalibration(cam, [gpu.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])], params)
    T, r = calib.estimate_pose_bfgs(T0)
    assert r["iterations"] >= 1 and len(seen) == r["iterations"] and r["final_cost"] < r["initial_cost"], r
    d = np.linalg.inv(T0) @ T
    assert np.linalg.norm(d[:3, 3]) <= 0.2 and np.arccos(np.clip(0.5 * (np.trace(d[:3, :3]) - 1), -1, 1)) <= np.deg2rad(2.0)
    # the costs are the reference functor's values on the cloud culled at T0 (view_culling.cpp + nid_cost.hpp)
    ocam = oracle.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    fov = oracle.estimate_camera_fov(ocam, bag["width"], bag["height"])
    idx = oracle.view_cull(ocam, bag["width"], bag["height"], fov, True, bag["points"], T0)
    pts, ins = bag["points"][idx], bag["intensities"][idx]
    ok0, c0, _ = oracle.nid_cost_bspline_grad(ocam, bag["image"], pts, ins, 16, _sophus_params(T0))
    ok1, c1, g1 = oracle.nid_cost_bspline_grad(ocam, bag["image"], pts, ins, 16, _sophus_params(T))
    assert ok0 and ok1 and abs(c0 - r["initial_cost"]) < 1e-9 and abs(c1 - r["final_cost"]) < 1e-9
    assert [c for _, c in calib.trace] == sorted([c for _, c in calib.trace], reverse=True)  # monotone descent
    # the outer loop (visual_camera_calibration.cpp:35-68) around it
    params.max_outer_iterations = 2
    T2 = calib.calibrate(T0)
    assert calib.stats["outer_iterations"] >= 1 and np.isfinite(T2).all()


@pytest.mark.parametrize("model", util.MODELS)
def test_mode_b_golden_fixtures(gpu, model):
    """K2 / K3 against the committed vectors of the reference functor (tests/golden/mode_b_*.npz)."""
    g = np.load(os.path.join(GOLDEN, f"mode_b_{model}.npz"))
    cam = gpu.create_camera(model, g["intrinsics"], g["distortion"])
    cost = gpu.NIDCost(cam, gpu.VisualLiDARData(g["image"], g["points"].astype(np.float64), g["intensities"].astype(np.float64)), 16)
    ok, nid = cost.evaluate(g["T_params"])
    assert ok.all() and np.abs(nid - g["nid_double_functor"]).max() < 1e-9
    ok, nid, grad = cost.evaluate_with_gradient(g["T_params"])
    assert ok.all() and np.abs(nid - g["nid_jet_functor"]).max() < 1e-9
    assert np.abs(grad - g["grad"]).max() < 1e-8 * max(1.0, np.abs(g["grad"]).max())
