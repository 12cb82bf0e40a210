"""Pins the oracle (oracle/vlcal_oracle.c) against the REFERENCE's own sources of the path.

The reference side is what the reference's code returned for these seeded inputs: create_camera.cpp + camera/*.hpp,
dfo/nelder_mead.hpp, estimate_fov.cpp, cost_calculator_nid.cpp, view_culling.cpp, visual_camera_calibration.cpp,
generate_lidar_image.cpp and nid_cost.hpp, compiled against the stand-in third-party headers of oracle/ref_standin/
(oracle/ref_shim.cpp, `make -C oracle ref`).  Those answers are stored in tests/golden/reference_outputs.json
(tests/golden/make_reference_outputs.py writes it from oracle/_ref/libvlcal_ref.so), so the comparison needs nothing
outside the repository.  Small results are stored as values; large arrays as a SHA-256 of their canonical bytes (NaNs
folded to one bit pattern, signed zeros kept), so every comparison below stays bit for bit.  Eigen's own reduction
orders are restated, not pinned, by the stand-ins (oracle/ref_standin/Eigen/Core lists the conventions); the NID
tolerance of the GPU tests (1e-12 on the entropy tail) covers what the stand-in cannot pin.  CPU-only."""
import glob
import hashlib
import json
import os

import numpy as np
import pytest

import util as U
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "reference_outputs.json")


def digest(a, fold_zeros=False) -> str:
    """Canonical digest of an array: kind, shape and the SHA-256 of its bytes (float64 with one NaN pattern, or int64).
    fold_zeros: -0.0 counts as 0.0 (comparisons by difference)."""
    a = np.asarray(a)
    if a.dtype.kind == "f":
        a = np.where(np.isnan(a), np.nan, a.astype(np.float64))
        if fold_zeros:
            a = a + 0.0
    else:
        a = a.astype(np.int64)
    a = np.ascontiguousarray(a)
    return f"{a.dtype.kind}{list(a.shape)}:{hashlib.sha256(a.tobytes()).hexdigest()}"


def same(a, b) -> bool:
    """Scalar equality with NaN == NaN."""
    return a == b or (a != a and b != b)


def load_golden() -> dict:
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def ref():
    return load_golden()


def _rcam(R, model):
    intr, dist, (W, H) = U.CAMERAS[model]
    return R.Camera(model, intr, dist)


def cameras(model):
    intr, dist, (W, H) = U.CAMERAS[model]
    return O.create_camera(model, intr, dist), W, H


def special_points():
    e = 1e-300
    return np.array(
        [[0, 0, 0], [0, 0, 1], [0, 0, -1], [1, 0, 0], [0, 1, 0], [0, -1, 0], [1e-4, 0, 1e-4], [0, 1e-2, 1e-2], [3, 4, 1e-9], [1e-3, 1e-3, 1.0], [e, e, e], [1e200, 1e200, 1e200],
         [np.nan, 0, 1], [np.inf, 0, 1], [0.5, -0.25, 2.0], [-7.0, 3.0, 0.1], [2.0, 2.0, -0.5], [0.0, 0.0, 1e-320]], dtype=np.float64)


def _projection_points():
    rng = np.random.default_rng(11)
    return np.concatenate([rng.normal(size=(30000, 3)) * rng.uniform(0.01, 40.0, (30000, 1)), special_points()])


@pytest.mark.parametrize("model", U.MODELS)
def test_projection_bit_exact(ref, model):
    oc, W, H = cameras(model)
    uv_o = np.array([O.project(oc, p) for p in _projection_points()])
    assert digest(uv_o) == ref[f"projection/{model}"]  # signed zeros included


REJECT_DISTORTIONS = ([], [-0.04], [-0.04, 0.08, 1e-4, -3e-4, -0.04, 9.0, 9.0])
REJECT_POINT = np.array([[0.3, -0.2, 1.5]])


def test_create_camera_rejections(ref):
    g = ref["create_camera"]
    assert g["unknown_model_is_null"] and g["short_intrinsics_is_null"]  # create_camera.cpp:49-50, :19-22
    assert O.create_camera("no_such_model", [1, 1, 1, 1], []) is None
    assert O.create_camera("plumb_bob", [1, 1, 1], []) is None
    # short distortion lists are zero-padded, long ones truncated (:24-27)
    for dist, want in zip(REJECT_DISTORTIONS, g["padded_projection"]):
        oc = O.create_camera("plumb_bob", [400, 410, 320, 240], dist)
        assert np.array_equal(np.array([O.project(oc, REJECT_POINT[0])]), np.array(want))


@pytest.mark.parametrize("model", U.MODELS)
def test_estimate_camera_fov_bit_exact(ref, model):
    oc, W, H = cameras(model)
    # odd sizes: integer halves (:37)
    assert [O.estimate_camera_fov(oc, W, H), O.estimate_camera_fov(oc, W // 2 + 1, H // 3)] == ref[f"fov/{model}"]


def _objectives():
    def rosenbrock(x):
        return float(100.0 * (x[1] - x[0] ** 2) ** 2 + (1.0 - x[0]) ** 2)

    def bowl(x):
        return float(np.sum((x - np.arange(len(x)) * 0.1) ** 2))

    def plateau(x):  # many exact ties: the sort / comparison order decides the trajectory
        return float(np.floor(4.0 * np.abs(x).sum()) / 4.0)

    def with_nan(x):  # NaN scores take the reference's comparison path
        return float("nan") if x[0] > 0.15 else float(np.sum(x * x) + np.sin(5.0 * x[-1]))

    def ridge(x):
        return float(abs(x[0] - x[1]) + 0.01 * np.sum(x * x))

    return {"rosenbrock": rosenbrock, "bowl": bowl, "plateau": plateau, "with_nan": with_nan, "ridge": ridge}


def _nm_trials(n):
    rng = np.random.default_rng(5 + n)
    out = []
    for trial, kw in enumerate([dict(), dict(init_step=1e-3, convergence_var_thresh=1e-10, max_iterations=60), dict(init_step=0.5, max_iterations=7)]):
        out.append((rng.uniform(-0.3, 0.3, n) if trial else np.zeros(n), kw))
    return out


def nm_record(r) -> dict:
    """A Nelder-Mead run: every objective evaluation in order (x, y), the result and its flags."""
    calls = np.array([np.concatenate([x, [y]]) for x, y in r["calls"]])
    return {"evaluations": len(r["calls"]), "calls": digest(calls), "converged": bool(r["converged"]), "num_iterations": int(r["num_iterations"]),
            "x": [float(v) for v in r["x"]], "y": float(r["y"])}


@pytest.mark.parametrize("n", [2, 3, 6])
@pytest.mark.parametrize("name", list(_objectives().keys()))
def test_nelder_mead_trajectory_identical(ref, n, name):
    f = _objectives()[name]
    for trial, ((x0, kw), want) in enumerate(zip(_nm_trials(n), ref[f"nelder_mead/{name}/{n}"])):
        got = nm_record(O.nelder_mead(f, x0, **kw))
        assert got["evaluations"] == want["evaluations"] and got["calls"] == want["calls"], (name, n, trial)
        assert got["converged"] == want["converged"] and got["num_iterations"] == want["num_iterations"]
        assert np.array_equal(got["x"], want["x"]) and same(got["y"], want["y"])


def _nid_problem(model, bins):
    pr = U.random_problem(model, n=30000, seed=21, f32=(bins == 16))
    return pr, U.random_poses(pr["T"], 4, seed=3)


@pytest.mark.parametrize("model", U.MODELS)
@pytest.mark.parametrize("bins", [16, 8])
def test_nid_calculate_bit_exact(ref, model, bins):
    oc, W, H = cameras(model)
    fov = O.estimate_camera_fov(oc, W, H)
    pr, Ts = _nid_problem(model, bins)
    got = [O.nid_calculate(oc, pr["image"], pr["points"], pr["intensities"], bins, fov, T)[0] for T in Ts]
    assert got == ref[f"nid/{model}/{bins}"]


def _edge_inputs():
    """(points, intensities) of the edge cases: no inliers, out-of-range / NaN values, a single point."""
    pr = U.random_problem("plumb_bob", n=2000, seed=2)
    behind = pr["points"].copy()
    behind[:, 0] = -np.abs(behind[:, 0]) - 1.0
    ins = pr["intensities"].copy()
    ins[::7] = 1.0
    ins[1::7] = -0.5
    ins[2::7] = 3.0
    ins[3::97] = np.nan
    pts = pr["points"].copy()
    pts[5::211, 1] = np.nan
    pts[6::211, 2] = 1e30
    return pr, [(behind, pr["intensities"]), (pts, ins), (pr["points"][:1], pr["intensities"][:1])]


def test_nid_calculate_edge_cases(ref):
    oc, W, H = cameras("plumb_bob")
    fov = O.estimate_camera_fov(oc, W, H)
    pr, cases = _edge_inputs()
    got = [O.nid_calculate(oc, pr["image"], p, i, 16, fov, pr["T"])[0] for p, i in cases]
    want = ref["nid_edge_cases"]
    assert np.isnan(got[0]) and np.isnan(want[0])  # no inliers -> 0/0 (cost_calculator_nid.cpp:54-57)
    assert got[1] == want[1]
    assert same(got[2], want[2])


def _cull_problem(model):
    pr = U.random_problem(model, n=40000, seed=33)
    return pr, U.random_poses(pr["T"], 2, seed=8)


@pytest.mark.parametrize("model", U.MODELS)
@pytest.mark.parametrize("depth", [True, False])
def test_view_culling_indices_identical(ref, model, depth):
    oc, W, H = cameras(model)
    fov = O.estimate_camera_fov(oc, W, H)
    pr, Ts = _cull_problem(model)
    assert [digest(O.view_cull(oc, W, H, fov, depth, pr["points"], T)) for T in Ts] == ref[f"view_cull/{model}/{depth}"]


def _fixture_files(prefix):
    files = sorted(glob.glob(os.path.join(HERE, "golden", f"{prefix}_*.npz")))
    assert len(files) == len(U.MODELS)
    return [(os.path.basename(p)[len(prefix) + 1:-len(".npz")], np.load(p)) for p in files]


def test_golden_fixtures_match_the_reference(ref):
    """The committed fixtures (made from the oracle, tests/golden/make_golden.py) are what the reference's code returns."""
    for model, g in _fixture_files("mode_a"):
        want = ref[f"golden_mode_a/{model}"]
        assert float(g["max_fov"]) == want["fov"]
        assert g["nid"].tolist() == want["nid"]
        assert digest(g["cull_indices"]) == want["cull"]


def _sophus_params(T):
    from scipy.spatial.transform import Rotation

    q = Rotation.from_matrix(T[:3, :3]).as_quat()  # x y z w
    return np.concatenate([q, T[:3, 3]])


def _bspline_value_cases(model):
    pr = U.random_problem(model, n=8000, seed=71)
    return pr, list(zip((16, 16, 8), U.random_poses(pr["T"], 3, seed=5)))


@pytest.mark.parametrize("model", U.MODELS)
def test_bspline_nid_value_bit_exact(ref, model):
    """NIDCost::operator()<double> (include/vlcal/costs/nid_cost.hpp:36-107), the value half of the BFGS branch."""
    oc, W, H = cameras(model)
    pr, cases = _bspline_value_cases(model)
    for (bins, T), (ok_r, nid_r) in zip(cases, ref[f"bspline_value/{model}"]):
        ok_o, nid_o, _ = O.nid_cost_bspline(oc, pr["image"], pr["points"], pr["intensities"], bins, _sophus_params(T))
        assert ok_r and ok_o and nid_r == nid_o, (nid_r, nid_o)


FAR_POINTS = np.array([[1.0, 5e3, 0.0, 1.0]] * 10)  # far off to the side: every projection lands outside the image


def test_bspline_failure_flag(ref):
    oc, W, H = cameras("plumb_bob")
    pr = U.random_problem("plumb_bob", n=100, seed=72)
    ok_o, _, _ = O.nid_cost_bspline(oc, pr["image"], FAR_POINTS, np.full(10, 0.5), 16, _sophus_params(pr["T"]))
    assert ref["bspline_failure_flag"] is False and ok_o is False  # no inliers -> NaN -> the functor returns false (nid_cost.hpp:98-102)


def _best_cost_poses(init_T, trace):
    """Poses the reference hands to params.callback: evaluations that improve on the best cost so far (:112-116)."""
    best, out = np.finfo(np.float64).max, []
    for row in trace:
        if row[6] < best:
            best = row[6]
            out.append(O.isometry_mul(init_T, O.se3_expmap(row[:6])))
    return out


ESTIMATE_POSE_CASES = [("plumb_bob", 1), ("plumb_bob", 2), ("fisheye", 1), ("equirectangular", 2)]


def _estimate_pose_problem(model, n_bags):
    bags = []
    for b in range(n_bags):
        pr = U.random_problem(model, n=6000 + 500 * b, seed=90 + b)
        bags.append((pr["image"], pr["points"], pr["intensities"]))
    return bags, U.random_poses(pr["T"], 1, seed=12, rot_deg=0.5, trans=0.02)[0]


def calibration_record(r) -> dict:
    """A calibrate_nelder_mead result: the final pose and the poses handed to params.callback."""
    return {"T": r["T"].reshape(-1).tolist(), "num_callbacks": int(r["num_callbacks"]), "callback_T": digest(r["callback_T"], fold_zeros=True)}


@pytest.mark.parametrize("model,n_bags", ESTIMATE_POSE_CASES)
def test_estimate_pose_nelder_mead_identical(ref, model, n_bags):
    """VisualCameraCalibration::estimate_pose_nelder_mead (visual_camera_calibration.cpp:70-139) through calibrate() with
    one outer iteration: culling at the start pose, one cost object per bag, objective sum in bag order, best-cost
    callbacks, result init_T * Expmap(x).  (GTSAM's Expmap and Eigen's Isometry product are stand-ins on the reference
    side -- restated like the oracle's; everything else is the reference's code.)"""
    oc, W, H = cameras(model)
    bags, T0 = _estimate_pose_problem(model, n_bags)
    p = O.default_calib_params()
    p.max_inner_iterations = 40
    p.max_outer_iterations = 1
    a = O.estimate_pose_nelder_mead(oc, bags, T0, p)
    want = ref[f"estimate_pose/{model}/{n_bags}"]
    assert a["T"].reshape(-1).tolist() == want["T"]
    poses = _best_cost_poses(T0, a["trace"])
    assert len(poses) == want["num_callbacks"]
    assert digest(np.array(poses).reshape(-1, 4, 4), fold_zeros=True) == want["callback_T"]


CALIBRATE_KWARGS = (dict(max_outer_iterations=3, max_inner_iterations=25, delta_trans_thresh=1e-9, delta_rot_thresh=1e-9),  # never converges: 3 outer iterations
                    dict(max_outer_iterations=5, max_inner_iterations=25),  # default thresholds: stops after the first
                    dict(max_outer_iterations=2, max_inner_iterations=30, disable_z_buffer_culling=True, nelder_mead_init_step=5e-3))


def _calibrate_problem():
    pr = U.random_problem("plumb_bob", n=8000, seed=95)
    return [(pr["image"], pr["points"], pr["intensities"])], U.random_poses(pr["T"], 1, seed=13, rot_deg=0.5, trans=0.02)[0]


def test_calibrate_outer_loop_identical(ref):
    """VisualCameraCalibration::calibrate (visual_camera_calibration.cpp:35-68): re-culling at every outer iteration and
    the delta_t / delta_r termination test."""
    oc, W, H = cameras("plumb_bob")
    bags, T0 = _calibrate_problem()
    for kw, want in zip(CALIBRATE_KWARGS, ref["calibrate_outer"]):
        p = O.default_calib_params()
        p.max_outer_iterations, p.max_inner_iterations = kw["max_outer_iterations"], kw["max_inner_iterations"]
        p.delta_trans_thresh = kw.get("delta_trans_thresh", p.delta_trans_thresh)
        p.delta_rot_thresh = kw.get("delta_rot_thresh", p.delta_rot_thresh)
        p.disable_z_buffer_culling = int(kw.get("disable_z_buffer_culling", False))
        p.nelder_mead_init_step = kw.get("nelder_mead_init_step", p.nelder_mead_init_step)
        assert O.calibrate(oc, bags, T0, p)["T"].reshape(-1).tolist() == want, kw


def _bspline_grad_cases(model):
    pr = U.random_problem(model, n=6000, seed=75)
    return pr, list(zip((16, 8), U.random_poses(pr["T"], 2, seed=6)))


@pytest.mark.parametrize("model", U.MODELS)
def test_bspline_nid_gradient_bit_exact(ref, model):
    """NIDCost::operator()<ceres::Jet<double, 7>> (what AutoDiffFirstOrderFunction evaluates in the BFGS branch,
    visual_camera_calibration.cpp:211): residual and its 7 partials, reference functor + stand-in Jet vs the oracle."""
    oc, W, H = cameras(model)
    pr, cases = _bspline_grad_cases(model)
    for (bins, T), (ok_r, nid_r, g_r) in zip(cases, ref[f"bspline_grad/{model}"]):
        ok_o, nid_o, g_o = O.nid_cost_bspline_grad(oc, pr["image"], pr["points"], pr["intensities"], bins, _sophus_params(T))
        assert ok_r and ok_o and nid_r == nid_o and g_o.tolist() == g_r, (nid_r, nid_o, g_r, g_o)
        assert np.abs(g_o).max() > 1e-4


def _smooth_problem():
    pr = U.random_problem("fisheye", n=6000, seed=76)
    H, W = pr["image"].shape
    yy, xx = np.mgrid[0:H, 0:W]
    img = (127 + 100 * np.sin(xx / 37.0) * np.cos(yy / 23.0)).astype(np.uint8)
    return pr, img, _sophus_params(pr["T"])


def test_bspline_gradient_is_the_derivative_of_the_value(ref):
    """Independent of any Jet arithmetic: central differences of the reference's double functor on a smooth image."""
    oc, W, H = cameras("fisheye")
    pr, img, tp = _smooth_problem()
    _, _, g = O.nid_cost_bspline_grad(oc, img, pr["points"], pr["intensities"], 16, tp)
    fd = np.array(ref["bspline_central_differences"])
    assert np.abs(g - fd).max() < 1e-5 * max(1.0, np.abs(g).max()), (g, fd)


def _random_camera(model, rng):
    W, H = int(rng.integers(64, 400)), int(rng.integers(48, 300))
    f = rng.uniform(0.4, 1.6) * W
    intr = [f, f * rng.uniform(0.9, 1.1), W * rng.uniform(0.4, 0.6), H * rng.uniform(0.4, 0.6)]
    if model == "plumb_bob":
        dist = list(rng.normal(0, [0.05, 0.05, 1e-3, 1e-3, 0.02]))
    elif model == "fisheye":
        dist = list(rng.normal(0, [0.02, 0.01, 0.005, 0.002]))
    elif model == "atan":
        dist = [float(rng.choice([0.0, 1e-8, rng.uniform(0.2, 1.2)]))]  # includes the d0 < 1e-7 branch (atan.hpp:17)
    elif model == "omnidir":
        intr = intr + [rng.uniform(0.5, 1.5)]
        dist = list(rng.normal(0, [0.05, 0.02, 1e-3, 1e-3]))
    elif model == "equirectangular":
        intr, dist = [float(W), float(H)], []
    else:
        dist = list(rng.normal(0, [0.05, 0.05, 1e-3, 1e-3, 0.02, 0.05, 0.03, 0.01]))
    return intr, dist, W, H


def _fuzz_trials(model):
    rng = np.random.default_rng(1000 + U.MODELS.index(model))
    for trial in range(8):
        intr, dist, W, H = _random_camera(model, rng)
        pts = rng.normal(size=(3000, 3)) * rng.uniform(0.05, 30.0, (3000, 1))
        pr = U.random_problem(model, n=4000, seed=2000 + trial, size=(W, H))
        Ts = U.random_poses(pr["T"], 2, seed=trial, rot_deg=4.0, trans=0.3)
        yield dict(intr=intr, dist=dist, W=W, H=H, pts=pts, pr=pr, Ts=Ts, bins=int(rng.choice([4, 16, 64])))


@pytest.mark.parametrize("model", U.MODELS)
def test_fuzz_random_cameras_projection_fov_nid_culling(ref, model):
    """Random intrinsics / distortions / image sizes (the fixed presets above could hide a branch): projection, FoV, NID and
    culling of the oracle against the reference's code, bit for bit."""
    for trial, (c, want) in enumerate(zip(_fuzz_trials(model), ref[f"fuzz/{model}"])):
        oc, pr = O.create_camera(model, c["intr"], c["dist"]), c["pr"]
        assert digest(np.array([O.project(oc, p) for p in c["pts"]])) == want["projection"], (model, trial)
        fov = O.estimate_camera_fov(oc, c["W"], c["H"])
        assert fov == want["fov"], (model, trial, c["intr"], c["dist"])
        got = [O.nid_calculate(oc, pr["image"], pr["points"], pr["intensities"], c["bins"], fov, T)[0] for T in c["Ts"]]
        assert all(same(a, b) for a, b in zip(got, want["nid"])), (model, trial, got, want["nid"])
        assert digest(O.view_cull(oc, c["W"], c["H"], fov, True, pr["points"], c["Ts"][0])) == want["cull"]


def test_mode_b_golden_fixtures_match_reference_and_oracle(ref):
    """tests/golden/mode_b_*.npz were written from the reference functor (make_golden.py); the reference build returned
    exactly them and the oracle must reproduce them exactly."""
    for model, g in _fixture_files("mode_b"):
        oc = O.create_camera(model, g["intrinsics"], g["distortion"])
        pts, ins = g["points"].astype(np.float64), g["intensities"].astype(np.float64)
        for k, (tp, want) in enumerate(zip(g["T_params"], ref[f"golden_mode_b/{model}"])):
            ok_o, nid_o, grad_o = O.nid_cost_bspline_grad(oc, g["image"], pts, ins, 16, tp)
            assert want["ok"] and ok_o and nid_o == want["nid_jet"] == g["nid_jet_functor"][k]
            assert want["grad"] == g["grad"][k].tolist() and np.array_equal(grad_o, g["grad"][k])
            assert want["nid_double"] == g["nid_double_functor"][k] == O.nid_cost_bspline(oc, g["image"], pts, ins, 16, tp)[1]


def _lidar_image_problem(model):
    pr = U.random_problem(model, n=30000, seed=5)
    pts = np.concatenate([pr["points"], pr["points"][:2000]])  # exact duplicates: equal squared ranges
    ins = np.concatenate([pr["intensities"], (pr["intensities"][:2000] + 0.5) % 1.0])
    return pr, pts, ins


@pytest.mark.parametrize("model", U.MODELS)
def test_generate_lidar_image_equals_the_reference(ref, model):
    """generate_lidar_image (src/vlcal/preprocess/generate_lidar_image.cpp:8-41): the oracle's intensity image and index map
    equal the reference's own code bit for bit, including the tie rule (of equal squared ranges the last point wins)."""
    pr, pts, ins = _lidar_image_problem(model)
    cam = O.create_camera(model, pr["intrinsics"], pr["distortion"])
    a = O.generate_lidar_image(cam, pr["W"], pr["H"], pr["T"], pts, ins)
    assert [digest(a[0]), digest(a[1])] == ref[f"lidar_image/{model}"]
    assert (a[1] >= 30000).sum() > 100  # duplicates won their pixels


def reference_outputs(R) -> dict:
    """What the reference's code returns for every input above (R: oracle/reference.py over oracle/_ref/libvlcal_ref.so);
    tests/golden/make_reference_outputs.py stores it as tests/golden/reference_outputs.json."""
    out = {}
    for model in U.MODELS:
        intr, dist, (W, H) = U.CAMERAS[model]
        rc = _rcam(R, model)
        out[f"projection/{model}"] = digest(R.project(rc, _projection_points()))
        out[f"fov/{model}"] = [R.estimate_camera_fov(rc, W, H), R.estimate_camera_fov(rc, W // 2 + 1, H // 3)]
        for bins in (16, 8):
            pr, Ts = _nid_problem(model, bins)
            out[f"nid/{model}/{bins}"] = R.nid_calculate(rc, pr["image"], pr["points"], pr["intensities"], bins, Ts).tolist()
        pr, Ts = _cull_problem(model)
        for depth in (True, False):
            out[f"view_cull/{model}/{depth}"] = [digest(R.view_cull(rc, W, H, depth, pr["points"], T)) for T in Ts]
        pr, cases = _bspline_value_cases(model)
        out[f"bspline_value/{model}"] = [list(R.nid_cost_bspline(rc, pr["image"], pr["points"], pr["intensities"], bins, _sophus_params(T))) for bins, T in cases]
        pr, cases = _bspline_grad_cases(model)
        rows = []
        for bins, T in cases:
            ok, nid, g = R.nid_cost_bspline_jet(rc, pr["image"], pr["points"], pr["intensities"], bins, _sophus_params(T))
            rows.append([ok, nid, g.tolist()])
        out[f"bspline_grad/{model}"] = rows
        trials = []
        for c in _fuzz_trials(model):
            fc, pr = R.Camera(model, c["intr"], c["dist"]), c["pr"]
            trials.append({"projection": digest(R.project(fc, c["pts"])), "fov": R.estimate_camera_fov(fc, c["W"], c["H"]),
                           "nid": R.nid_calculate(fc, pr["image"], pr["points"], pr["intensities"], c["bins"], c["Ts"]).tolist(),
                           "cull": digest(R.view_cull(fc, c["W"], c["H"], True, pr["points"], c["Ts"][0]))})
        out[f"fuzz/{model}"] = trials
        pr, pts, ins = _lidar_image_problem(model)
        inten, index = R.generate_lidar_image(R.Camera(model, pr["intrinsics"], pr["distortion"]), pr["W"], pr["H"], pr["T"], pts, ins)
        out[f"lidar_image/{model}"] = [digest(inten), digest(index)]
    out["create_camera"] = {
        "unknown_model_is_null": R.Camera("no_such_model", [1, 1, 1, 1], []).handle is None,
        "short_intrinsics_is_null": R.Camera("plumb_bob", [1, 1, 1], []).handle is None,
        "padded_projection": [R.project(R.Camera("plumb_bob", [400, 410, 320, 240], d), REJECT_POINT).tolist() for d in REJECT_DISTORTIONS],
    }
    for n in (2, 3, 6):
        for name, f in _objectives().items():
            out[f"nelder_mead/{name}/{n}"] = [nm_record(R.nelder_mead(f, x0, **kw)) for x0, kw in _nm_trials(n)]
    pr, cases = _edge_inputs()
    rc = _rcam(R, "plumb_bob")
    out["nid_edge_cases"] = [float(R.nid_calculate(rc, pr["image"], p, i, 16, [pr["T"]])[0]) for p, i in cases]
    for model, g in _fixture_files("mode_a"):
        H, W = g["image"].shape
        fc = R.Camera(model, g["intrinsics"], g["distortion"])
        pts, ins = g["points"].astype(np.float64), g["intensities"].astype(np.float64)
        out[f"golden_mode_a/{model}"] = {"fov": R.estimate_camera_fov(fc, W, H), "nid": R.nid_calculate(fc, g["image"], pts, ins, 16, g["poses"]).tolist(),
                                         "cull": digest(R.view_cull(fc, W, H, True, pts, g["poses"][0]))}
    for model, g in _fixture_files("mode_b"):
        fc = R.Camera(model, g["intrinsics"], g["distortion"])
        pts, ins = g["points"].astype(np.float64), g["intensities"].astype(np.float64)
        rows = []
        for tp in g["T_params"]:
            ok, nid, grad = R.nid_cost_bspline_jet(fc, g["image"], pts, ins, 16, tp)
            rows.append({"ok": ok, "nid_jet": nid, "grad": grad.tolist(), "nid_double": R.nid_cost_bspline(fc, g["image"], pts, ins, 16, tp)[1]})
        out[f"golden_mode_b/{model}"] = rows
    pr = U.random_problem("plumb_bob", n=100, seed=72)
    out["bspline_failure_flag"] = R.nid_cost_bspline(rc, pr["image"], FAR_POINTS, np.full(10, 0.5), 16, _sophus_params(pr["T"]))[0]
    for model, n_bags in ESTIMATE_POSE_CASES:
        bags, T0 = _estimate_pose_problem(model, n_bags)
        out[f"estimate_pose/{model}/{n_bags}"] = calibration_record(R.calibrate_nelder_mead(_rcam(R, model), bags, T0, max_outer_iterations=1, max_inner_iterations=40))
    bags, T0 = _calibrate_problem()
    out["calibrate_outer"] = [R.calibrate_nelder_mead(rc, bags, T0, **kw)["T"].reshape(-1).tolist() for kw in CALIBRATE_KWARGS]
    pr, img, tp = _smooth_problem()
    fc = _rcam(R, "fisheye")
    fd = []
    for k in range(7):
        a, b = tp.copy(), tp.copy()
        a[k] += 1e-6
        b[k] -= 1e-6
        fd.append((R.nid_cost_bspline(fc, img, pr["points"], pr["intensities"], 16, a)[1] - R.nid_cost_bspline(fc, img, pr["points"], pr["intensities"], 16, b)[1]) / 2e-6)
    out["bspline_central_differences"] = fd
    return out
