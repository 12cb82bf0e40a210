"""The CUDA path against the REFERENCE's own code, directly: what the reference's sources of the path (compiled with
oracle/ref_shim.cpp into oracle/_ref/libvlcal_ref.so) return for these problems is stored in
tests/golden/reference_outputs.json (tests/golden/make_reference_outputs.py).  Everything here is also implied by
(CUDA == oracle, tests/test_gpu_parity.py) and (oracle == reference, tests/test_reference_pin.py); this file closes the
triangle without the oracle in between.

`reference_side()` computes the reference's answers; a CPU test checks the stored answers against the oracle so that the
GPU test cannot fail (or pass) because of a mistake in the stored record."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import util
from test_reference_pin import calibration_record, digest, load_golden

NID_TOL = 1e-12
MODELS = ["plumb_bob", "fisheye", "equirectangular"]


def _problem(model="plumb_bob"):
    from direct_visual_lidar_calibration_b200 import synthetic as S

    if model == "plumb_bob":
        bag = S.make_bag("pinhole_640x480", "frustum", 30000, config_index=21, scale=0.5)
        T_init = S.perturb(bag["T_gt"], (0.3, -0.3, 0.3), (0.01, -0.01, 0.01))
        return {"model": bag["camera_model"], "intrinsics": bag["intrinsics"], "distortion": bag["distortion"], "W": bag["width"], "H": bag["height"], "image": bag["image"],
                "points": bag["points"], "intensities": bag["intensities"], "T": T_init}
    return util.random_problem(model, n=20000, seed=31)


def _sophus_params(T):
    return np.concatenate([Rotation.from_matrix(T[:3, :3]).as_quat(), T[:3, 3]])


def _poses(pr):
    return util.random_poses(pr["T"], 3, seed=17, rot_deg=1.0, trans=0.05)


def reference_side(R, pr, inner_iterations=40):
    """What the reference's code returns for this problem (mode A NID at 3 poses, culling, one inner Nelder-Mead solve, a
    two-iteration outer loop, mode B value + gradient)."""
    rc = R.Camera(pr["model"], pr["intrinsics"], pr["distortion"])
    bags = [(pr["image"], pr["points"], pr["intensities"])]
    out = {"fov": R.estimate_camera_fov(rc, pr["W"], pr["H"]), "nid": R.nid_calculate(rc, pr["image"], pr["points"], pr["intensities"], 16, _poses(pr)).tolist(),
           "cull": digest(R.view_cull(rc, pr["W"], pr["H"], True, pr["points"], pr["T"]))}
    out["inner"] = calibration_record(R.calibrate_nelder_mead(rc, bags, pr["T"], max_outer_iterations=1, max_inner_iterations=inner_iterations))
    outer = R.calibrate_nelder_mead(rc, bags, pr["T"], max_outer_iterations=2, max_inner_iterations=inner_iterations, delta_trans_thresh=1e-9, delta_rot_thresh=1e-9)
    out["outer_T"] = outer["T"].reshape(-1).tolist()
    sub = slice(0, 5000)
    ok, nid, grad = R.nid_cost_bspline_jet(rc, pr["image"], pr["points"][sub], pr["intensities"][sub], 16, _sophus_params(pr["T"]))
    out["modeb"] = [ok, nid, grad.tolist()]
    return out


def reference_outputs(R) -> dict:
    return {f"cuda_vs_reference/{model}": reference_side(R, _problem(model)) for model in MODELS}


@pytest.fixture(scope="module")
def ref():
    return load_golden()


def test_reference_side_helper_agrees_with_the_oracle(oracle, ref):
    pr = _problem()
    want = ref["cuda_vs_reference/plumb_bob"]
    O = oracle
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(cam, pr["W"], pr["H"])
    assert fov == want["fov"]
    assert [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], 16, fov, T)[0] for T in _poses(pr)] == want["nid"]
    assert digest(O.view_cull(cam, pr["W"], pr["H"], fov, True, pr["points"], pr["T"])) == want["cull"]
    p = O.default_calib_params()
    p.max_inner_iterations, p.max_outer_iterations = 40, 1
    bags = [(pr["image"], pr["points"], pr["intensities"])]
    assert O.estimate_pose_nelder_mead(cam, bags, pr["T"], p)["T"].reshape(-1).tolist() == want["inner"]["T"]
    p.max_outer_iterations, p.delta_trans_thresh, p.delta_rot_thresh = 2, 1e-9, 1e-9
    assert O.calibrate(cam, bags, pr["T"], p)["T"].reshape(-1).tolist() == want["outer_T"]
    ok, nid, grad = O.nid_cost_bspline_grad(cam, pr["image"], pr["points"][:5000], pr["intensities"][:5000], 16, _sophus_params(pr["T"]))
    assert [ok, nid] == want["modeb"][:2] and grad.tolist() == want["modeb"][2]


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_cuda_path_equals_the_reference_build(gpu, ref, model):
    V = gpu
    pr = _problem(model)
    want = ref[f"cuda_vs_reference/{model}"]
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    data = V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])
    cost = V.CostCalculatorNID(cam, data)
    assert cost.max_fov == want["fov"]
    nid = cost.calculate_batch(_poses(pr))
    assert np.all(np.abs(nid - np.array(want["nid"])) < NID_TOL), np.abs(nid - np.array(want["nid"])).max()
    assert digest(V.ViewCulling(cam, (pr["W"], pr["H"])).cull_indices(pr["points"], pr["T"])) == want["cull"]
    # mode B: value and the 7 partials of the reference functor instantiated with Jets
    ok_r, nid_r, grad_r = want["modeb"]
    grad_r = np.array(grad_r)
    nc = V.NIDCost(cam, V.VisualLiDARData(pr["image"], pr["points"][:5000], pr["intensities"][:5000]), 16)
    ok, nid_b, grad = nc.evaluate_with_gradient(_sophus_params(pr["T"])[None])
    assert bool(ok[0]) == ok_r and abs(nid_b[0] - nid_r) < 1e-9 and np.abs(grad[0] - grad_r).max() < 1e-8 * max(1.0, np.abs(grad_r).max())
    if model != "plumb_bob":
        return  # the solves below replay thousands of comparisons of NID values; they are pinned on the pinhole scene
    # inner solve and outer loop: identical decisions -> identical pose, same number of best-cost callbacks
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 40
    calib = V.VisualCameraCalibration(cam, [data], params)
    T, r = calib.estimate_pose_nelder_mead(pr["T"])
    assert T.reshape(-1).tolist() == want["inner"]["T"] and len(calib.trace) == want["inner"]["num_callbacks"]
    assert digest(np.array([Tg for Tg, _ in calib.trace]).reshape(-1, 4, 4), fold_zeros=True) == want["inner"]["callback_T"]
    params.max_outer_iterations, params.delta_trans_thresh, params.delta_rot_thresh = 2, 1e-9, 1e-9
    T2 = V.VisualCameraCalibration(cam, [data], params).calibrate(pr["T"])
    assert np.abs(T2 - np.array(want["outer_T"]).reshape(4, 4)).max() < 1e-15
