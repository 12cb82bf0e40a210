"""GPU checks of `assess` and of the persistent kernel's solve axis (vlcal_estimate_poses_nelder_mead_ctx).

Bar: every solve of a multi-solve launch returns the same x, cost, iteration count and evaluation counts as a single-solve
launch from the same start over the same bags (bit for bit); the stencil scores equal the pose-list scores and the
oracle; an assessment of a synthetic scene at its true pose runs end to end."""
import json

import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import CostCalculatorNID, NIDCostParams, VisualLiDARData, VlcalError, create_camera, score_poses
from direct_visual_lidar_calibration_b200 import assess as A
from direct_visual_lidar_calibration_b200 import calibration as _VC
from direct_visual_lidar_calibration_b200 import synthetic as _S
from direct_visual_lidar_calibration_b200._lib import ERR_UNSUPPORTED

pytestmark = pytest.mark.gpu


def _costs(model, n_bags, bins, n=20000):
    costs = []
    for b in range(n_bags):
        pr = util.random_problem(model, n=n + 3001 * b, seed=11 + b)
        cam = create_camera(model, pr["intrinsics"], pr["distortion"])
        costs.append(CostCalculatorNID(cam, VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), NIDCostParams(bins)))
    return costs, pr["T"]


def _shrinks(r):
    # batches: the initial simplex (7 poses), then 3 poses per iteration or 6 per shrink
    return (r["num_evaluations_computed"] - 7 - 3 * (r["num_batches"] - 1)) // 3


@pytest.mark.parametrize("model", ["plumb_bob", "equirectangular"])
@pytest.mark.parametrize("bins", [16, 32])
@pytest.mark.parametrize("n_bags", [1, 3])
def test_solve_axis_equals_single_solves(model, bins, n_bags):
    costs, T = _costs(model, n_bags, bins)
    params = _VC.VisualCameraCalibrationParams()
    params.nid_bins = bins
    sizes = [1, 2, 7, 64] if n_bags == 1 else [1, 2, 7, 40]
    shrinks = 0
    try:
        for S in sizes:
            starts = np.stack(util.random_poses(T, S, seed=S, rot_deg=0.5, trans=0.02))
            mask = np.ones((S, n_bags), dtype=bool)
            if n_bags > 1:  # leave-one-out masks on some solves
                for s in range(1, S, 2):
                    mask[s, s % n_bags] = False
            Ts, rs = _VC.estimate_poses_on_costs(costs, starts, mask, params)
            for s in range(S):
                sub = [c for c, m in zip(costs, mask[s]) if m]
                T1, r1 = _VC.estimate_pose_on_costs(sub, starts[s], params)
                assert np.array_equal(rs[s]["x"], r1["x"]), (S, s)
                assert rs[s]["y"] == r1["y"] or (np.isnan(rs[s]["y"]) and np.isnan(r1["y"]))
                for key in ("num_iterations", "num_evaluations", "num_evaluations_computed", "num_batches", "converged"):
                    assert rs[s][key] == r1[key], (S, s, key)
                assert np.array_equal(Ts[s], T1)
                shrinks += _shrinks(r1) > 0
        assert shrinks > 0  # some solve took a shrink iteration
        for c in costs:
            c.reset_profile()
        _VC.estimate_poses_on_costs(costs, starts, mask, params)
        assert costs[0].profile()["kernel_launches"] == 1  # all S solves in one launch
        # more solves than one launch takes (65 > 64), or than the device holds blocks for (64 x 3 bags > one block per SM)
        with pytest.raises(VlcalError) as e:
            _VC.estimate_poses_on_costs(costs, np.repeat(T[None], 65 if n_bags == 1 else 64, axis=0), None, params)
        assert e.value.code == ERR_UNSUPPORTED
    finally:
        for c in costs:
            c.close()


def test_solve_axis_refuses_double_clouds():
    pr = util.random_problem("plumb_bob", n=5000, seed=3, f32=False)
    cam = create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    cost = CostCalculatorNID(cam, VisualLiDARData(pr["image"], pr["points"], pr["intensities"]))
    try:
        assert not cost.points_are_f32
        with pytest.raises(VlcalError) as e:
            _VC.estimate_poses_on_costs([cost], pr["T"][None])
        assert e.value.code == ERR_UNSUPPORTED
    finally:
        cost.close()


def test_solve_axis_refuses_more_than_32_bins():
    pr = util.random_problem("plumb_bob", n=5000, seed=4)
    cam = create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    cost = CostCalculatorNID(cam, VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), NIDCostParams(33))
    try:
        with pytest.raises(VlcalError) as e:
            _VC.estimate_poses_on_costs([cost], pr["T"][None])
        assert e.value.code == ERR_UNSUPPORTED
    finally:
        cost.close()


def test_stencil_scores_equal_pose_list_and_oracle():
    from oracle import oracle as O

    model = "plumb_bob"
    pr = util.random_problem(model, n=20000, seed=5)
    cam = create_camera(model, pr["intrinsics"], pr["distortion"])
    cost = CostCalculatorNID(cam, VisualLiDARData(pr["image"], pr["points"], pr["intensities"]))
    try:
        poses = A.tangent_poses(pr["T"], np.concatenate([A.profile_offsets(5).reshape(-1, 6), A.hessian_stencil(A.HESSIAN_STEP)]))
        f = score_poses([cost], poses)
        for k in range(0, len(poses), 8):
            np.testing.assert_array_equal(f[k : k + 8], cost.calculate_batch(poses[k : k + 8]))
        ocam = O.create_camera(model, pr["intrinsics"], pr["distortion"])
        fov = O.estimate_camera_fov(ocam, pr["W"], pr["H"])
        for k in (0, 17, 31, len(poses) - 1):
            ref, _ = O.nid_calculate(ocam, pr["image"], pr["points"], pr["intensities"], 16, fov, poses[k])
            assert abs(f[k] - ref) < 1e-12
    finally:
        cost.close()


def test_agreement_map_equals_numpy_from_the_oracle():
    import viewer_oracle as VO
    from oracle import oracle as O

    from direct_visual_lidar_calibration_b200.points_color_updater import agreement_map

    for model, bins in (("plumb_bob", 16), ("equirectangular", 32)):
        pr = util.random_problem(model, n=30000, seed=21)
        cam = create_camera(model, pr["intrinsics"], pr["distortion"])
        T = pr["T"]
        pmi, hist, bgr, index = agreement_map(cam, pr["image"], T, pr["points"], pr["intensities"], bins, point_radius=1, blend_weight=0.7)
        ocam = O.create_camera(model, pr["intrinsics"], pr["distortion"])
        W, H = pr["W"], pr["H"]
        _, ref_hist = O.nid_calculate(ocam, pr["image"], pr["points"], pr["intensities"], bins, O.estimate_camera_fov(ocam, W, H), T)
        np.testing.assert_array_equal(hist, ref_hist)
        cost = CostCalculatorNID(cam, VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), NIDCostParams(bins))
        np.testing.assert_array_equal(cost.calculate_batch(T[None], return_hist=True)[1][0], hist)  # calculate's histogram
        cost.close()
        # numpy: every point's joint bin from the oracle's decision, its PMI from the oracle's histogram
        pix, _ = VO.classify(O, ocam, W, H, VO.cost_cos_fov(O, ocam, W, H), T, pr["points"])
        ib = np.clip(VO._cast_int_x86(pr["image"].reshape(-1)[np.maximum(pix, 0)] / 255.0 * bins), 0, bins - 1)
        lb = np.clip(VO._cast_int_x86(np.asarray(pr["intensities"]) * bins), 0, bins - 1)
        N = ref_hist.sum()
        ca, cb = ref_hist.sum(axis=1), ref_hist.sum(axis=0)
        with np.errstate(all="ignore"):
            ref = np.log((ref_hist[ib, lb] * float(N)) / (ca[ib].astype(np.float64) * cb[lb]))
        ref[pix < 0] = np.nan
        assert np.array_equal(np.isnan(pmi), np.isnan(ref)) and np.isnan(pmi).sum() < len(pmi)
        ok = ~np.isnan(ref)
        assert np.abs(pmi[ok] - ref[ok]).max() < 1e-12
        # the splat: viewer_oracle's z-buffer overlay with the colormap coordinate in place of the intensity
        shade = 0.5 + ref / (2.0 * 2.0)
        ref_bgr, ref_index = VO.overlay(O, ocam, pr["image"], T, pr["points"], shade, 1, 0.7)
        np.testing.assert_array_equal(index, ref_index)
        np.testing.assert_array_equal(bgr, ref_bgr)


def _calibrated(bags, cam):
    data = [VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    T0 = _S.perturb(bags[0]["T_gt"], (0.3, -0.3, 0.3), (0.01, -0.01, 0.01))
    return data, _VC.VisualCameraCalibration(cam, data, _VC.VisualCameraCalibrationParams()).calibrate(T0)


def test_assess_well_textured_scene(tmp_path):
    bags = [_S.make_bag("pinhole_640x480", "frustum", 100_000, config_index=0, bag_index=b) for b in range(3)]
    cam = create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    data, T = _calibrated(bags, cam)
    # starts the inner solve resolves: from 0.5 deg / 2 cm its simplex (init step 1e-3) collapses on the piecewise-constant
    # objective about 2 cm from T (measured), so the return check starts within its reach
    rep = A.assess(cam, data, ["a", "b", "c"], T, starts=8, start_rot_deg=0.1, start_trans=0.002, dst_path=str(tmp_path))
    json.loads(json.dumps(rep))
    sm = rep["summary"]
    print(json.dumps({"summary": sm, "warnings": rep["warnings"], "curvature": rep["local"]["sum"]["curvature"]}))
    assert len(rep["solves"]) == 8 + 3 and [s["kind"] for s in rep["solves"]].count("leave_one_out") == 3
    assert sm["max_trans"] <= A.AWAY_TRANS and sm["max_rot_deg"] <= A.AWAY_ROT_DEG and sm["ended_away"] == 0  # (a)
    assert rep["warnings"] == []  # (b)
    assert all((tmp_path / f"{n}_agreement.png").exists() for n in "abc")


def _stripe_wall(n=150_000, seed=0):
    """A wall 5 m ahead of the LiDAR whose texture varies along LiDAR y only (vertical stripes), and the pinhole image of
    it through the synthetic ground truth: moving along LiDAR z changes nothing."""
    rng = np.random.default_rng(seed)
    stripe = lambda y: 0.5 + 0.45 * np.sin(2.0 * np.pi * y / 0.6)  # noqa: E731
    pts = np.stack([np.full(n, 5.0), rng.uniform(-4, 4, n), rng.uniform(-3, 3, n)], axis=1).astype(np.float32).astype(np.float64)  # float clouds
    T = _S.gt_T_camera_lidar()
    fx, fy, cx, cy, W, H = 400.0, 400.0, 320.0, 240.0, 640, 480
    u, v = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    d_c = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], axis=-1)
    R, t = T[:3, :3], T[:3, 3]
    d_l = d_c @ R  # R^T d per pixel
    o = -R.T @ t
    s = (5.0 - o[0]) / d_l[..., 0]
    image = np.clip(np.rint(stripe(o[1] + s * d_l[..., 1]) * 255.0), 0, 255).astype(np.uint8)
    return [fx, fy, cx, cy], image, np.concatenate([pts, np.ones((n, 1))], axis=1), stripe(pts[:, 1]).astype(np.float32).astype(np.float64), T


def test_assess_flags_the_axis_a_striped_wall_leaves_free():
    intr, image, pts, inten, T = _stripe_wall()
    cam = create_camera("plumb_bob", intr, [0.0, 0.0, 0.0, 0.0, 0.0])
    rep = A.assess(cam, [VisualLiDARData(image, pts, inten)], ["wall"], T, starts=4, start_rot_deg=0.3, start_trans=0.01)
    print(json.dumps({"weak": rep["local"]["sum"]["weak_axes"], "curvature": rep["local"]["sum"]["curvature"], "warnings": rep["warnings"]}))
    assert "tz" in rep["local"]["sum"]["weak_axes"]  # (c): translation along LiDAR z moves along the stripes
    assert "ty" not in rep["local"]["sum"]["weak_axes"]  # across the stripes
    assert any("axis tz is weakly constrained" in w for w in rep["warnings"])
