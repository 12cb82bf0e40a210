"""The pose sweep kernel (vlcal_nid_sweep_poses / _search_set) against the oracle and against the existing evaluators, and
initial_guess_search end to end on synthetic bags whose ground truth it is not told."""
import os

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import util
from direct_visual_lidar_calibration_b200 import _lib
from direct_visual_lidar_calibration_b200 import initial_guess as ig
from direct_visual_lidar_calibration_b200 import initial_guess_search as igs
from direct_visual_lidar_calibration_b200 import io as vio
from direct_visual_lidar_calibration_b200 import synthetic as S
from search_oracle import OracleScorer
from test_gpu_round1_edges import DYADIC_PINHOLE, _edge_cloud, _edge_intensities, _grey_ramp, _pr_from_points, _special_points, _translations

pytestmark = pytest.mark.gpu

THREADS = 256  # threads of one sweep block


def _cost(V, pr, bins=16):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    return V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), V.NIDCostParams(bins))


def _oracle_eval(O, pr, Ts, bins=16):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(cam, pr["W"], pr["H"])
    out = [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], bins, fov, T, omp=pr["points"].shape[0] > 4096) for T in Ts]
    return np.array([o[0] for o in out]), np.stack([o[1] for o in out])


def _problem(model, n, seed):
    pr = util.random_problem(model, n=max(n, 16), seed=seed)
    pr["points"], pr["intensities"] = pr["points"][:n], pr["intensities"][:n]
    return pr


def _wide_poses(T, count, seed):
    """Poses spread as a global search spreads them: a third near T, the rest anywhere."""
    near = util.random_poses(T, count, seed=seed, rot_deg=8.0, trans=0.3)
    far = Rotation.random(count, random_state=seed).as_matrix()
    out = near.copy()
    out[2::3, :3, :3] = far[2::3]
    return out


def _check(cost, O, pr, Ts, bins=16, oracle_rows=None):
    """sweep == calculate_batch bit for bit (NID and histograms); histograms and NaN pattern == the oracle's."""
    nid, hist = ig.sweep_poses([cost], Ts, return_hist=True)
    ref_nid, ref_hist = cost.calculate_batch(Ts, return_hist=True)
    assert np.array_equal(hist, ref_hist)
    assert np.array_equal(nid, ref_nid, equal_nan=True)
    rows = np.arange(len(Ts)) if oracle_rows is None else oracle_rows
    o_nid, o_hist = _oracle_eval(O, pr, Ts[rows], bins)
    assert np.array_equal(hist[rows], o_hist)
    assert np.array_equal(np.isnan(nid[rows]), np.isnan(o_nid))
    m = ~np.isnan(o_nid)
    assert np.all(np.abs(nid[rows][m] - o_nid[m]) < 1e-12)
    return nid


@pytest.mark.parametrize("model", util.MODELS)
def test_sweep_equals_oracle_over_cloud_sizes(gpu, oracle, model):
    for n in (0, 1, 31, 32, 33, THREADS - 1, THREADS, THREADS + 1, 16384, 65536 + 1):
        pr = _problem(model, n, seed=100 + n % 97)
        nid = _check(_cost(gpu, pr), oracle, pr, _wide_poses(pr["T"], 9, seed=n), oracle_rows=None if n <= 16384 else np.arange(3))
        assert n > 0 or np.isnan(nid).all()


@pytest.mark.parametrize("model", util.MODELS)
def test_sweep_equals_oracle_over_pose_counts(gpu, oracle, model):
    pr = _problem(model, 3000, seed=7)
    cost = _cost(gpu, pr)
    blocks, per_block = _lib.C.c_int(), _lib.C.c_int()
    _lib.check(_lib.load_library().vlcal_nid_sweep_launch_shape(cost.handle, _lib.C.byref(blocks), _lib.C.byref(per_block)))
    assert blocks.value >= 1 and per_block.value >= 1
    for P in (1, 7, 8, 9, 1000, blocks.value * per_block.value + 1):  # the last: one block takes a second group, of one pose
        Ts = _wide_poses(pr["T"], P, seed=P)
        _check(cost, oracle, pr, Ts, oracle_rows=None if P <= 9 else np.r_[0:4, P - 3 : P])


def test_a_list_where_no_pose_sees_a_point(gpu, oracle):
    pr = _problem("plumb_bob", 5000, seed=3)
    pr["points"] = pr["points"][pr["points"][:, 0] > 1.0]  # all in front of the LiDAR
    pr["intensities"] = pr["intensities"][: pr["points"].shape[0]]
    back = pr["T"].copy()
    back[:3, :3] = np.diag([-1.0, 1.0, -1.0]) @ back[:3, :3]  # the camera looks the other way
    Ts = util.random_poses(back, 13, seed=1, rot_deg=1.0, trans=0.01)
    nid = _check(_cost(gpu, pr), oracle, pr, Ts)
    assert np.isnan(nid).all()


@pytest.mark.parametrize("offset_px", [1e-7, 0.0])
def test_points_on_truncation_and_image_edges(gpu, oracle, offset_px):
    """Every point within offset_px of a column edge at every pose (dyadic pinhole: the projection is exact), plus the
    special points on the (-1, 0) strip, the last row / column and the FoV edge: almost everything takes the queue to the
    exact path."""
    rng = np.random.default_rng(40)
    intr, dist = DYADIC_PINHOLE
    pts = np.concatenate([_edge_cloud(40, 8, rng), _special_points(640, 480).astype(np.float32).astype(np.float64)])
    pts = pts[np.isfinite(pts).all(axis=1)]
    pr = _pr_from_points("plumb_bob", pts, seed=41, intr=intr, dist=dist)
    pr["image"] = _grey_ramp(pr["W"], pr["H"])
    pr["intensities"] = _edge_intensities(16, pts.shape[0], rng, f32=True)
    Ts = _translations(np.eye(4), [(offset_px / 512.0, 1e-5 * k, 0.0) for k in range(6)])
    _check(_cost(gpu, pr), oracle, pr, Ts)


def test_fov_edge_equirectangular_and_fisheye(gpu, oracle):
    for model in ("equirectangular", "fisheye"):
        rng = np.random.default_rng(50)
        pts = _edge_cloud(30, 4, rng, model="equirectangular")  # x = 0: the seam and the centre column
        pr = _pr_from_points(model, pts, seed=51)
        _check(_cost(gpu, pr), oracle, pr, _translations(np.eye(4), [(0.0, 1e-5 * k, 0.0) for k in range(5)]))


def test_several_bags_sum_in_bag_order(gpu, oracle):
    from direct_visual_lidar_calibration_b200.cost import score_poses

    prs = [_problem("plumb_bob", n, seed=60 + i) for i, n in enumerate((5000, 777, 0))]
    for pr in prs[1:]:
        pr["image"] = np.ascontiguousarray(np.roll(prs[0]["image"], 17, axis=1))
    costs = [_cost(gpu, pr) for pr in prs]
    Ts = _wide_poses(prs[0]["T"], 50, seed=5)
    two = ig.sweep_poses(costs[:2], Ts)
    assert np.array_equal(two, score_poses(costs[:2], Ts), equal_nan=True)
    singles = [ig.sweep_poses([c], Ts) for c in costs[:2]]
    assert np.array_equal(two, (0.0 + singles[0]) + singles[1], equal_nan=True)
    three = ig.sweep_poses(costs, Ts)  # the empty bag's NaN reaches every sum
    assert np.array_equal(three, score_poses(costs, Ts), equal_nan=True) and np.isnan(three).all()
    swapped = ig.sweep_poses(costs[1::-1], Ts)
    assert np.array_equal(swapped, score_poses(costs[1::-1], Ts), equal_nan=True)


@pytest.mark.parametrize("bins", [8, 32])
def test_other_bin_counts(gpu, oracle, bins):
    pr = _problem("omnidir", 4000, seed=70)
    pr["intensities"] = _edge_intensities(bins, 4000, np.random.default_rng(71), f32=True)
    cam = gpu.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    cost = gpu.CostCalculatorNID(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), gpu.NIDCostParams(bins))
    _check(cost, oracle, pr, _wide_poses(pr["T"], 10, seed=2), bins=bins)


def test_refusals(gpu):
    pr = _problem("plumb_bob", 1000, seed=80)
    Ts = util.random_poses(pr["T"], 3)
    cam = gpu.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    wide = gpu.CostCalculatorNID(cam, gpu.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), gpu.NIDCostParams(64))
    with pytest.raises(gpu.VlcalError, match="bins = 64 exceeds 32") as e:
        ig.sweep_poses([wide], Ts)
    assert e.value.code == _lib.ERR_UNSUPPORTED
    prd = util.random_problem("plumb_bob", n=1000, seed=81, f32=False)
    double = _cost(gpu, prd)
    assert not double.points_are_f32
    with pytest.raises(gpu.VlcalError, match="double layout") as e:
        ig.sweep_poses([double], Ts)
    assert e.value.code == _lib.ERR_UNSUPPORTED
    other = _problem("fisheye", 1000, seed=82)
    with pytest.raises(gpu.VlcalError, match="must share") as e:
        ig.sweep_poses([_cost(gpu, pr), _cost(gpu, other)], Ts)
    assert e.value.code == _lib.ERR_UNSUPPORTED


def test_device_generated_search_sets_equal_the_host_lists_bit_for_bit(gpu):
    prior = np.eye(4)
    prior[:3, :3] = Rotation.from_rotvec([0.3, -1.1, 0.7]).as_matrix()
    prior[:3, 3] = [0.11, -0.23, 0.35]
    sets = [ig.rotation_set(9.0), ig.rotation_set(7.0, prior, 35.0)]
    cands = sets[1].poses(np.arange(0, sets[1].n_poses, max(1, sets[1].n_poses // 5)))
    sets += [ig.local_set(cands, 1.5, 0.15, 2), ig.local_set(cands[:2], 0.1875, 0.01875, 1)]
    for s in sets:
        host, dev = s.poses(), s.device_poses()
        assert host.shape == dev.shape == (s.n_poses, 4, 4)
        assert np.array_equal(host.view(np.uint64), dev.view(np.uint64))
    # and the scores of a set are the scores of its list
    pr = _problem("plumb_bob", 2000, seed=90)
    cost = _cost(gpu, pr)
    scores, inliers, kernel_ms = ig.sweep_search_set([cost], sets[2])
    assert kernel_ms > 0.0
    _, hist = ig.sweep_poses([cost], sets[2].poses(), return_hist=True)
    assert np.array_equal(inliers, hist.reshape(len(hist), -1).sum(axis=1))
    assert np.array_equal(scores, ig.sweep_poses([cost], sets[2].poses()), equal_nan=True)


def test_large_clouds_take_the_persistent_kernel(gpu):
    from direct_visual_lidar_calibration_b200.cost import score_poses

    L = _lib.load_library()
    limit = int(L.vlcal_nid_sweep_max_points())
    pr = util.random_problem("plumb_bob", n=limit + 1, seed=95)
    cost = _cost(gpu, pr)
    Ts = _wide_poses(pr["T"], 20, seed=3)
    nid = ig.sweep_poses([cost], Ts)
    assert L.vlcal_nid_sweep_last_kernel_ms() == 0.0  # not the sweep kernel
    assert np.array_equal(nid, score_poses([cost], Ts), equal_nan=True)
    assert np.array_equal(nid, ig.sweep_poses([cost], Ts, kernel_only=True), equal_nan=True)
    assert L.vlcal_nid_sweep_last_kernel_ms() > 0.0
    local = ig.local_set(Ts[:2], 1.0, 0.1, 1)
    scores, inliers, _ = ig.sweep_search_set([cost, cost], local)
    assert np.array_equal(scores, score_poses([cost, cost], local.poses()), equal_nan=True)
    _, hist = cost.calculate_batch(local.poses(), return_hist=True)
    assert np.array_equal(inliers, 2 * hist.reshape(len(hist), -1).sum(axis=1))


# ---- the search, end to end ------------------------------------------------------------------------------------------------------

def _angle_deg(A, B):
    return float(ig.rotation_angle_deg(A[:3, :3], B[:3, :3]))


def _moved(bag, seed):
    """The same scene with the LiDAR frame turned by ~40 deg about a seeded axis and shifted by 0.15 m: the cloud moves
    into the new frame (re-rounded to float32), the image stays, the ground truth follows."""
    rng = np.random.default_rng(seed)
    axis, shift = rng.normal(size=3), rng.normal(size=3)
    M = np.eye(4)
    M[:3, :3] = Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.radians(40.0)).as_matrix()
    M[:3, 3] = 0.15 * shift / np.linalg.norm(shift)
    pts = (bag["points"][:, :3] @ M[:3, :3].T + M[:3, 3]).astype(np.float32).astype(np.float64)
    out = dict(bag)
    out["points"] = np.ascontiguousarray(np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1))
    out["T_gt"] = bag["T_gt"] @ vio.invert_isometry(M)
    return out


def _search(gpu, bag, **kw):
    scorer = igs.SweepScorer(bag["camera_model"], bag["intrinsics"], bag["distortion"], [gpu.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])])
    try:
        return igs.run_search(scorer, log=lambda *_: None, **kw)
    finally:
        scorer.close()


E2E_BAGS = {"pinhole": ("pinhole_1920x1080", "os1_64"), "equirectangular": ("equirect_3840x1920", "sphere")}


@pytest.fixture(scope="module", params=list(E2E_BAGS))
def e2e_bag(request):
    key, pattern = E2E_BAGS[request.param]
    return S.make_bag(key, pattern, 200_000, config_index=9)


def test_search_without_a_prior_finds_the_ground_truth(gpu, e2e_bag):
    for bag in (e2e_bag, _moved(e2e_bag, seed=11)):
        rep = _search(gpu, bag)
        T = rep["T_camera_lidar"]
        assert _angle_deg(T, bag["T_gt"]) < 1.0
        assert np.linalg.norm(vio.invert_isometry(T)[:3, 3] - vio.invert_isometry(bag["T_gt"])[:3, 3]) < 0.05
        assert rep["levels"][0]["poses"] == np.prod(ig.rotation_set_counts(3.0)) and rep["levels"][-1]["scale"] == 1


def test_search_around_a_prior_25_degrees_off(gpu, e2e_bag):
    bag = _moved(e2e_bag, seed=12)
    prior = vio.invert_isometry(S.perturb(bag["T_gt"], (14.0, -15.0, 14.5), (0.1, -0.1, 0.05)))
    assert 24.0 < _angle_deg(prior, vio.invert_isometry(bag["T_gt"])) < 26.0
    rep = _search(gpu, bag, prior_T_lidar_camera=prior, rot_range_deg=40.0)
    T = rep["T_camera_lidar"]
    assert rep["levels"][0]["poses"] < 0.1 * np.prod(ig.rotation_set_counts(3.0))
    assert _angle_deg(T, bag["T_gt"]) < 1.0
    assert np.linalg.norm(vio.invert_isometry(T)[:3, 3] - vio.invert_isometry(bag["T_gt"])[:3, 3]) < 0.05


def test_toy_search_equals_the_checker_level_by_level(gpu, oracle):
    bag = _moved(S.make_bag("pinhole_640x480", "frustum", 4000, config_index=9, bag_index=1), seed=13)
    kw = dict(rot_step_deg=20.0, keep=8, trans_range=0.3)
    rep = _search(gpu, bag, **kw)
    checker = OracleScorer(oracle, bag["camera_model"], bag["intrinsics"], bag["distortion"], [(bag["image"], bag["points"], bag["intensities"])])
    ref = igs.run_search(checker, log=lambda *_: None, **kw)
    assert len(rep["candidates"]) == len(ref["candidates"]) >= 5
    for level, (a, b) in enumerate(zip(rep["candidates"], ref["candidates"])):
        # the same candidates with the same scores; poses whose scores agree to the last few bits may swap places, because
        # the oracle adds the entropy terms in another order than the kernels
        assert a["poses"].shape == b["poses"].shape, level
        ka = np.lexsort(a["poses"].reshape(len(a["poses"]), -1).T)
        kb = np.lexsort(b["poses"].reshape(len(b["poses"]), -1).T)
        assert np.array_equal(a["poses"][ka], b["poses"][kb]), level
        assert np.abs(a["nid"][ka] - b["nid"][kb]).max() < 1e-12, level
        assert np.abs(a["nid"] - b["nid"]).max() < 1e-12, level
    assert np.array_equal(rep["T_camera_lidar"], ref["T_camera_lidar"])


def test_cli_then_calibrate(gpu, oracle, tmp_path, capsys):
    from direct_visual_lidar_calibration_b200 import calibrate as calib_cli

    bags = S.write_initial_guess_dataset(str(tmp_path), n_bags=2, seed=5)
    for b in range(2):
        os.remove(tmp_path / f"bag{b}_matches.json")  # nothing from a matcher
    assert calib_cli.main([str(tmp_path)]) == 1  # no initial guess yet
    capsys.readouterr()
    assert igs.main([str(tmp_path)]) == 0
    out = capsys.readouterr().out
    assert "level 0: 1/8 image" in out and "--- T_lidar_camera ---" in out
    cfg = vio.load_calib_json(str(tmp_path))
    assert set(cfg) == {"camera", "meta", "results"} and list(cfg["results"]) == ["init_T_lidar_camera_auto"]
    T_gt = bags[0]["T_gt"]
    T_init = vio.invert_isometry(vio.tum_to_T(cfg["results"]["init_T_lidar_camera_auto"]))
    assert _angle_deg(T_init, T_gt) < 1.0 and np.linalg.norm(T_init[:3, 3] - T_gt[:3, 3]) < 0.05
    assert os.path.exists(tmp_path / "initial_guess_search.json")
    assert calib_cli.main([str(tmp_path), "--registration_type", "nid_nelder_mead"]) == 0
    cfg = vio.load_calib_json(str(tmp_path))
    T = vio.invert_isometry(vio.tum_to_T(cfg["results"]["T_lidar_camera"]))
    assert _angle_deg(T, T_gt) < 0.5 and np.linalg.norm(T[:3, 3] - T_gt[:3, 3]) < 0.03
    ocam = oracle.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    ref = oracle.calibrate(ocam, [(b["image"], b["points"], b["intensities"]) for b in bags], T_init)
    assert np.abs(T - ref["T"]).max() < 1e-9
