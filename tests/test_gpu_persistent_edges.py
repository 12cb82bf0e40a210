"""GPU edge suite of the persistent cooperative kernel (K1p, csrc/nid_persistent.cuh): the kernel that scores every pose
list (calculate_batch, score_poses) and runs every Nelder-Mead inner solve by default, held to the CPU oracle at the
shapes, pose counts, bag partitions, bin counts and point placements where its bookkeeping could go wrong.

Bar (the suite's): integer histograms bit-identical to oracle.nid_calculate, NID within 1e-12 of the oracle with NaN
exactly where the oracle has NaN, and bit-identical results across K1p configurations (poses per pass, bag grouping,
solver modes).  Every case also checks cost.profile() to show that it ran the path it is meant to test -- one
persistent launch per call, the expected passes, deferred point-poses, delta passes."""
import math

import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import calibration as _VC
from direct_visual_lidar_calibration_b200 import synthetic as _S

pytestmark = pytest.mark.gpu
NID_TOL = 1e-12
PK_THREADS = 768  # threads per block; pk_grid_size asks for ceil(N / 768) blocks, capped at one block per SM
PK_WARPS = 24
TILE_K2, TILE_K4 = 64, 128  # 32 lanes x K points per lane
DYADIC_PINHOLE = ([512.0, 512.0, 320.0, 240.0], [])  # plumb_bob without distortion: u = 512 x / z + 320 is exact for dyadic points


@pytest.fixture(scope="module")
def sms():
    import torch

    return int(torch.cuda.get_device_properties(0).multi_processor_count)


def _cost(V, pr, bins=16):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    return V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), V.NIDCostParams(bins))


def _oracle_eval(O, pr, Ts, bins=16):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(cam, pr["W"], pr["H"])
    big = pr["points"].shape[0] * len(Ts) > 2_000_000
    out = [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], bins, fov, T, omp=big) for T in Ts]
    return np.array([o[0] for o in out]), np.stack([o[1] for o in out])


def _assert_nid(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    m = ~np.isnan(a)
    assert np.all(np.abs(a[m] - b[m]) < NID_TOL), np.abs(a[m] - b[m]).max()


def _assert_matches_oracle(O, pr, Ts, nid, hist, bins=16):
    ref_nid, ref_hist = _oracle_eval(O, pr, Ts, bins)
    assert int(np.abs(hist.astype(np.int64) - ref_hist).sum()) == 0
    _assert_nid(nid, ref_nid)
    return ref_nid, ref_hist


def _scored(cost, Ts, chunk=8):
    """calculate_batch with the histograms, asserting that it was ONE persistent launch of ceil(P / chunk) passes."""
    cost.reset_profile()
    nid, hist = cost.calculate_batch(Ts, return_hist=True)
    prof = cost.profile()
    assert prof["kernel_launches"] == 1 and prof["passes"] == -(-len(Ts) // chunk), prof
    return nid, hist, prof


def _problem(model, n, seed, **kw):
    if n == 0:
        pr = util.random_problem(model, n=16, seed=seed, **kw)
        pr["points"], pr["intensities"] = pr["points"][:0], pr["intensities"][:0]
        return pr
    return util.random_problem(model, n=n, seed=seed, **kw)


def _shape_sizes(sms, tile):
    """Cloud sizes at the kernel's bookkeeping edges: empty, one tile +- 1, one tile per warp of a block, one block,
    the grid's saturation (one block per SM) and clouds where every warp of the saturated grid owns exactly k tiles."""
    warps = sms * PK_WARPS
    edges = {0, 1, 2, tile - 1, tile, tile + 1, PK_WARPS * tile - 1, PK_WARPS * tile + 1, PK_THREADS - 1, PK_THREADS + 1, sms * PK_THREADS - 1, sms * PK_THREADS + 1}
    for k in (1, 2):
        edges |= {warps * tile * k - 1, warps * tile * k, warps * tile * k + 1}
    return sorted(edges)


# ---- 1. shapes ---------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("model", util.MODELS)
def test_shapes_at_tile_block_and_grid_edges(gpu, oracle, sms, model):
    for i, n in enumerate(_shape_sizes(sms, TILE_K2)):
        pr = _problem(model, n, seed=100 + i)
        Ts = util.random_poses(pr["T"], 17, seed=i)  # chunks of 8 + 8 + 1
        nid, hist, _ = _scored(_cost(gpu, pr), Ts)
        _assert_matches_oracle(oracle, pr, Ts, nid, hist)
        if n > 1000:
            assert hist.sum() > 0.2 * n, (n, hist.sum())


@pytest.mark.parametrize("model", ["plumb_bob", "omnidir", "rational_polynomial"])
def test_shapes_with_four_points_per_lane(gpu, oracle, sms, model):
    """set_kernel_variant(3): 128-point tiles (the models whose classifier is light enough for K = 4)."""
    for i, n in enumerate(s for s in _shape_sizes(sms, TILE_K4) if s not in (0, 1, 2)):
        pr = _problem(model, n, seed=200 + i)
        Ts = util.random_poses(pr["T"], 17, seed=i)
        cost = _cost(gpu, pr)
        nid2, hist2, _ = _scored(cost, Ts)
        assert cost.last_points_per_lane() == 2
        cost.set_kernel_variant(3)
        nid4, hist4, _ = _scored(cost, Ts)
        assert cost.last_points_per_lane() == 4
        assert np.array_equal(hist2, hist4) and np.array_equal(nid2, nid4, equal_nan=True)
        if i % 3 == 0:
            _assert_matches_oracle(oracle, pr, Ts, nid4, hist4)


def test_cloud_larger_than_l2_serpentine_passes(gpu, oracle):
    """4e6 points (64 MB of float4, above the H100's 50 MB L2): one pose per pass, so the passes alternate forward and
    backward over every warp's tiles; the counts must not depend on the order."""
    pr = util.random_problem("plumb_bob", n=4_000_000, seed=300)
    Ts = util.random_poses(pr["T"], 3, seed=1)
    cost = _cost(gpu, pr)
    cost.set_poses_per_pass(1)
    nid, hist, _ = _scored(cost, Ts, chunk=1)
    _assert_matches_oracle(oracle, pr, Ts, nid, hist)
    cost.set_poses_per_pass(8)
    nid8, hist8, _ = _scored(cost, Ts)
    assert np.array_equal(hist, hist8) and np.array_equal(nid, nid8)


# ---- 2. pose lists -----------------------------------------------------------------------------------------------------


def test_pose_list_lengths_and_poses_per_pass(gpu, oracle):
    pr = util.random_problem("plumb_bob", n=30000, seed=400)
    Ts = util.random_poses(pr["T"], 1000, seed=2, rot_deg=3.0, trans=0.2)
    cost = _cost(gpu, pr)
    nid, hist, _ = _scored(cost, Ts)  # 125 chunks: the two-ahead gate and both accumulator buffers cycle many times
    ref_nid, ref_hist = _assert_matches_oracle(oracle, pr, Ts, nid, hist)
    for P in list(range(1, 18)) + [64]:  # every list is a prefix of the long one
        n, h, _ = _scored(cost, Ts[:P])
        assert np.array_equal(h, ref_hist[:P])
        assert np.array_equal(n, nid[:P], equal_nan=True)
    for k in range(1, 9):
        cost.set_poses_per_pass(k)
        for P in (1, 17, 37):
            n, h, _ = _scored(cost, Ts[:P], chunk=k)
            assert np.array_equal(h, ref_hist[:P]) and np.array_equal(n, nid[:P], equal_nan=True), (k, P)


def test_empty_pose_list_is_refused_before_any_launch(gpu):
    pr = util.random_problem("plumb_bob", n=5000, seed=401)
    cost = _cost(gpu, pr)
    cost.reset_profile()
    for call in (lambda: cost.calculate_batch(np.zeros((0, 4, 4))), lambda: cost.calculate_batch(np.zeros((0, 4, 4)), return_hist=True),
                 lambda: gpu.score_poses([cost], np.zeros((0, 4, 4)))):
        with pytest.raises(gpu.VlcalError) as e:
            call()
        assert e.value.code == -1
    assert cost.profile()["kernel_launches"] == 0
    nid, hist, _ = _scored(cost, pr["T"][None])  # the context is still usable
    assert hist.sum() > 1000


# ---- 3. bags -----------------------------------------------------------------------------------------------------------


def _bag_problems(sizes, seed):
    """Bags of one camera and image size, each with its own cloud and image.  The points of bags of 1 ... 64 points lie
    5 m in front of the camera near the image centre, so that they are inliers at every pose of the tests and those
    bags have a finite score (a bag with no inlier scores NaN, and so does every sum that holds it)."""
    out = []
    for b, n in enumerate(sizes):
        pr = _problem("plumb_bob", n, seed=seed + b)
        if 0 < n <= 64:
            rng = np.random.default_rng(seed + b)
            pc = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n), np.full(n, 5.0)], axis=1)
            R, t = pr["T"][:3, :3], pr["T"][:3, 3]
            pr["points"][:, :3] = ((pc - t) @ R).astype(np.float32).astype(np.float64)  # cloud frame
        out.append(pr)
    return out


def _sum_in_bag_order(parts):
    s = np.zeros_like(parts[0])
    for p in parts:
        s = s + p
    return s


@pytest.mark.parametrize("sizes", [
    [300_000, 64, 20_000, 1_537, 100_000, 65, 5_000, 300],
    [1_000_000, 1, 64, 250_000, 2, 40_000, 769, 0],
])
def test_score_poses_on_one_to_eight_unequal_bags(gpu, oracle, sizes):
    """Every prefix of the bag list in one launch: each bag's score equal to its own calculate_batch (itself held to the
    oracle), summed in bag order.  Every bag but the empty one scores finite at every pose, so the sums of 1 ... 7 bags
    compare numbers; the empty bag, last, makes the 8-bag sum NaN at exactly every pose."""
    prs = _bag_problems(sizes, seed=500 + len(sizes) + sizes[0] % 7)
    costs = [_cost(gpu, pr) for pr in prs]
    Ts = util.random_poses(prs[0]["T"], 17, seed=3)
    alone = []
    for pr, c in zip(prs, costs):
        nid, hist, _ = _scored(c, Ts)
        _assert_matches_oracle(oracle, pr, Ts, nid, hist)
        assert np.isfinite(nid).all() == (pr["points"].shape[0] > 0), (pr["points"].shape[0], nid)
        alone.append(nid)
    for n_bags in range(1, 9):
        costs[0].reset_profile()
        got = gpu.score_poses(costs[:n_bags], Ts)
        prof = costs[0].profile()
        assert prof["kernel_launches"] == 1 and prof["passes"] == 3, (n_bags, prof)
        want = _sum_in_bag_order(alone[:n_bags])
        assert np.isfinite(want).all() == (min(sizes[:n_bags]) > 0)
        assert np.array_equal(got, want, equal_nan=True), n_bags
    assert np.isnan(got).all() == (0 in sizes)
    # nine bags exceed one launch (PK_MAX_BAGS = 8): the per-bag kernels, same numbers
    extra = _cost(gpu, _problem("plumb_bob", 3_000, seed=599))
    extra_nid = extra.calculate_batch(Ts)
    costs[0].reset_profile()
    got = gpu.score_poses(costs + [extra], Ts)
    assert costs[0].profile()["kernel_launches"] == 3  # one round-1 launch per 8 poses
    assert np.array_equal(got, _sum_in_bag_order(alone + [extra_nid]), equal_nan=True)
    # nine bags that all score finite (the empty one left out), so that the fallback's sum compares numbers too
    extra2 = _cost(gpu, _problem("plumb_bob", 4_000, seed=598))
    nine = [(c, a) for c, a, n in zip(costs, alone, sizes) if n > 0] + [(extra, extra_nid), (extra2, extra2.calculate_batch(Ts))]
    nine = nine[-9:]
    costs_9 = [c for c, _ in nine]
    costs_9[0].reset_profile()
    got = gpu.score_poses(costs_9, Ts)
    assert costs_9[0].profile()["kernel_launches"] == 3
    want = _sum_in_bag_order([a for _, a in nine])
    assert np.isfinite(want).all() and np.array_equal(got, want)


def test_score_poses_eight_bags_eight_poses_32_bins(gpu, oracle):
    """The every-block finalizer's worst case in pose-list mode: 8 bags x 8 poses of 32 x 32 bins."""
    prs = _bag_problems([20_000 + 3_000 * b for b in range(8)], seed=520)
    costs = [_cost(gpu, pr, bins=32) for pr in prs]
    Ts = util.random_poses(prs[0]["T"], 17, seed=4)
    alone = []
    for pr, c in zip(prs, costs):
        nid, hist, _ = _scored(c, Ts)
        _assert_matches_oracle(oracle, pr, Ts[:8], nid[:8], hist[:8], bins=32)
        alone.append(nid)
    assert np.array_equal(gpu.score_poses(costs, Ts), _sum_in_bag_order(alone), equal_nan=True)


def _synthetic_bag(n, cfg, scale=0.5):
    bag = _S.make_bag("pinhole_640x480", "frustum", n, config_index=cfg, scale=scale)
    bag["T_init"] = _S.perturb(bag["T_gt"], (0.3, -0.3, 0.3), (0.01, -0.01, 0.01))
    return bag


def _solve_modes(V, cam, datasets, T0, params, modes=(1, 3)):
    out = {}
    try:
        _VC.record_solve_trace(True)
        for mode in modes:
            V.set_solver_mode(mode)
            calib = V.VisualCameraCalibration(cam, datasets, params)
            T, r = calib.estimate_pose_nelder_mead(T0)
            out[mode] = (T, r, [c for _, c in calib.trace], _VC.last_solve_trace())
            assert len(out[mode][3]) == r["num_evaluations"] > 0
    finally:
        V.set_solver_mode(0)
        _VC.record_solve_trace(False)
    return out


def _assert_same_solve(a, b):
    (Ta, ra, ca, tra), (Tb, rb, cb, trb) = a, b
    assert np.array_equal(Ta, Tb) and np.array_equal(ra["x"], rb["x"])
    assert ra["y"] == rb["y"] or (math.isnan(ra["y"]) and math.isnan(rb["y"]))
    assert ra["num_iterations"] == rb["num_iterations"] and ra["num_evaluations"] == rb["num_evaluations"] and ra["converged"] == rb["converged"]
    assert np.array_equal(np.asarray(ca), np.asarray(cb), equal_nan=True)
    assert np.array_equal(tra, trb, equal_nan=True)


def _assert_trace_is_oracles(got, ref):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.array_equal(got[:, :6], ref[:, :6])
    _assert_nid(got[:, 6], ref[:, 6])


def _oracle_solve(O, cam_args, datasets, T0, iters, bins=16, criterion=None):
    ocam = O.create_camera(*cam_args)
    op = O.default_calib_params()
    op.max_inner_iterations, op.nid_bins = iters, bins
    if criterion is not None:
        op.nelder_mead_convergence_criteria = criterion
    return O.estimate_pose_nelder_mead(ocam, [(d.image, d.points, d.intensities) for d in datasets], T0, op)


def test_persistent_solve_eight_bags_32_bins(gpu, oracle):
    V = gpu
    bags = [_synthetic_bag(8_000 + 1_500 * k, cfg=3 + k % 4) for k in range(8)]
    cam_args = (bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    cam = V.create_camera(*cam_args)
    ds = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations, params.nid_bins = 25, 32
    out = _solve_modes(V, cam, ds, bags[0]["T_init"], params)
    _assert_same_solve(out[1], out[3])
    ref = _oracle_solve(oracle, cam_args, ds, bags[0]["T_init"], 25, bins=32)
    Tp, rp, _, trp = out[3]
    assert np.array_equal(rp["x"], ref["x"]) and rp["num_evaluations"] == ref["num_evaluations"] and np.abs(Tp - ref["T"]).max() == 0.0
    _assert_trace_is_oracles(trp, ref["trace"])


def _tiny_bag(V, bag, n, seed):
    """n points 4 .. 6 m in front of the camera near the image centre at bag["T_init"]: inliers at every pose of a solve
    from there, so the bag scores finite."""
    rng = np.random.default_rng(seed)
    pc = np.stack([rng.uniform(-0.3, 0.3, n), rng.uniform(-0.3, 0.3, n), rng.uniform(4.0, 6.0, n)], axis=1)
    R, t = bag["T_init"][:3, :3], bag["T_init"][:3, 3]
    pts = ((pc - t) @ R).astype(np.float32).astype(np.float64)
    return V.VisualLiDARData(bag["image"][::-1].copy(), pts, rng.integers(0, 256, n) / 256.0)


def test_persistent_solve_with_one_and_64_point_bags(gpu, oracle):
    """A 20 000-point bag with a 1-point and a 64-point bag in one launch (each gets at least one block of the grid);
    every bag scores finite, so the trajectory follows the sum of three real scores."""
    V = gpu
    b1 = _synthetic_bag(20_000, cfg=4)
    cam_args = (b1["camera_model"], b1["intrinsics"], b1["distortion"])
    cam = V.create_camera(*cam_args)
    ds = [V.VisualLiDARData(b1["image"], b1["points"], b1["intensities"]), _tiny_bag(V, b1, 1, 1), _tiny_bag(V, b1, 64, 2)]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 20
    out = _solve_modes(V, cam, ds, b1["T_init"], params)
    _assert_same_solve(out[1], out[3])
    ref = _oracle_solve(oracle, cam_args, ds, b1["T_init"], 20)
    assert np.isfinite(ref["trace"][:, 6]).all()
    assert np.array_equal(out[3][1]["x"], ref["x"]) and np.abs(out[3][0] - ref["T"]).max() == 0.0
    _assert_trace_is_oracles(out[3][3], ref["trace"])


def test_persistent_solve_with_an_empty_bag(gpu, oracle):
    """A 0-point bag scores NaN at every pose, and so does the objective (the sum over bags, as in the reference): this
    runs the launch with an empty bag's block share and the Nelder-Mead machine on an all-NaN objective, against the host
    loop and the oracle."""
    V = gpu
    b1 = _synthetic_bag(20_000, cfg=4)
    cam_args = (b1["camera_model"], b1["intrinsics"], b1["distortion"])
    cam = V.create_camera(*cam_args)
    ds = [V.VisualLiDARData(b1["image"], b1["points"], b1["intensities"]), V.VisualLiDARData(b1["image"][::-1].copy(), np.zeros((0, 4)), np.zeros(0))]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 15
    out = _solve_modes(V, cam, ds, b1["T_init"], params)
    _assert_same_solve(out[1], out[3])
    ref = _oracle_solve(oracle, cam_args, ds, b1["T_init"], 15)
    assert np.isnan(ref["trace"][:, 6]).all()
    _assert_trace_is_oracles(out[3][3], ref["trace"])


# ---- 4. bins -----------------------------------------------------------------------------------------------------------


def test_every_bin_count_in_pose_list_mode(gpu, oracle):
    pr = util.random_problem("fisheye", n=20_000, seed=600)
    Ts = util.random_poses(pr["T"], 9, seed=5)
    for bins in range(1, 33):
        nid, hist, _ = _scored(_cost(gpu, pr, bins), Ts)
        _assert_matches_oracle(oracle, pr, Ts, nid, hist, bins)


@pytest.mark.parametrize("bins", [1, 2, 3, 31, 32])
def test_solve_mode_bin_counts_against_the_host_loop(gpu, bins):
    V = gpu
    bags = [_synthetic_bag(15_000, cfg=5), _synthetic_bag(9_000, cfg=6)]
    cam = V.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    ds = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in bags]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations, params.nid_bins = 20, bins
    out = _solve_modes(V, cam, ds, bags[0]["T_init"], params)
    _assert_same_solve(out[1], out[3])
    # one bin: every inlier falls in the one joint bin, and the NID is -0 at every pose (as in the oracle), so that case
    # runs the machine on a constant objective -- every iteration shrinks; from two bins on the objective varies
    y = out[3][3][:, 6]
    assert np.isfinite(y).all() and (np.all(y == 0.0) == (bins == 1))


# ---- 5. deferred-pair queue saturated ----------------------------------------------------------------------------------


def _edge_points_pinhole(n, rng):
    """Camera-frame points (identity pose) whose projection under DYADIC_PINHOLE is EXACTLY on a column edge u = k and in
    the middle of a row: x, y, z dyadic, hence float32 and exact in u = 512 x / z + 320."""
    z = rng.choice([0.5, 1.0, 2.0, 4.0], n)
    k = rng.integers(1, 640, n)
    j = rng.integers(0, 480, n)
    return np.stack([(k - 320.0) / 512.0 * z, (j + 0.5 - 240.0) / 512.0 * z, z], axis=1)


def _edge_cloud(n_full_tiles, n_mixed_tiles, rng, model="plumb_bob"):
    """Tiles of 64 consecutive points: fully on pixel edges, or 3 edge points among 61 random ones."""
    if model == "plumb_bob":
        edge = lambda m: _edge_points_pinhole(m, rng)
    else:  # equirectangular: x = 0 is lon = 0 (u = W / 2) for z > 0 and the seam (u = W or 0) for z < 0
        def edge(m):
            d = _S.lidar_directions("sphere", m, rng) * rng.uniform(0.5, 20.0, (m, 1))
            d[:, 0] = 0.0
            return d
    # random points in front of the camera (the pose is the identity: camera frame = cloud frame)
    rand = lambda m: (_S.lidar_directions("frustum", m, rng) @ _S.R_CAMERA_LIDAR.T) * rng.uniform(0.5, 20.0, (m, 1))
    tiles = [edge(64) for _ in range(n_full_tiles)]
    for _ in range(n_mixed_tiles):
        t = rand(64)
        t[rng.choice(64, 3, replace=False)] = edge(3)
        tiles.append(t)
    order = rng.permutation(len(tiles))
    pts = np.concatenate([tiles[i] for i in order]).astype(np.float32).astype(np.float64)
    return pts


def _pr_from_points(model, pts, seed, intr=None, dist=None, size=None):
    pr = util.random_problem(model, n=pts.shape[0], seed=seed, size=size)
    pr["points"] = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1)
    if intr is not None:
        pr["intrinsics"], pr["distortion"] = intr, dist
    pr["T"] = np.eye(4)
    return pr


def _translations(T0, ts):
    out = []
    for t in ts:
        T = T0.copy()
        T[:3, 3] += t
        out.append(T)
    return np.stack(out)


@pytest.mark.parametrize("offset_px", [1e-7, -1e-8, 1e-9, 0.0])
def test_deferred_queue_saturated_pinhole(gpu, oracle, offset_px):
    """Every point within |offset| px of a column edge at every pose: 8 poses that differ by translations along the
    edge (y), all shifted across it by the same sub-ulp x translation (doubles of the pose, not of the float32 cloud)."""
    rng = np.random.default_rng(700)
    pts = _edge_cloud(1500, 0, rng)
    intr, dist = DYADIC_PINHOLE
    pr = _pr_from_points("plumb_bob", pts, seed=701, intr=intr, dist=dist)
    tx = offset_px / 512.0  # at z = 1; z in {0.5 .. 4} scales the offset by 2 .. 1/4
    Ts = _translations(np.eye(4), [(tx, 1e-5 * k, 0.0) for k in range(8)])
    ocam = oracle.create_camera("plumb_bob", intr, dist)
    for T in Ts:  # the oracle's own projection puts every point where the case says
        uv = oracle.project(ocam, pts + T[:3, 3])
        d = np.abs(uv[:, 0] - np.round(uv[:, 0]))
        assert d.max() <= abs(offset_px) * 2.5 + 1e-12 and (offset_px == 0.0 or d.min() >= abs(offset_px) / 4.5)
    cost = _cost(gpu, pr)
    assert cost.filter_enabled
    nid, hist, prof = _scored(cost, Ts)
    n_pp = pts.shape[0] * len(Ts)
    assert prof["deferred_plain"] / n_pp > 0.9, prof
    _assert_matches_oracle(oracle, pr, Ts, nid, hist)
    assert hist.sum() > 0.9 * n_pp


@pytest.mark.parametrize("model", ["plumb_bob", "equirectangular"])
def test_deferred_queue_mixed_full_and_partial_tiles(gpu, oracle, model):
    """Fully deferred tiles (512 pairs per tile and pass: the per-lane ballot path) between tiles with 24 deferred pairs
    (the prefix path, the warp's queue crossing its 32-pair drain point)."""
    rng = np.random.default_rng(710)
    pts = _edge_cloud(400, 1200, rng, model)
    if model == "plumb_bob":
        intr, dist = DYADIC_PINHOLE
        pr = _pr_from_points(model, pts, seed=711, intr=intr, dist=dist)
        Ts = _translations(np.eye(4), [(0.0, 1e-5 * k, 0.0) for k in range(8)])
        deferred_key = "deferred_plain"
    else:
        pr = _pr_from_points(model, pts, seed=711)
        Ts = _translations(np.eye(4), [(0.0, 2e-3 * k, 0.0) for k in range(8)])  # along the meridian: inside the delta gate
        deferred_key = "deferred_delta"
    cost = _cost(gpu, pr)
    nid, hist, prof = _scored(cost, Ts)
    n_edge = 400 * 64 + 1200 * 3
    assert prof[deferred_key] >= 0.9 * n_edge * len(Ts), prof
    if model == "equirectangular":
        assert prof["delta_passes"] == 1, prof
    _assert_matches_oracle(oracle, pr, Ts, nid, hist)


def test_deferred_queue_saturated_equirectangular(gpu, oracle):
    """Points on the meridian x = 0 (u = W / 2 exactly) and behind it on the seam, nudged by +-1e-9 .. 1e-7 px of pose
    translation: nearly every point-pose goes to the exact path, in plain and in delta passes."""
    rng = np.random.default_rng(720)
    pts = _edge_cloud(1500, 0, rng, "equirectangular")
    pr = _pr_from_points("equirectangular", pts, seed=721)
    ocam = oracle.create_camera("equirectangular", pr["intrinsics"], pr["distortion"])
    total_pp, deferred = 0, 0
    for off in (1e-7, -1e-9):
        # a translation tx moves lon by ~tx / r_xz, i.e. u by W tx / (2 pi r_xz) px
        tx = off * 2.0 * math.pi / pr["W"]
        for same in (True, False):  # 8 identical poses (plain classifier at P = 1 per pass) or 8 along the edge (delta)
            Ts = _translations(np.eye(4), [(tx, 0.0 if same else 1e-3 * k, 0.0) for k in range(8)])
            cost = _cost(gpu, pr)
            if same:
                cost.set_poses_per_pass(1)
            nid, hist, prof = _scored(cost, Ts, chunk=1 if same else 8)
            assert prof["delta_passes"] == (0 if same else 1), prof
            _assert_matches_oracle(oracle, pr, Ts, nid, hist)
            uv = oracle.project(ocam, pts + Ts[0][:3, 3])
            d = np.abs(uv[:, 0] - np.round(uv[:, 0]))
            assert np.quantile(d, 0.99) < 1e-5 and d.max() < 1e-2  # up to ~1e-2 px only close to the poles (r_xz small)
            total_pp += pts.shape[0] * 8
            deferred += prof["deferred_plain"] + prof["deferred_delta"]
    assert deferred / total_pp > 0.9, deferred / total_pp


# ---- 6. the equirectangular delta step inside K1p -------------------------------------------------------------------------

DR_GATE, DT_GATE = np.float32(4e-3), np.float32(2e-2)


def _host_gate(T, T0):
    """lean_delta_pose's test: every entry of float32(T - T0) within the spread (rotation 4e-3, translation 2 cm)."""
    d = (T[:3, :] - T0[:3, :]).astype(np.float32)
    return bool(np.all(np.abs(d[:, :3]) <= DR_GATE) and np.all(np.abs(d[:, 3]) <= DT_GATE))


def _rot_z(T0, theta):
    c, s = math.cos(theta), math.sin(theta)
    R = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    T = T0.copy()
    T[:3, :3] = R @ T0[:3, :3]
    return T


def _rotation_at_gate(T0):
    """(theta inside, theta one float32 ulp of max |dR| above): bisection on the host's own float32 test."""
    f = lambda th: np.abs((_rot_z(T0, th)[:3, :3] - T0[:3, :3]).astype(np.float32)).max()
    lo, hi = 0.0, 0.01
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if f(mid) <= DR_GATE:
            lo = mid
        else:
            hi = mid
    assert f(lo) == DR_GATE and f(hi) == np.nextafter(DR_GATE, np.float32(1.0))
    return lo, hi


def _delta_problem(n, seed, T0, shifts):
    """Random equirectangular cloud plus points that sit exactly on u = W / 2 or the seam at pose k (x = -(t0 + shift_k))
    and near the poles (small z) at those poses."""
    rng = np.random.default_rng(seed)
    pr = util.random_problem("equirectangular", n=n, seed=seed)
    pts = pr["points"][:, :3].copy()
    m = 4000
    for k, s in enumerate(shifts):
        sel = slice(1000 + k * m, 1000 + (k + 1) * m)
        d = _S.lidar_directions("sphere", m, rng) * rng.uniform(0.5, 20.0, (m, 1))
        d[: m // 4, 2] = d[: m // 4, 2] * 1e-4 - T0[2, 3]  # camera z ~ 0: near the poles at pose k
        d[:, 0] = -(T0[0, 3] + s)
        pts[sel] = d
    pr["points"][:, :3] = pts.astype(np.float32).astype(np.float64)
    assert np.array_equal(pr["points"][1000 : 1000 + len(shifts) * m, 0], np.repeat(-(T0[0, 3] + np.asarray(shifts)), m))
    pr["T"] = T0
    return pr


def test_delta_gate_edges_through_the_persistent_kernel(gpu, oracle):
    T0 = np.eye(4)
    T0[:3, 3] = (0.125, -0.0625, 0.25)  # dyadic: t0 + float32 shifts are exact in double
    shifts = [0.0, 2.0**-9, -(2.0**-8), 3 * 2.0**-9, -(2.0**-7), 2.0**-7, -(3 * 2.0**-9), 2.0**-6]  # <= 1.6 cm: x only
    pr = _delta_problem(60_000, 800, T0, shifts)
    cost = _cost(gpu, pr)
    along = _translations(T0, [(s, 0.0, 0.0) for s in shifts])  # points on u = W/2 or the seam at every pose k >= 1
    th_in, th_out = _rotation_at_gate(T0)
    dt = float(DT_GATE)
    dt_above = float(np.nextafter(DT_GATE, np.float32(1.0)))
    cases = {  # name: (poses, delta pass expected)
        "along_edges": (along, True),
        "rotation_at_gate": (np.stack([T0, _rot_z(T0, th_in)] + list(along[2:])), True),
        "rotation_one_ulp_above": (np.stack([T0, _rot_z(T0, th_out)] + list(along[2:])), False),
        "translation_at_gate": (np.stack([T0, _translations(T0, [(0.0, 0.0, dt)])[0]] + list(along[2:])), True),
        "translation_above": (np.stack([T0, _translations(T0, [(0.0, 0.0, dt_above)])[0]] + list(along[2:])), False),
        "two_poses": (along[:2], True),
        "identical": (np.stack([T0] * 8), True),
        "one_pose": (along[:1], False),
    }
    for name, (Ts, inside) in cases.items():
        assert all(_host_gate(T, Ts[0]) for T in Ts[1:]) == inside or len(Ts) == 1, name
        nid, hist, prof = _scored(cost, Ts)
        assert prof["delta_passes"] == (1 if inside else 0), (name, prof)
        _assert_matches_oracle(oracle, pr, Ts, nid, hist)
    # chunks alternating in and out of the gate: the delta instance checks every chunk again
    far = util.random_poses(T0, 8, seed=9, rot_deg=5.0, trans=0.3)
    Ts = np.concatenate([along, far, along, far[::-1], along[:5]])
    nid, hist, prof = _scored(cost, Ts)
    assert prof["delta_passes"] == 3 and prof["delta_poses"] == 21, prof
    _assert_matches_oracle(oracle, pr, Ts, nid, hist)


def test_equirectangular_solve_takes_the_delta_step_and_follows_the_oracle(gpu, oracle):
    V = gpu
    pr = util.random_problem("equirectangular", n=12_000, seed=810)
    cam_args = (pr["model"], pr["intrinsics"], pr["distortion"])
    cam = V.create_camera(*cam_args)
    ds = [V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])]
    T0 = _S.perturb(pr["T"], (0.3, -0.2, 0.3), (0.01, 0.0, -0.01))
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 40
    out = _solve_modes(V, cam, ds, T0, params)
    _assert_same_solve(out[1], out[3])
    ref = _oracle_solve(oracle, cam_args, ds, T0, 40)
    assert np.array_equal(out[3][1]["x"], ref["x"]) and np.abs(out[3][0] - ref["T"]).max() == 0.0
    _assert_trace_is_oracles(out[3][3], ref["trace"])
    # the same solve on a cost object built from the cloud culled as the solve culls it (view culling at T0 with the
    # depth buffer), so that its profile shows the delta passes of the solve the oracle checks
    ocam = oracle.create_camera(*cam_args)
    idx = oracle.view_cull(ocam, pr["W"], pr["H"], oracle.estimate_camera_fov(ocam, pr["W"], pr["H"]), True, pr["points"], T0)
    cost = _cost(V, dict(pr, points=pr["points"][idx], intensities=pr["intensities"][idx]))
    try:
        _VC.record_solve_trace(True)
        for mode in (1, 3):
            V.set_solver_mode(mode)
            cost.reset_profile()
            T, r = _VC.estimate_pose_on_costs([cost], T0, params)
            assert np.array_equal(r["x"], ref["x"]) and r["num_evaluations"] == ref["num_evaluations"] and np.abs(T - ref["T"]).max() == 0.0
            _assert_trace_is_oracles(_VC.last_solve_trace(), ref["trace"])
    finally:
        V.set_solver_mode(0)
        _VC.record_solve_trace(False)
    prof = cost.profile()  # of the mode-3 solve
    assert prof["kernel_launches"] == 1 and prof["delta_passes"] > 0, prof


# ---- 7. special values inside full tiles --------------------------------------------------------------------------------


def _special_points(W, H):
    f = float(np.float32(1e30))
    nan, inf = float("nan"), float("inf")
    s = 2.0**-20
    rows = [
        [nan, 0.0, 1.0], [0.0, nan, 1.0], [0.0, 0.0, nan], [inf, 0.0, 1.0], [-inf, 0.0, 1.0], [0.0, 0.0, inf], [0.0, 0.0, -inf],
        [f, 0.0, 1.0], [0.0, f, 1.0], [0.0, 0.0, f], [f, f, f], [1.0, 0.0, f],
        [0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1e-3], [0.01, 0.01, 0.01], [-0.01, 0.0, -0.01],  # camera centre, z = 0
    ]
    for z in (1.0, 2.0):  # the (-1, 0) truncation strip and the last row / column (DYADIC_PINHOLE: exact)
        for u in (-1.0, -1.0 + s, -0.5, -s, 0.0, W - 1 + (1 - s), float(W)):
            rows.append([(u - 320.0) / 512.0 * z, 0.5 / 512.0 * z, z])
        for v in (-1.0, -1.0 + s, -0.5, -s, H - 1 + (1 - 1e-7), H - 1 + (1 - s), float(H)):
            rows.append([0.5 / 512.0 * z, (v - 240.0) / 512.0 * z, z])
    return np.array(rows)


@pytest.mark.parametrize("model", util.MODELS)
def test_special_values_inside_full_tiles(gpu, oracle, model):
    rng = np.random.default_rng(900)
    pr = util.random_problem(model, n=100_000, seed=901)
    if model == "plumb_bob":
        pr["intrinsics"], pr["distortion"] = DYADIC_PINHOLE
    sp = _special_points(pr["W"], pr["H"]).astype(np.float32).astype(np.float64)
    pts = pr["points"][:, :3].copy()
    at = 50_000 - 50_000 % 64 + 5  # the middle of full tiles (and, with 4 copies spread out, of several warps' shares)
    for c in range(4):
        pts[at + c * 7_001 : at + c * 7_001 + sp.shape[0]] = sp
    pr["points"][:, :3] = pts
    Ts = np.concatenate([np.eye(4)[None], _translations(np.eye(4), [(0.0, 0.0, 1e-3)]), util.random_poses(pr["T"], 6, seed=7)])
    cost = _cost(gpu, pr)
    assert cost.points_are_f32
    nid, hist, _ = _scored(cost, Ts)
    _assert_matches_oracle(oracle, pr, Ts, nid, hist)


# ---- the persistent solve's evaluation trace ---------------------------------------------------------------------------


@pytest.mark.parametrize("iters", [10, 60])
def test_full_evaluation_trace_of_a_shrinking_solve_host_and_persistent(gpu, oracle, iters):
    """Constant image and intensities: the NID is the same at every pose, so every iteration ends in a shrink and
    evaluates n + 3 = 9 poses -- 7 + 9 I evaluations, every one of which the trace must carry in the host loop (mode 1)
    and in the persistent solve (mode 3)."""
    V = gpu
    pr = util.random_problem("plumb_bob", n=2000, seed=1)
    pr["image"] = np.full_like(pr["image"], 128)
    pr["intensities"] = np.full_like(pr["intensities"], 0.5)
    cam_args = (pr["model"], pr["intrinsics"], pr["distortion"])
    cam = V.create_camera(*cam_args)
    ds = [V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"])]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = iters
    params.nelder_mead_convergence_criteria = 0.0
    out = _solve_modes(V, cam, ds, pr["T"], params, modes=(1, 3))
    ref = _oracle_solve(oracle, cam_args, ds, pr["T"], iters, criterion=0.0)
    assert ref["num_evaluations"] == 7 + 9 * iters == len(ref["trace"])
    for mode in (1, 3):
        _, r, _, tr = out[mode]
        assert r["num_evaluations"] == ref["num_evaluations"], mode
        _assert_trace_is_oracles(tr, ref["trace"])
    _assert_same_solve(out[1], out[3])


def test_full_evaluation_trace_of_an_ordinary_solve_host_and_persistent(gpu, oracle):
    V = gpu
    bag = _synthetic_bag(20_000, cfg=3)
    cam_args = (bag["camera_model"], bag["intrinsics"], bag["distortion"])
    cam = V.create_camera(*cam_args)
    ds = [V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])]
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations = 60
    out = _solve_modes(V, cam, ds, bag["T_init"], params, modes=(1, 3))
    ref = _oracle_solve(oracle, cam_args, ds, bag["T_init"], 60)
    for mode in (1, 3):
        _assert_trace_is_oracles(out[mode][3], ref["trace"])
    _assert_same_solve(out[1], out[3])
