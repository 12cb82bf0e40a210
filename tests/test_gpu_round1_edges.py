"""GPU edge suite of the round-1 NID kernels (csrc/nid_kernels.cuh): nid_hist_exact_kernel, nid_hist_filter_kernel at 2
and 4 points per lane, and nid_finalize.  They score every context the persistent kernel refuses -- double-layout clouds,
33 ... 128 bins, cameras without the lean classifier, an attached peer exchange -- and run solver mode 1.

Bar (the one of the persistent kernel's suite): integer histograms bit-identical to oracle.nid_calculate, NID within 1e-12
of the oracle with NaN exactly where the oracle has NaN, and bit-identical results across kernel instances and across ways
of chunking the same poses.  Every case checks cost.profile() against the launch geometry of nid_context.cu (computed
below from the same formulas, with the SM count read from the device), and that no persistent launch ran on the context."""
import math

import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import calibration as _VC
from test_gpu_persistent_edges import (DYADIC_PINHOLE, _assert_same_solve, _assert_trace_is_oracles, _edge_cloud, _oracle_solve, _pr_from_points, _solve_modes,
                                       _special_points, _synthetic_bag, _translations)

pytestmark = pytest.mark.gpu
NID_TOL = 1e-12
NID_THREADS = 256                      # threads per block of the round-1 kernels
NID_SMEM_FOR_POSES = 100 * 1024 - 4096  # nid_ctx_create: max_poses = min(8, this / (4 bins^2))
NID_HIST_TARGET = 64 * 1024            # launch_geometry: histogram copies while P bins^2 4 B fit twice
HEAVY = ("fisheye", "equirectangular", "atan")  # select_kernel: always 2 points per lane
GEOMETRY_BINS = [16, 17, 22, 23, 32, 33, 55, 56, 64, 90, 91, 110, 111, 128]


@pytest.fixture(scope="module")
def sms():
    import torch

    return int(torch.cuda.get_device_properties(0).multi_processor_count)


# ---- launch geometry of nid_context.cu / nid_kernels.cuh -------------------------------------------------------------


def max_poses(bins):
    return max(1, min(8, NID_SMEM_FOR_POSES // (4 * bins * bins)))


def launches(P, bins):
    return -(-P // max_poses(bins))


def geometry(P, bins):
    """The switches of one launch of P <= max_poses poses: histogram copies, the finalizer's split over warps, warps per
    pose and whether pass 1's counts stay in registers for pass 2."""
    nb = bins * bins
    split = nb <= 1024
    wpp = max(1, 8 // P) if split else 1
    return {"max_poses": max_poses(bins), "copies": max(1, min(2, NID_HIST_TARGET // (P * nb * 4))),
            "split": split, "wpp": wpp, "single": nb <= wpp * 32 * 8}


def k4_window(sms):
    """First and last cloud size for which select_kernel picks 4 points per lane (96 <= N / (SMs * 16) <= 1100)."""
    per = sms * 2 * (NID_THREADS // 32)
    return 96 * per, 1101 * per - 1


def test_cases_cross_every_switch_of_the_launch_geometry():
    """The bin counts and pose counts of test_pose_counts_at_every_geometry_boundary reach both sides of every switch."""
    seen = {}
    for bins in GEOMETRY_BINS:
        for P in range(1, 18):
            for c in range(launches(P, bins)):
                g = geometry(min(max_poses(bins), P - c * max_poses(bins)), bins)
                for k, v in g.items():
                    seen.setdefault(k, set()).add(v)
    assert seen["max_poses"] == {8, 7, 6, 3, 2, 1}
    assert seen["split"] == seen["single"] == {True, False}
    assert seen["copies"] == {1, 2} and seen["wpp"] == {1, 2, 4, 8}
    assert [max_poses(b) for b in (55, 56, 64, 90, 91, 110, 111, 128)] == [8, 7, 6, 3, 2, 2, 1, 1]
    # the pairs either side of the single register pass: 22 / 23 bins at two warps per pose, 16 / 17 at one, 32 / 33 at split
    assert geometry(3, 22)["single"] and not geometry(3, 23)["single"]
    assert geometry(5, 16)["single"] and not geometry(5, 17)["single"]
    assert geometry(1, 32)["split"] and not geometry(1, 33)["split"]


# ---- helpers ----------------------------------------------------------------------------------------------------------


def _cost(V, pr, bins=16, variant=0):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    cost = V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), V.NIDCostParams(bins))
    cost.set_kernel_variant(variant)
    return cost


def _scored(cost, Ts, bins):
    """calculate_batch with the histograms, asserting that it ran the round-1 kernels: ceil(P / max_poses) launches of
    one pass each, and never the persistent kernel on this context."""
    cost.reset_profile()
    nid, hist = cost.calculate_batch(Ts, return_hist=True)
    prof = cost.profile()
    assert prof["kernel_launches"] == prof["passes"] == launches(len(Ts), bins), (len(Ts), bins, prof)
    assert prof["poses_total"] == len(Ts) and cost.last_points_per_lane() == 0, prof
    return nid, hist


def _oracle_eval(O, pr, Ts, bins=16):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(cam, pr["W"], pr["H"])
    big = pr["points"].shape[0] * len(Ts) > 2_000_000
    out = [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], bins, fov, T, omp=big) for T in Ts]
    return np.array([o[0] for o in out]), np.stack([o[1] for o in out]).reshape(len(Ts), bins, bins)


def _assert_nid(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    m = ~np.isnan(a)
    assert np.all(np.abs(a[m] - b[m]) < NID_TOL), np.abs(a[m] - b[m]).max()


def _assert_oracle(nid, hist, ref):
    ref_nid, ref_hist = ref
    assert int(np.abs(hist.astype(np.int64) - ref_hist).sum()) == 0
    _assert_nid(nid, ref_nid)


def _assert_identical(a, b):
    (na, ha), (nb, hb) = a, b
    assert np.array_equal(ha, hb) and np.array_equal(na, nb, equal_nan=True)


def _grey_ramp(W, H):
    """Every grey value 0 ... 255 in every run of 256 pixels of a row, so that every edge of the image-bin LUT is hit."""
    y, x = np.mgrid[0:H, 0:W]
    return ((x + 13 * y) % 256).astype(np.uint8)


def _edge_intensities(bins, n, rng, f32):
    """Intensities on and one ulp either side of every lidar-bin edge k / bins (float32 ulps for the float4 layout),
    plus 0, -0, 1 - ulp, 1, values above 1, negative values, NaN and +-inf (lidar_bin_of's clamps and the x86 cast)."""
    dt = np.float32 if f32 else np.float64
    vals = [0.0, -0.0, 1.0, 1.5, 7.0, -0.25, -1e-30, 1e30, math.nan, math.inf, -math.inf, float(np.nextafter(dt(1), dt(0)))]
    for k in range(bins + 1):
        c = dt(k / bins)
        vals += [float(c), float(np.nextafter(c, dt(-1))), float(np.nextafter(c, dt(2)))]
    vals = np.array(vals, dtype=dt).astype(np.float64)
    out = rng.integers(0, 256, n) / 256.0
    m = min(n, 3 * len(vals))
    out[rng.permutation(n)[:m]] = np.resize(vals, m)
    return out


def _problem(model, n, seed, **kw):
    pr = util.random_problem(model, n=max(n, 16), seed=seed, **kw)
    if n == 0:
        pr["points"], pr["intensities"] = pr["points"][:0], pr["intensities"][:0]
    return pr


# ---- 1. every bin count --------------------------------------------------------------------------------------------------


def test_every_bin_count_through_the_exact_kernel_and_the_filter(gpu, oracle):
    base = util.random_problem("plumb_bob", n=3000, seed=1000)
    base["image"] = _grey_ramp(base["W"], base["H"])
    Ts = util.random_poses(base["T"], 3, seed=10)
    rng = np.random.default_rng(1001)
    for bins in range(1, 129):
        pr = dict(base, intensities=_edge_intensities(bins, 3000, rng, f32=True))
        ref = _oracle_eval(oracle, pr, Ts, bins)
        assert ref[1].sum() > 1500
        exact = _cost(gpu, pr, bins, variant=1)
        assert exact.points_are_f32
        got = _scored(exact, Ts, bins)
        _assert_oracle(*got, ref)
        filt = _cost(gpu, pr, bins, variant=4)
        assert filt.filter_enabled
        _assert_identical(_scored(filt, Ts, bins), got)
        if bins > 32:  # above the persistent kernel's bin range variants 2 / 3 pick the round-1 filter's K = 2 / K = 4
            for v in (2, 3):
                filt.set_kernel_variant(v)
                _assert_identical(_scored(filt, Ts, bins), got)
        # the same cloud with intensities one double ulp from the edges: double layout, exact kernel
        pr64 = dict(base, intensities=_edge_intensities(bins, 3000, rng, f32=False))
        c64 = _cost(gpu, pr64, bins)
        assert not c64.points_are_f32 and not c64.filter_enabled
        _assert_oracle(*_scored(c64, Ts, bins), _oracle_eval(oracle, pr64, Ts, bins))


# ---- 2. pose counts at the geometry boundaries ---------------------------------------------------------------------------


@pytest.mark.parametrize("bins", GEOMETRY_BINS)
def test_pose_counts_at_every_geometry_boundary(gpu, oracle, bins):
    pr = util.random_problem("plumb_bob", n=6000, seed=1100 + bins)
    pr["image"] = _grey_ramp(pr["W"], pr["H"])
    Ts = util.random_poses(pr["T"], 17, seed=bins)
    ref = _oracle_eval(oracle, pr, Ts, bins)
    cost = _cost(gpu, pr, bins, variant=4)
    assert cost.filter_enabled
    full = _scored(cost, Ts, bins)
    _assert_oracle(*full, ref)
    for P in range(1, 18):  # every list is a prefix of the long one
        nid, hist = _scored(cost, Ts[:P], bins)
        _assert_identical((nid, hist), (full[0][:P], full[1][:P]))
    for p in range(17):  # every pose alone
        _assert_identical(_scored(cost, Ts[p : p + 1], bins), (full[0][p : p + 1], full[1][p : p + 1]))
    # long and short calls alternating: the self-cleaning accumulators and the block ticket leave no residue
    for P in (17, 1, 8, 17, 2):
        _assert_identical(_scored(cost, Ts[:P], bins), (full[0][:P], full[1][:P]))
    exact = _cost(gpu, pr, bins, variant=1)
    for P in sorted({1, max_poses(bins), max_poses(bins) + 1, 17}):
        _assert_identical(_scored(exact, Ts[:P], bins), (full[0][:P], full[1][:P]))


# ---- 3. shapes -------------------------------------------------------------------------------------------------------------


def _shape_sizes(model, sms):
    """Cloud sizes at the kernels' bookkeeping edges: a warp +- 1, a block +- 1, the saturated grid's threads +- 1 for
    1, 2, 4 and 8 blocks per SM (the warps of the filter's grid x 32, whatever the occupancy), a cloud for which the exact
    kernel's grid-stride loop runs more than once at any occupancy, and (models that may take 4 points per lane) both
    ends of the K = 4 window +- 1."""
    sizes = {0, 1, 31, 32, 33, 255, 256, 257, 2 * sms * 8 * NID_THREADS + 1}
    for k in (1, 2, 4, 8):
        sizes |= {sms * k * NID_THREADS - 1, sms * k * NID_THREADS + 1}
    if model not in HEAVY:
        lo, hi = k4_window(sms)
        sizes |= {lo - 1, lo, lo + 1, hi - 1, hi, hi + 1}
    return sorted(sizes)


@pytest.mark.parametrize("model", util.MODELS)
def test_shapes_through_the_exact_kernel_and_the_filter(gpu, oracle, sms, model):
    for i, n in enumerate(_shape_sizes(model, sms)):
        pr = _problem(model, n, seed=1200 + i)
        Ts = util.random_poses(pr["T"], 3, seed=i)
        ref = _oracle_eval(oracle, pr, Ts)
        exact = _scored(_cost(gpu, pr, 16, variant=1), Ts, 16)
        _assert_oracle(*exact, ref)
        filt = _cost(gpu, pr, 16, variant=4)
        assert filt.filter_enabled
        _assert_identical(_scored(filt, Ts, 16), exact)
        if n > 1000:
            assert exact[1].sum() > 0.2 * n, (n, exact[1].sum())


def test_two_million_points(gpu, oracle):
    pr = util.random_problem("plumb_bob", n=2_000_000, seed=1300)
    Ts = util.random_poses(pr["T"], 3, seed=13)
    ref = _oracle_eval(oracle, pr, Ts)
    exact = _scored(_cost(gpu, pr, 16, variant=1), Ts, 16)
    _assert_oracle(*exact, ref)
    filt = _cost(gpu, pr, 16, variant=4)
    _assert_identical(_scored(filt, Ts, 16), exact)
    for bins in (64, 128):  # the filter at K = 2 and K = 4: one launch of 3 poses at 64 bins, three launches at 128
        ref = _oracle_eval(oracle, pr, Ts, bins)
        c = _cost(gpu, pr, bins, variant=2)
        got = _scored(c, Ts, bins)
        _assert_oracle(*got, ref)
        c.set_kernel_variant(3)
        _assert_identical(_scored(c, Ts, bins), got)


# ---- 4. the filter's deferred queue saturated --------------------------------------------------------------------------------


@pytest.mark.parametrize("offset_px", [1e-7, 0.0])
def test_deferred_queue_of_the_round1_filter(gpu, oracle, sms, offset_px):
    """Every point within offset_px of a column edge at all 8 poses (dyadic pinhole, as in the persistent kernel's suite):
    more than 90 % of the point-poses go through the per-warp queue to the exact path, at K = 2 and K = 4."""
    rng = np.random.default_rng(1400)
    intr, dist = DYADIC_PINHOLE
    lo, _ = k4_window(sms)
    tx = offset_px / 512.0
    Ts = _translations(np.eye(4), [(tx, 1e-5 * k, 0.0) for k in range(8)])
    for n_tiles in (1500, lo // 64 + 8):  # variant 4 at 16 bins: K = 2, then K = 4
        pr = _pr_from_points("plumb_bob", _edge_cloud(n_tiles, 0, rng), seed=1401, intr=intr, dist=dist)
        n = pr["points"].shape[0]
        assert (lo <= n) == (n_tiles > 1500)
        for bins, variants in ((16, (4,)), (64, (2, 3))):
            ref = _oracle_eval(oracle, pr, Ts, bins)
            cost = _cost(gpu, pr, bins, variant=4)
            assert cost.filter_enabled
            n_pp, uncertain, mismatches, _ = cost.debug_filter_check(Ts)  # variant 4: the round-1 classifier
            assert mismatches == 0 and n_pp == n * 8 and uncertain / n_pp > 0.9, (n_pp, uncertain)
            exact = _scored(_cost(gpu, pr, bins, variant=1), Ts, bins)
            _assert_oracle(*exact, ref)
            assert exact[1].sum() > 0.9 * n * 8
            for v in variants:
                cost.set_kernel_variant(v)
                _assert_identical(_scored(cost, Ts, bins), exact)


# ---- 5. double layout --------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("model", util.MODELS)
def test_double_layout_with_special_values_inside_full_blocks(gpu, oracle, model):
    pr = util.random_problem(model, n=40_000, seed=1500, f32=False)
    if model == "plumb_bob":
        pr["intrinsics"], pr["distortion"] = DYADIC_PINHOLE
    sp = _special_points(pr["W"], pr["H"])
    pts = pr["points"][:, :3].copy()
    at = 20_000 - 20_000 % NID_THREADS + 37  # inside full blocks of the exact kernel
    for c in range(4):
        pts[at + c * 5_003 : at + c * 5_003 + sp.shape[0]] = sp
    pr["points"][:, :3] = pts
    assert not np.array_equal(pts[:1000].astype(np.float32).astype(np.float64), pts[:1000])
    Ts = np.concatenate([np.eye(4)[None], _translations(np.eye(4), [(0.0, 0.0, 1e-3)]), util.random_poses(pr["T"], 6, seed=15)])
    for bins in (16, 128):
        cost = _cost(gpu, pr, bins)
        assert not cost.points_are_f32 and not cost.filter_enabled
        _assert_oracle(*_scored(cost, Ts, bins), _oracle_eval(oracle, pr, Ts, bins))


# ---- 6. a camera without the lean classifier ---------------------------------------------------------------------------------


def test_wide_pinhole_without_the_filter_takes_the_exact_kernel(gpu, oracle):
    """A distortion-free pinhole whose estimated FoV reaches ~87 degrees: no fp32 filter bounds (cos(FoV) < 0.05), so no
    persistent kernel either -- the default variant runs the round-1 exact kernel."""
    pr = util.random_problem("plumb_bob", n=20_000, seed=1600)
    pr["intrinsics"], pr["distortion"] = [18.0, 18.0, 320.0, 240.0], []
    Ts = util.random_poses(pr["T"], 9, seed=16)
    for bins in (16, 64):
        cost = _cost(gpu, pr, bins)
        assert cost.points_are_f32 and not cost.filter_enabled
        assert 87.0 < math.degrees(cost.max_fov) < 88.0 and math.cos(cost.max_fov) < 0.05
        got = _scored(cost, Ts, bins)
        _assert_oracle(*got, _oracle_eval(oracle, pr, Ts, bins))
        assert got[1].sum() > 1000
        for v in (2, 3, 4):
            cost.set_kernel_variant(v)
            _assert_identical(_scored(cost, Ts, bins), got)


# ---- 7. solves ------------------------------------------------------------------------------------------------------------------


def _solve_setup(V, bag, bins, iters):
    cam_args = (bag["camera_model"], bag["intrinsics"], bag["distortion"])
    params = V.VisualCameraCalibrationParams()
    params.max_inner_iterations, params.nid_bins = iters, bins
    return cam_args, V.create_camera(*cam_args), params


@pytest.mark.parametrize("bins", [33, 55])
def test_host_loop_above_32_bins(gpu, oracle, bins):
    """Mode 1 (one round-1 launch per batch) at bin counts the persistent kernel refuses, 8 poses per launch."""
    V = gpu
    bag = _synthetic_bag(20_000, cfg=3)
    cam_args, cam, params = _solve_setup(V, bag, bins, 25)
    ds = [V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])]
    out = _solve_modes(V, cam, ds, bag["T_init"], params, modes=(1,))
    ref = _oracle_solve(oracle, cam_args, ds, bag["T_init"], 25, bins=bins)
    T, r, _, tr = out[1]
    assert np.array_equal(r["x"], ref["x"]) and r["num_evaluations"] == ref["num_evaluations"] and np.abs(T - ref["T"]).max() == 0.0
    _assert_trace_is_oracles(tr, ref["trace"])


@pytest.mark.parametrize("bins", [64, 128])
def test_host_loop_with_several_launches_per_batch(gpu, oracle, bins):
    """64 bins: 6 poses per launch, so the 7-pose initial simplex takes 2 launches; 128 bins: one pose per launch."""
    V = gpu
    bag = _synthetic_bag(20_000, cfg=4)
    cam_args, cam, params = _solve_setup(V, bag, bins, 15)
    ref = _oracle_solve(oracle, cam_args, [V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])], bag["T_init"], 15, bins=bins)
    # a cost object on the cloud culled as the solve culls it, so that its profile shows the solve's launches
    ocam = oracle.create_camera(*cam_args)
    W, H = bag["image"].shape[1], bag["image"].shape[0]
    idx = oracle.view_cull(ocam, W, H, oracle.estimate_camera_fov(ocam, W, H), True, bag["points"], bag["T_init"])
    cost = V.CostCalculatorNID(cam, V.VisualLiDARData(bag["image"], bag["points"][idx], bag["intensities"][idx]), V.NIDCostParams(bins))
    try:
        _VC.record_solve_trace(True)
        V.set_solver_mode(1)
        cost.reset_profile()
        T, r = _VC.estimate_pose_on_costs([cost], bag["T_init"], params)
        tr = _VC.last_solve_trace()
    finally:
        V.set_solver_mode(0)
        _VC.record_solve_trace(False)
    assert np.array_equal(r["x"], ref["x"]) and r["num_evaluations"] == ref["num_evaluations"] and np.abs(T - ref["T"]).max() == 0.0
    _assert_trace_is_oracles(tr, ref["trace"])
    prof = cost.profile()
    assert prof["poses_total"] == r["num_evaluations_computed"], (prof, r)
    if max_poses(bins) == 1:
        assert prof["kernel_launches"] == r["num_evaluations_computed"], (prof, r)
    else:
        assert r["num_batches"] < prof["kernel_launches"] <= 2 * r["num_batches"], (prof, r)
    assert cost.last_points_per_lane() == 0


def _double_layout_bag(n, cfg, seed):
    bag = _synthetic_bag(n, cfg=cfg)
    rng = np.random.default_rng(seed)
    bag["points"] = bag["points"].copy()
    bag["points"][:, :3] += rng.uniform(-1e-7, 1e-7, (n, 3))  # no longer float32-representable
    return bag


def test_double_layout_solve_auto_and_host_loop(gpu, oracle):
    V = gpu
    bag = _double_layout_bag(15_000, 5, 1700)
    cam_args, cam, params = _solve_setup(V, bag, 16, 20)
    ds = [V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])]
    assert not V.CostCalculatorNID(cam, ds[0]).points_are_f32
    out = _solve_modes(V, cam, ds, bag["T_init"], params, modes=(0, 1))  # 0: the persistent kernel refuses, host loop
    _assert_same_solve(out[0], out[1])
    ref = _oracle_solve(oracle, cam_args, ds, bag["T_init"], 20)
    T, r, _, tr = out[1]
    assert np.array_equal(r["x"], ref["x"]) and np.abs(T - ref["T"]).max() == 0.0
    _assert_trace_is_oracles(tr, ref["trace"])


def test_mixed_layout_bags_solve_and_score_poses(gpu, oracle):
    """One float4 bag and one double-layout bag: pk_supported refuses the pair, so solves take the host loop and
    score_poses scores each context with the round-1 kernels and sums in context order."""
    V = gpu
    b1 = _synthetic_bag(15_000, cfg=3)
    b2 = _double_layout_bag(9_000, 6, 1800)
    cam_args, cam, params = _solve_setup(V, b1, 16, 20)
    ds = [V.VisualLiDARData(b["image"], b["points"], b["intensities"]) for b in (b1, b2)]
    out = _solve_modes(V, cam, ds, b1["T_init"], params, modes=(0, 1))
    _assert_same_solve(out[0], out[1])
    ref = _oracle_solve(oracle, cam_args, ds, b1["T_init"], 20)
    T, r, _, tr = out[0]
    assert np.array_equal(r["x"], ref["x"]) and np.abs(T - ref["T"]).max() == 0.0
    _assert_trace_is_oracles(tr, ref["trace"])
    with pytest.raises(V.VlcalError):  # mode 3 needs the persistent kernel, which refuses this pair
        _solve_modes(V, cam, ds, b1["T_init"], params, modes=(3,))

    costs = [V.CostCalculatorNID(cam, d) for d in ds]
    assert costs[0].points_are_f32 and not costs[1].points_are_f32
    Ts = util.random_poses(b1["T_init"], 17, seed=18, rot_deg=1.0, trans=0.05)
    prs = [{"model": cam_args[0], "intrinsics": cam_args[1], "distortion": cam_args[2], "W": b["image"].shape[1], "H": b["image"].shape[0],
            "image": b["image"], "points": b["points"], "intensities": b["intensities"]} for b in (b1, b2)]
    refs = [_oracle_eval(oracle, pr, Ts)[0] for pr in prs]
    for c in costs:
        c.reset_profile()
    got = V.score_poses(costs, Ts)
    for c in costs:
        prof = c.profile()
        assert prof["kernel_launches"] == prof["passes"] == launches(17, 16) and c.last_points_per_lane() == 0, prof
    _assert_nid(got, (0.0 + refs[0]) + refs[1])
    alone = [c.calculate_batch(Ts) for c in costs]
    assert np.array_equal(got, (0.0 + alone[0]) + alone[1], equal_nan=True)
    for a, rf in zip(alone, refs):
        _assert_nid(a, rf)
