"""GPU suite of K1s, the pose sweep kernel (nid_pose_sweep_kernel, csrc/nid_sweep.cuh), at its structural edges against
the CPU oracle: the slot of a pose in its group of 4, the per-warp deferral queue (64 entries, drained 32 at a time),
special coordinates and intensities, every bin count up to 32, up to 8 bags, the size threshold of the persistent kernel
hand-over and device-generated search sets.  Every histogram must be the oracle's bit for bit and every NID within
1e-12 (NaN where the oracle has NaN); vlcal_nid_debug_sweep_last_deferred shows that the sweep itself reached the exact
path.  The decision edges of the fp32 filter (cone, guards, pixel edges, large translations) go through K1s in
tests/test_gpu_filter_decision_edges.py."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import util
from direct_visual_lidar_calibration_b200 import _lib
from direct_visual_lidar_calibration_b200 import initial_guess as ig
from direct_visual_lidar_calibration_b200.cost import score_poses
from test_gpu_round1_edges import DYADIC_PINHOLE, _edge_intensities, _grey_ramp, _pr_from_points, _special_points, _translations

pytestmark = pytest.mark.gpu
NID_TOL = 1e-12


def _cost(V, pr, bins=16, max_fov=None):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    return V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), V.NIDCostParams(bins), max_fov=max_fov)


def _oracle(O, pr, Ts, bins=16, max_fov=None):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    fov = O.estimate_camera_fov(cam, pr["W"], pr["H"]) if max_fov is None else max_fov
    out = [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], bins, fov, T, omp=len(pr["points"]) > 4096) for T in Ts]
    return np.array([o[0] for o in out]), np.stack([o[1] for o in out])


def _assert_nid(a, b):
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    m = ~np.isnan(b)
    assert np.all(np.abs(a[m] - b[m]) < NID_TOL), np.abs(a[m] - b[m]).max()


def _sweep(costs, Ts):
    """K1s whatever the cloud size: (NID, bag 0's histograms, deferred (point, pose) pairs)."""
    nid, hist = ig.sweep_poses(costs, Ts, return_hist=True, kernel_only=True)
    return nid, hist, int(_lib.load_library().vlcal_nid_debug_sweep_last_deferred())


def _check(V, O, pr, Ts, bins=16, max_fov=None, rows=None):
    """K1s against the oracle (at `rows` of Ts, default all) and against calculate_batch bit for bit. -> deferred pairs."""
    cost = _cost(V, pr, bins, max_fov)
    nid, hist, deferred = _sweep([cost], Ts)
    rows = np.arange(len(Ts)) if rows is None else rows
    ref_nid, ref_hist = _oracle(O, pr, Ts[rows], bins, max_fov)
    assert np.array_equal(hist[rows], ref_hist), int(np.abs(hist[rows].astype(np.int64) - ref_hist).sum())
    _assert_nid(nid[rows], ref_nid)
    assert np.array_equal(nid, cost.calculate_batch(Ts), equal_nan=True)
    cost.close()
    return deferred


# ---- dyadic pinhole edge clouds: u = 512 (x + t_x) / z + 320 is exact --------------------------------------------------------

OFF_EDGE = 0.5 / 512.0  # a translation that moves every z = 1 point half a pixel off its column edge


def _pinhole(points, seed):
    intr, dist = DYADIC_PINHOLE
    pr = _pr_from_points("plumb_bob", points, seed=seed, intr=intr, dist=dist)
    pr["image"] = _grey_ramp(pr["W"], pr["H"])
    return pr


def _on_edge(m, rng):
    """m points at z = 1 exactly on a column edge at t = 0 (and half a pixel off it at t_x = OFF_EDGE)."""
    u = rng.integers(40, 600, m).astype(np.float64)
    v = rng.integers(40, 440, m) + 0.5
    return np.stack([(u - 320.0) / 512.0, (v - 240.0) / 512.0, np.ones(m)], axis=1)


def _off_edge(m, rng):
    p = _on_edge(m, rng)
    p[:, 0] += 0.25 / 512.0  # a quarter pixel from the edge at t = 0, three quarters at OFF_EDGE
    return p


def _group_poses(targets, P):
    """P poses: those in `targets` put the edge points on their edges, the others half a pixel off."""
    return _translations(np.eye(4), [(0.0 if j in targets else OFF_EDGE, 0.0, 0.0) for j in range(P)])


def test_targeted_pose_in_every_slot_of_a_group(gpu, oracle):
    """The edge points are on their edges at one slot s of every group of 4 only: P = 1 ... 9, and with one and three
    poses beyond the launch's resident blocks x 4 (a block's second group, partial)."""
    rng = np.random.default_rng(1)
    n_edge = 700
    pts = np.concatenate([_on_edge(n_edge, rng), _off_edge(1300, rng)])[rng.permutation(2000)]
    pr = _pinhole(pts, seed=2)
    blocks, per_block = _lib.C.c_int(), _lib.C.c_int()
    cost = _cost(gpu, pr)
    _lib.check(_lib.load_library().vlcal_nid_sweep_launch_shape(cost.handle, _lib.C.byref(blocks), _lib.C.byref(per_block)))
    assert per_block.value == 4
    big = blocks.value * 4
    for P in list(range(1, 10)) + [big + 1, big + 3]:
        for s in range(min(P, 4)):
            targets = {j for j in range(P) if j % 4 == s}
            Ts = _group_poses(targets, P)
            rows = None if P <= 9 else np.r_[0:8, P - 8 : P]
            deferred = _check(gpu, oracle, pr, Ts, rows=rows)
            # every edge point defers at every targeted pose, next to nothing else does
            assert n_edge * len(targets) <= deferred <= n_edge * len(targets) + 0.01 * len(pts) * P, (P, s, deferred)


@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("n_mod", [0, 1, 31, 255])
def test_deferral_queue_rows_and_tails(gpu, oracle, k, n_mod):
    """Rows of 32 points in which 0, 1, 31 or 32 lanes defer, at k of the group's 4 poses: the warp queue crosses 32
    after every pose index and reaches 63, and the tail drain takes every fill 1 ... 31 over the cases.  n % 256 (and
    n % 32) of 1, 31 and 255 leave stale lanes in the last row, which still run the classifier."""
    rng = np.random.default_rng(10 * k + n_mod)
    pattern = rng.choice([0, 1, 31, 32], 64)
    rows = [np.concatenate([_on_edge(c, rng), _off_edge(32 - c, rng)]) for c in pattern]
    pts = np.concatenate(rows)
    n = len(pts) - 256 + n_mod if n_mod else len(pts)
    pts = pts[:n]
    n_edge = int(sum(min(c, max(0, n - 32 * r)) for r, c in enumerate(pattern)))
    pr = _pinhole(pts, seed=11)
    Ts = _group_poses(set(range(k)), 4)
    deferred = _check(gpu, oracle, pr, np.concatenate([Ts, Ts[::-1]]))
    assert 2 * k * n_edge <= deferred <= 2 * k * n_edge + 0.01 * 8 * n, (deferred, n_edge)


@pytest.mark.parametrize("model", util.MODELS)
def test_special_values(gpu, oracle, model):
    """NaN, +-inf and 1e30 coordinates, the camera centre and the truncation strips at lane 0 and lane 31 of a row, at
    the cloud's last point and in the row prefetched while the first is classified; NaN, negative and above-1
    intensities."""
    rng = np.random.default_rng(20)
    pr = util.random_problem(model, n=3000, seed=21)
    if model == "plumb_bob":
        pr["intrinsics"], pr["distortion"] = DYADIC_PINHOLE
    sp = _special_points(pr["W"], pr["H"]).astype(np.float32).astype(np.float64)
    m = len(sp)
    pts = pr["points"][:, :3].copy()
    slots = [np.arange(0, 32 * m, 32), np.arange(31, 32 * m + 31, 32)[: m] + 32 * m, np.arange(256, 256 + m), np.arange(3000 - m, 3000)]
    for at in slots:
        assert at.max() < 3000
        pts[at] = sp[rng.permutation(m)]
    pr["points"][:, :3] = pts
    pr["intensities"] = _edge_intensities(16, 3000, rng, f32=True)
    Ts = np.concatenate([np.eye(4)[None], util.random_poses(pr["T"], 6, seed=22)])
    _check(gpu, oracle, pr, Ts)


def test_every_bin_count(gpu, oracle):
    """bins = 1 ... 32 (one bin: the oracle's NID is -0); the histogram layout is image_bin + lidar_bin * bins."""
    rng = np.random.default_rng(30)
    pr = util.random_problem("omnidir", n=3000, seed=31)
    Ts = util.random_poses(pr["T"], 5, seed=32)
    for bins in range(1, 33):
        pr["intensities"] = _edge_intensities(bins, 3000, rng, f32=True)
        cost = _cost(gpu, pr, bins)
        nid, hist, _ = _sweep([cost], Ts)
        ref_nid, ref_hist = _oracle(oracle, pr, Ts, bins)
        assert np.array_equal(hist, ref_hist), bins
        _assert_nid(nid, ref_nid)
        if bins == 1:
            assert np.all(ref_nid == 0.0) and np.all(np.signbit(ref_nid)) and np.array_equal(np.signbit(nid), np.signbit(ref_nid))
        # raw layout of hist_out: index image_bin + lidar_bin * bins (sweep_poses returns [P, image_bin, lidar_bin])
        raw = np.empty((len(Ts), bins * bins), dtype=np.int32)
        handles = (_lib.C.c_void_p * 1)(cost.handle)
        out = np.empty(len(Ts))
        from direct_visual_lidar_calibration_b200.camera import _dp
        from direct_visual_lidar_calibration_b200.cost import T_to_colmajor

        _lib.check(_lib.load_library().vlcal_nid_debug_sweep_kernel(handles, 1, _dp(T_to_colmajor(Ts)), len(Ts), _dp(out), raw.ctypes.data))
        assert np.array_equal(raw.reshape(len(Ts), bins, bins), np.swapaxes(ref_hist, 1, 2)), bins
        cost.close()


def test_eight_bags_and_a_ninth(gpu, oracle):
    """8 bags of unequal sizes, then the same with an empty bag 0: scores summed in bag order (bit-equal to score_poses),
    hist_out from bag 0 only, inliers the sums of every bag's histograms; a ninth bag is refused."""
    sizes = [900, 70, 33, 4000, 31, 257, 2500, 64, 0]
    prs = []
    for b, n in enumerate(sizes):
        pr = util.random_problem("plumb_bob", n=max(n, 16), seed=40 + b)
        pr["points"], pr["intensities"] = pr["points"][:n], pr["intensities"][:n]
        if b:
            pr["image"] = np.ascontiguousarray(np.roll(prs[0]["image"], 7 * b, axis=1))
        prs.append(pr)
    Ts = util.random_poses(prs[0]["T"], 9, seed=41, rot_deg=5.0, trans=0.2)
    for order in (list(range(8)), [8] + list(range(1, 8))):
        costs = [_cost(gpu, prs[i]) for i in order]
        nid, hist, _ = _sweep(costs, Ts)
        assert np.array_equal(nid, score_poses(costs, Ts), equal_nan=True)
        ref = [_oracle(oracle, prs[i], Ts) for i in order]
        assert np.array_equal(hist, ref[0][1])  # bag 0 only, also when it is empty
        total = ref[0][0]
        for r_nid, _ in ref[1:]:
            total = total + r_nid
        _assert_nid(nid, total)
        assert np.isnan(nid).all() == (order[0] == 8)
        sset = ig.SearchSet(Ts[:, :3, :3], np.eye(3)[None], np.zeros((1, 3)), np.zeros((1, 3)))  # pose i: R_i, t = 0
        s_nid, inliers, _ = ig.sweep_search_set(costs, sset)
        s_ref = [_oracle(oracle, prs[i], sset.poses()) for i in order]
        assert np.array_equal(inliers, sum(h.reshape(len(h), -1).sum(axis=1) for _, h in s_ref))
        assert np.array_equal(s_nid, score_poses(costs, sset.poses()), equal_nan=True)
        for c in costs:
            c.close()
    costs = [_cost(gpu, prs[0]) for _ in range(9)]
    with pytest.raises(gpu.VlcalError, match="at most 8") as e:
        _sweep(costs, Ts)
    assert e.value.code == _lib.ERR_UNSUPPORTED


@pytest.mark.parametrize("n_bags", [1, 2, 8])
def test_size_threshold(gpu, oracle, n_bags):
    """Clouds of exactly vlcal_nid_sweep_max_points() points in total and one more: the first runs the sweep kernel, the
    second the persistent kernel (kernel time 0), with the same scores; the search-set fallback's inliers are the sums
    of calculate_batch's histograms."""
    L = _lib.load_library()
    limit = int(L.vlcal_nid_sweep_max_points())
    base = util.random_problem("plumb_bob", n=limit + 1, seed=50)
    Ts = util.random_poses(base["T"], 6, seed=51, rot_deg=10.0, trans=0.3)
    sset = ig.local_set(Ts[:1], 2.0, 0.1, 0)
    for total in (limit, limit + 1):
        cuts = np.linspace(0, total, n_bags + 1).astype(int)
        cuts[1] += 1 if n_bags > 1 else 0  # unequal bags
        prs = [dict(base, points=base["points"][a:b], intensities=base["intensities"][a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
        costs = [_cost(gpu, pr) for pr in prs]
        nid = ig.sweep_poses(costs, Ts)
        ms = float(L.vlcal_nid_sweep_last_kernel_ms())
        assert (ms > 0.0) == (total == limit), (total, ms)
        assert np.array_equal(nid, score_poses(costs, Ts), equal_nan=True)
        assert np.array_equal(nid, ig.sweep_poses(costs, Ts, kernel_only=True), equal_nan=True)
        scores, inliers, _ = ig.sweep_search_set(costs, sset)
        assert np.array_equal(scores, score_poses(costs, sset.poses()), equal_nan=True)
        hists = [c.calculate_batch(sset.poses(), return_hist=True)[1] for c in costs]
        assert np.array_equal(inliers, sum(h.reshape(len(h), -1).sum(axis=1) for h in hists))
        if n_bags == 1:
            ref_nid, _ = _oracle(oracle, prs[0], Ts[:2])
            _assert_nid(nid[:2], ref_nid)
        for c in costs:
            c.close()


def test_search_sets_against_the_oracle(gpu, oracle):
    """Tables of one entry on each axis, indices that repeat, are unsorted and include the first and last flat index,
    and the refusals of search_set_check; scores at the device-generated poses against oracle.nid_calculate at
    SearchSet.poses()."""
    pr = util.random_problem("fisheye", n=2500, seed=60)
    cost = _cost(gpu, pr)
    R0, t0 = pr["T"][:3, :3], pr["T"][:3, 3]
    one = ig.SearchSet(np.eye(3)[None], R0[None], (R0.T @ t0)[None], np.zeros((1, 3)))
    assert one.n_poses == 1 and np.allclose(one.poses()[0], pr["T"])
    loc = ig.local_set(util.random_poses(pr["T"], 2, seed=61, rot_deg=3.0, trans=0.05), 1.0, 0.05, 1)
    full = loc.n_poses
    idx = np.array([full - 1, 0, 17, 17, full // 2, 0, 3, full - 1, 250, 9])
    picked = ig.SearchSet(loc.left, loc.base, loc.center, loc.offset, indices=idx)
    for s in (one, picked):
        P = s.poses()
        assert np.array_equal(P.view(np.uint64), s.device_poses().view(np.uint64))
        scores, inliers, _ = ig.sweep_search_set([cost], s)
        ref_nid, ref_hist = _oracle(oracle, pr, P)
        _assert_nid(scores, ref_nid)
        assert np.array_equal(inliers, ref_hist.reshape(len(P), -1).sum(axis=1))
    scores = ig.sweep_search_set([cost], picked)[0]
    assert np.array_equal(scores[[0, 1, 2]], scores[[7, 5, 3]], equal_nan=True)  # repeated indices, repeated scores
    # refusals: NULL tables, non-positive counts, a count that disagrees with the tables, an index out of range
    L = _lib.load_library()
    out = np.empty(full + 1)
    handles = (_lib.C.c_void_p * 1)(cost.handle)
    from direct_visual_lidar_calibration_b200.camera import _dp

    bad = []
    s = loc.as_struct()
    s.n_poses = full + 1
    bad.append(s)
    s = loc.as_struct()
    s.n_left = 0
    bad.append(s)
    s = loc.as_struct()
    s.left = None
    bad.append(s)
    wrong = np.array([0, full], dtype=np.int32)
    s = picked.as_struct()
    s.indices, s.n_poses = wrong.ctypes.data_as(_lib.C.POINTER(_lib.C.c_int32)), 2
    bad.append(s)
    neg = np.array([-1], dtype=np.int32)
    s = picked.as_struct()
    s.indices, s.n_poses = neg.ctypes.data_as(_lib.C.POINTER(_lib.C.c_int32)), 1
    bad.append(s)
    for s in bad:
        assert L.vlcal_nid_sweep_search_set(handles, 1, _lib.C.byref(s), _dp(out)) == _lib.ERR_INVALID_ARGUMENT
    cost.close()


@pytest.mark.parametrize("model", util.MODELS)
def test_cone_at_rotations_over_so3(gpu, oracle, model):
    """FoV-cone points at random rotations and at members of rotation_set(9.0); beyond 90 degrees for fisheye, omnidir
    and equirectangular."""
    from test_gpu_filter_decision_edges import CONE_FOVS, _cone_points, _problem

    rng = np.random.default_rng(70 + len(model))
    fov = CONE_FOVS[model][-1]
    rs = ig.rotation_set(9.0)
    Rs = np.concatenate([Rotation.random(4, random_state=71).as_matrix(), rs.poses(rng.choice(rs.n_poses, 4, replace=False))[:, :3, :3]])
    Ts = np.tile(np.eye(4), (len(Rs), 1, 1))
    Ts[:, :3, :3] = Rs
    Ts[:, :3, 3] = rng.uniform(-0.3, 0.3, (len(Rs), 3))
    groups = [_cone_points(rng, 150, fov, eps, T)[0] for T in Ts for eps in (0.0, 1e-9, -1e-9, 1e-7, -1e-7)]
    pr, _ = _problem(model, np.concatenate(groups), n_plain=3000, seed=72)
    deferred = _check(gpu, oracle, pr, Ts, max_fov=fov)
    assert deferred > 0.5 * sum(len(g) for g in groups)
