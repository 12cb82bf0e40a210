"""Mode B on the GPU at its edges: K2 (nid_bspline_kernel, value) and K3 (nid_bspline_grad_kernel, value + gradient)
against the exact-sum reference of tests/mode_b_reference.py (itself checked against the oracle by
tests/test_mode_b_reference_host.py), under certified bounds instead of flat tolerances:

  every bin       |hist_gpu - fsum| <= taps * (2^-(F+1) + (8/9) proj_tol) + (|hist_gpu| + |fsum|) 2^-53
  inlier counts   exact, per lidar bin
  NID             within R.nid_bound (the bin bound propagated through the entropies), and within the rounding of the
                  double entropy tail (>= 1e-12 never needed unless |Hip| is tiny) of the same formula evaluated on the
                  kernel's own histogram -- that isolates the finalize, including its h_image row sums.

F is the kernels' fixed-point fraction bits, min(40, 62 - ceil(log2 n)); proj_tol the per-model projection tolerance
(0 where the projection is the oracle's bits)."""
import math

import numpy as np
import pytest

import mode_b_reference as R
import util
from direct_visual_lidar_calibration_b200 import synthetic as _S

util.S = _S
pytestmark = pytest.mark.gpu
U = R.U
ERR_UNSUPPORTED = -6


def _cost(V, pr, bins=16, points=None, intensities=None):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    pts = pr["points"] if points is None else points
    ins = pr["intensities"] if intensities is None else intensities
    return V.NIDCost(cam, V.VisualLiDARData(pr["image"], pts, ins), bins)


def _exact(O, pr, tp, bins=16, points=None, intensities=None):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    pts = pr["points"] if points is None else points
    ins = pr["intensities"] if intensities is None else intensities
    return R.Exact(O, cam, pr["image"], pts, ins, bins, tp)


def _check_value(ex, n, model, W, H, ok, nid, hist=None):
    """One pose of K2 (with its histogram) or of K3 (value only) against the exact reference."""
    F = R.fixed_bits(n)
    tol = R.PROJ_TOL[model]
    # a verdict the two projections could disagree on would make the comparison meaningless; none is that close
    assert ex.decision_margin(W, H) > 2 * tol
    ref_ok = bool(np.isfinite(ex.nid))
    assert bool(ok) == ref_ok
    if hist is not None:
        assert np.array_equal(np.rint(hist.sum(axis=0)), ex.points)  # exact inlier count per lidar bin
        bound = R.hist_bound(ex, hist, F, tol)
        assert np.all(np.abs(hist - ex.hist) <= bound), (np.abs(hist - ex.hist) - bound).max()
    if not ref_ok:
        assert not np.isfinite(nid)
        return
    assert abs(nid - float(ex.nid)) <= R.nid_bound(ex, F, tol), (nid, float(ex.nid), R.nid_bound(ex, F, tol))
    if hist is not None:
        Hi, Hp, Hip, self_nid = R.nid_from_gpu_hist(hist)
        assert abs(nid - float(self_nid)) <= max(1e-12, R.nid_rounding_bound(Hi, Hp, Hip, self_nid, ex.bins)), (nid, float(self_nid))


def _tps(pr, P, seed=3):
    return np.stack([R.sophus_params(T) for T in util.random_poses(pr["T"], P, seed=seed)])


# ---------------------------------------------------------------------------------------------------------------------
# shapes: all models, both layouts, N in {0, 1, 255, 257, 100003}, P in {1, 8, 9, 17}
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("f32", [True, False])
@pytest.mark.parametrize("model", util.MODELS)
def test_k2_shapes(gpu, oracle, model, f32):
    pr = util.random_problem(model, n=100003, seed=101, f32=f32)
    W, H = pr["W"], pr["H"]
    tps = _tps(pr, 17)
    cost = _cost(gpu, pr)
    ok, nid, hist = cost.evaluate(tps, return_hist=True)  # launches of 8 + 8 + 1 poses
    for p in (0, 7, 8, 16):  # both sides of each launch boundary
        ex = _exact(oracle, pr, tps[p])
        assert ex.n_inliers > 10000
        _check_value(ex, 100003, model, W, H, ok[p], nid[p], hist[p])
    for P in (1, 8, 9):  # a shorter list computes the same bits as the head of the longer one
        okP, nidP, histP = cost.evaluate(tps[:P], return_hist=True)
        assert np.array_equal(okP, ok[:P]) and np.array_equal(nidP, nid[:P]) and np.array_equal(histP, hist[:P])
    # K3 on the same cloud: value under the same bound, gradient against the oracle's Jet evaluation
    okg, nidg, grad = cost.evaluate_with_gradient(tps[:2])
    ocam = oracle.create_camera(model, pr["intrinsics"], pr["distortion"])
    for p in range(2):
        _check_value(_exact(oracle, pr, tps[p]), 100003, model, W, H, okg[p], nidg[p])
        _check_grad_vs_oracle(oracle, ocam, pr, tps[p], grad[p], 16)
    for n in (0, 1, 255, 257):  # empty, one point, one block minus one, one block plus two (ragged grid-stride)
        pts, ins = pr["points"][:n], pr["intensities"][:n]
        c = _cost(gpu, pr, points=pts, intensities=ins)
        ok_n, nid_n, hist_n = c.evaluate(tps, return_hist=True)
        for p in range(17):
            ex = _exact(oracle, pr, tps[p], points=pts, intensities=ins)
            _check_value(ex, n, model, W, H, ok_n[p], nid_n[p], hist_n[p])
        for P in (1, 8, 9):
            o, v, h = c.evaluate(tps[:P], return_hist=True)
            assert np.array_equal(o, ok_n[:P]) and np.array_equal(v, nid_n[:P], equal_nan=True) and np.array_equal(h, hist_n[:P])


def _check_grad_vs_oracle(oracle, ocam, pr, tp, grad, bins, points=None, intensities=None):
    """K3's gradient against the oracle's Jet functor.  Both compute the same sums of ~16 n terms in different orders
    (double atomics vs serial); with n = 1e5 that reorders at most 16e5 * 2^-53 ~ 2e-10 of the sum of |terms|, which for
    these clouds stays within 1e-8 of max(1, |grad|) (the terms cancel by at most ~50x)."""
    pts = pr["points"] if points is None else points
    ins = pr["intensities"] if intensities is None else intensities
    rok, _, rgrad = oracle.nid_cost_bspline_grad(ocam, pr["image"], pts, ins, bins, tp)
    if rok:
        assert np.abs(grad - rgrad).max() <= 1e-8 * max(1.0, np.abs(rgrad).max()), (grad, rgrad)


# ---------------------------------------------------------------------------------------------------------------------
# bin counts: every launch chunk size (8, 4, 2, 1 poses), the divisors of 255, the shared-memory limits
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("bins", [1, 2, 5, 15, 17, 33, 51, 64, 85, 112])
def test_k2_bin_counts(gpu, oracle, bins):
    pr = util.random_problem("plumb_bob", n=30000, seed=102)
    tps = _tps(pr, 9, seed=6)  # 9 poses: 8+1, 4+4+1, 2+2+2+2+1 or 9x1 launches depending on bins
    cost = _cost(gpu, pr, bins)
    ok, nid, hist = cost.evaluate(tps, return_hist=True)
    for p in range(9):
        ex = _exact(oracle, pr, tps[p], bins)
        _check_value(ex, 30000, "plumb_bob", pr["W"], pr["H"], ok[p], nid[p], hist[p])
        o1, n1, h1 = cost.evaluate(tps[p : p + 1], return_hist=True)  # batch == single, bit for bit
        assert o1[0] == ok[p] and n1[0] == nid[p] and np.array_equal(h1[0], hist[p])
    ok2, nid2, hist2 = cost.evaluate(tps, return_hist=True)  # run == rerun (integer accumulation)
    assert np.array_equal(ok, ok2) and np.array_equal(nid, nid2) and np.array_equal(hist, hist2)
    if bins > 1:
        assert hist.sum() > 9 * 10000


@pytest.mark.parametrize("bins", [1, 5, 17, 51, 56])
def test_k3_bin_counts(gpu, oracle, bins):
    pr = util.random_problem("plumb_bob", n=20000, seed=103)
    tps = _tps(pr, 2, seed=7)
    ok, nid, grad = _cost(gpu, pr, bins).evaluate_with_gradient(tps)
    ocam = oracle.create_camera("plumb_bob", pr["intrinsics"], pr["distortion"])
    for p in range(2):
        _check_value(_exact(oracle, pr, tps[p], bins), 20000, "plumb_bob", pr["W"], pr["H"], ok[p], nid[p])
        if bins > 1:  # one bin: NID is identically 0 and its gradient pure rounding, amplified by 1 / Hip ~ 1e6
            _check_grad_vs_oracle(oracle, ocam, pr, tps[p], grad[p], bins)


def test_bins_beyond_the_shared_memory_limits_are_refused(gpu):
    pr = util.random_problem("plumb_bob", n=1000, seed=104)
    tp = _tps(pr, 1)
    with pytest.raises(gpu.VlcalError) as e:
        _cost(gpu, pr, 113).evaluate(tp)
    assert e.value.code == ERR_UNSUPPORTED
    with pytest.raises(gpu.VlcalError) as e:
        _cost(gpu, pr, 57).evaluate_with_gradient(tp)
    assert e.value.code == ERR_UNSUPPORTED
    ok, nid = _cost(gpu, pr, 57).evaluate(tp)  # K2 still serves 57 bins
    assert ok[0] and np.isfinite(nid[0])


# ---------------------------------------------------------------------------------------------------------------------
# points on the decision edges, clamped footprints, tiny images; invalid inputs
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("size", [None, (1, 1), (2, 3), (5, 2), (3, 5)])
@pytest.mark.parametrize("model", util.MODELS)
def test_edge_points(gpu, oracle, model, size):
    for f32 in (False, True):
        pr = R.edge_problem(oracle, model, size=size, seed=11, f32=f32)
        n = pr["points"].shape[0]
        cost = _cost(gpu, pr)
        tps = np.stack([pr["tp"], pr["tp"]])
        ok, nid, hist = cost.evaluate(tps, return_hist=True)
        ex = _exact(oracle, pr, pr["tp"])
        assert ex.n_inliers > (100 if size is None else 20)
        _check_value(ex, n, model, pr["W"], pr["H"], ok[0], nid[0], hist[0])
        assert nid[1] == nid[0] and np.array_equal(hist[1], hist[0])
        okg, nidg, _ = cost.evaluate_with_gradient(pr["tp"][None])
        _check_value(ex, n, model, pr["W"], pr["H"], okg[0], nidg[0])


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("model", util.MODELS)
def test_invalid_inputs(gpu, oracle, model, f32):
    pr = R.invalid_problem(model, seed=13)
    if f32:  # the same specials on the float4 layout (NaN, Inf, -0.5, 1.0, 1.7 are float32 values)
        pr["points"] = pr["points"].astype(np.float32).astype(np.float64)
        ins = pr["intensities"]
        pr["intensities"] = np.where(np.isfinite(ins) & (ins >= 0) & (ins < 1), np.floor(ins * 256) / 256, ins)
    cost = _cost(gpu, pr)
    ok, nid, hist = cost.evaluate(pr["tps"], return_hist=True)
    okg, nidg, _ = cost.evaluate_with_gradient(pr["tps"])
    n = pr["points"].shape[0]
    for p, tp in enumerate(pr["tps"]):
        ex = _exact(oracle, pr, tp)
        assert ex.n_inliers > 100
        _check_value(ex, n, model, pr["W"], pr["H"], ok[p], nid[p], hist[p])
        _check_value(ex, n, model, pr["W"], pr["H"], okg[p], nidg[p])


# ---------------------------------------------------------------------------------------------------------------------
# gradient against central differences of K2 (no oracle)
# ---------------------------------------------------------------------------------------------------------------------


def _value_error_bound(hist, bins, F):
    """Certified |NID_gpu - NID_exact| from the kernel's own histogram alone: S inliers carry 16 S taps, each rounded by
    <= 2^-(F+1), so sum_b |dp_b| <= 16 * 2^-(F+1) + 2 (nb + bins) u and each entropy moves by <= L times that (L =
    |ln 1e-6| + 1, as in R.nid_bound); the double tail adds R.nid_rounding_bound."""
    Hi, Hp, Hip, nid = R.nid_from_gpu_hist(hist)
    Hi, Hp, Hip = abs(float(Hi)), abs(float(Hp)), abs(float(Hip))
    L = abs(math.log(R.EPS_LOG)) + 1.0
    dH = L * (16 * 2.0 ** -(F + 1) + 2 * (bins * bins + bins) * U)
    h = Hip - dH
    return dH / h + (Hi + Hp) * dH / (Hip * h) + R.nid_rounding_bound(Hi, Hp, Hip, nid, bins)


@pytest.mark.parametrize("model", ["plumb_bob", "fisheye", "equirectangular"])
def test_gradient_vs_central_differences(gpu, oracle, model):
    """K3's d NID / d (qx qy qz qw tx ty tz) against (K2(x + h e_k) - K2(x - h e_k)) / 2h.

    The configuration is smooth: the quaternion is scaled off the unit sphere by 1.01 (the functor is a polynomial in
    q, and both kernels evaluate it as such), and only points >= 3 px inside the image at that pose are kept.  Over
    +-2h no point moves by more than 0.2 px, so none crosses the border and the cost is a C2 function of the pose (the
    cubic B-spline weights are C2 across knots).  Error of the central difference D(h) against K3's derivative:
      noise        each K2 value is within e of the exact functor (_value_error_bound), so D(h) is within e / h;
      truncation   f'''(xi) h^2 / 6; estimated from the two step sizes, |D(2h) - D(h)| = (3/6) h^2 |f'''| + O(noise),
                   so |D(h) - f'| <= |D(2h) - D(h)| / 3 + e / h (+ e / 2h for the noise inside D(2h)), taken x4;
      K3 itself    sums the partials in double atomics: within 1e-9 of max |grad| (the reordering bound of
                   _check_grad_vs_oracle, x10 for the 2x larger cloud).
    h = 2e-6 for q (du/dq <= 2 f |p| / z ~ 2e4 px: <= 0.04 px) and 2e-5 m for t (<= 0.01 px)."""
    pr = util.random_problem(model, n=60000, seed=105, f32=(model != "fisheye"))
    tp = R.sophus_params(pr["T"])
    tp[:4] *= 1.01
    ex = _exact(oracle, pr, tp)
    keep = ex.inlier.copy()
    keep[keep] = (ex.u[keep] >= 3) & (ex.u[keep] <= pr["W"] - 3) & (ex.v[keep] >= 3) & (ex.v[keep] <= pr["H"] - 3)
    pts, ins = pr["points"][keep], pr["intensities"][keep]
    n = int(keep.sum())
    assert n > 20000
    cost = _cost(gpu, pr, points=pts, intensities=ins)
    hs = np.array([2e-6] * 4 + [2e-5] * 3)
    poses = [tp]
    for k in range(7):
        for m in (1, -1, 2, -2):
            x = tp.copy()
            x[k] += m * hs[k]
            poses.append(x)
    ok, nid, hist = cost.evaluate(np.stack(poses), return_hist=True)
    assert ok.all()
    assert np.all(np.rint(hist.sum(axis=(1, 2))) == n)  # every point stays an inlier over +-2h
    okg, nidg, grad = cost.evaluate_with_gradient(tp[None])
    assert okg[0]
    F = R.fixed_bits(n)
    e = max(_value_error_bound(hist[i], 16, F) for i in range(len(poses)))
    gscale = np.abs(grad[0]).max()
    for k in range(7):
        f1p, f1m, f2p, f2m = nid[1 + 4 * k : 5 + 4 * k]
        h = hs[k]
        D1, D2 = (f1p - f1m) / (2 * h), (f2p - f2m) / (4 * h)
        tol = 4 * (abs(D2 - D1) / 3 + e / h + e / (2 * h)) + 1e-9 * gscale
        assert abs(grad[0][k] - D1) <= tol, (k, grad[0][k], D1, tol)
    assert gscale > 1e-3  # a real gradient, not a vacuous comparison
    assert all(abs(grad[0][k]) > 0 for k in range(7))


# ---------------------------------------------------------------------------------------------------------------------
# fixed-point headroom: more than 2^24 points' weight in one bin (closed forms, no oracle)
# ---------------------------------------------------------------------------------------------------------------------

N_BIG = 2**24 + 2**20  # F = 37
# plumb_bob without distortion at the identity pose: u = fx x / z + cx, so points are placed by pixel directly
BIG_CAM = ("plumb_bob", [400.0, 410.0, 320.0, 240.0], [0.0, 0.0, 0.0, 0.0, 0.0])
BIG_W, BIG_H = 640, 480
IDENTITY = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
# each point's 16 double weights sum to 1 within 60 u < 2^-46 (four betas of <= 6 rounded operations each, times the 16
# products), an error the fixed-point bound does not contain: charged per point on top of 16 * 2^-(F+1)
SUM_ONE = 2.0**-46


def _big_cloud(u, v, rng):
    """float32-representable points with (u, v) at the identity pose, depth 2 .. 10 m (the float rounding moves them
    by < 1e-4 px)."""
    _, (fx, fy, cx, cy), _ = BIG_CAM
    z = rng.uniform(2.0, 10.0, u.size)
    pts = np.empty((u.size, 4))
    pts[:, 0] = ((u - cx) / fx) * z
    pts[:, 1] = ((v - cy) / fy) * z
    pts[:, 2] = z
    pts[:, :3] = pts[:, :3].astype(np.float32)
    pts[:, 3] = 1.0
    return pts


def _headroom_case(gpu, image, pts, ins, counts):
    """K2 and K3 on a cloud whose points each put all 16 taps into one joint bin: bin b must hold counts[b] (exactly
    known), the NID must be the closed form of those counts, and the gradient 0 (no bin changes under a small move)."""
    model, intr, dist = BIG_CAM
    cam = gpu.create_camera(model, intr, dist)
    cost = gpu.NIDCost(cam, gpu.VisualLiDARData(image, pts, ins), 16)
    F = R.fixed_bits(pts.shape[0])
    assert F == R.fixed_bits(N_BIG)
    ok, nid, hist = cost.evaluate(IDENTITY[None], return_hist=True)
    okg, nidg, grad = cost.evaluate_with_gradient(IDENTITY[None])
    del cost
    hist = hist[0]
    # per bin: 16 taps per point rounded by <= 2^-(F+1) each, the per-point sum-to-one error, the conversion to double
    bound = counts * (16 * 2.0 ** -(F + 1) + SUM_ONE) + np.abs(hist) * U
    assert np.all(np.abs(hist - counts) <= bound), (hist[counts > 0], counts[counts > 0])
    assert np.array_equal(np.rint(hist.sum(axis=0)), counts.sum(axis=0))  # lidar marginal = inlier counts
    assert np.array_equal(np.rint(hist.sum(axis=1)), counts.sum(axis=1))  # image marginal
    ex = _Closed(counts)
    b = R.nid_bound(ex, F, 0.0, extra_per_tap=SUM_ONE / 16)
    assert ok[0] and okg[0]
    assert abs(nid[0] - float(ex.nid)) <= b, (nid[0], float(ex.nid), b)
    assert abs(nidg[0] - float(ex.nid)) <= b, (nidg[0], float(ex.nid), b)
    return nid[0], nidg[0], grad[0], b


class _Closed:
    """The exact histograms of a cloud whose points each fall into one joint bin: counts[image_bin, lidar_bin]."""

    def __init__(self, counts):
        self.bins = counts.shape[0]
        self.hist = counts.astype(np.float64)
        self.hist_image = self.hist.sum(axis=1)
        self.taps = 16 * counts
        self.taps_image = self.taps.sum(axis=1)
        self.points = counts.sum(axis=0)
        self.Hi, self.Hp, self.Hip, self.nid = R.entropies(self.hist, self.hist_image, self.points)


# The gradient is 0 exactly: every point keeps all 16 taps in its bin under a small move, and the tap derivatives of
# one point sum to zero.  What remains is rounding: per point |sum of 16 computed derivative taps| <= 16 u (|U| + |V|)
# with |U|, |V| <= 2 f |p| / z * (1 + |x / z|) < 1e4 px per unit pose parameter here, i.e. < 2e-11 per point; even
# without any cancellation between points that is 2e-11 in p, and d NID ~ dp / Hip with |Hip| >= 1e-6 in these clouds:
# 2e-5.
# The double atomics' reordering of those near-cancelling sums stays of the same order; 1e-4 leaves that x5.
GRAD_ZERO = 1e-4


def test_fixed_point_headroom_one_bin(gpu):
    """2^24 + 2^20 points, constant image, constant intensity: all weight in one joint bin.  With 2^-40 fixed point that
    bin wraps modulo 2^64 (N 2^40 > 2^64) and NID comes out ~1; the exact NID is 0."""
    rng = np.random.default_rng(201)
    u = rng.uniform(10.0, BIG_W - 10.0, N_BIG)
    v = rng.uniform(10.0, BIG_H - 10.0, N_BIG)
    pts = _big_cloud(u, v, rng)
    del u, v
    image = np.full((BIG_H, BIG_W), 128, dtype=np.uint8)
    ins = np.full(N_BIG, 0.5)
    counts = np.zeros((16, 16), dtype=np.int64)
    counts[int(128 * (1.0 / 255.0) * 16), 8] = N_BIG
    nid, nidg, grad, b = _headroom_case(gpu, image, pts, ins, counts)
    # Hip = -(1 + eta) ln(1 + eta + 1e-6) ~ -1e-6 amplifies a relative bin error eta into NID ~ 1e6 eta; b certifies
    # |NID| <= 2e-3 from the worst-case rounding, the 16 N independent roundings give |eta| ~ 1e-15, i.e. |NID| ~ 1e-9
    assert b < 5e-3
    assert abs(nid) < 1e-6 and abs(nidg) < 1e-6, (nid, nidg)
    assert np.all(np.abs(grad) <= GRAD_ZERO), grad


def test_fixed_point_headroom_two_levels(gpu):
    """Same size, image 0 on the left half and 255 on the right, intensities 0.25 / 0.75, points >= 3 px from the
    dividing column: four bins with known counts and a non-degenerate NID.  97 % of the points are on the left, split
    between the two intensities: no joint bin reaches 2^24 points, but the left image-marginal row (the finalize's row
    sum) does -- with 2^-40 fixed point that sum is what wraps."""
    rng = np.random.default_rng(202)
    left = rng.random(N_BIG) < 0.97
    u = np.where(left, rng.uniform(10.0, BIG_W / 2 - 3.0, N_BIG), rng.uniform(BIG_W / 2 + 3.0, BIG_W - 10.0, N_BIG))
    v = rng.uniform(10.0, BIG_H - 10.0, N_BIG)
    pts = _big_cloud(u, v, rng)
    del u, v
    image = np.zeros((BIG_H, BIG_W), dtype=np.uint8)
    image[:, BIG_W // 2 :] = 255
    high = rng.random(N_BIG) < np.where(left, 0.5, 0.9)  # intensity and side correlated: MI > 0
    ins = np.where(high, 0.75, 0.25)
    counts = np.zeros((16, 16), dtype=np.int64)
    for side, ib in ((left, 0), (~left, 15)):
        for lvl, lb in ((high, 12), (~high, 4)):
            counts[ib, lb] = int(np.count_nonzero(side & lvl))
    assert counts.sum() == N_BIG and counts.max() < 2**24 < counts.sum(axis=1).max()
    del left, high
    nid, nidg, grad, b = _headroom_case(gpu, image, pts, ins, counts)
    assert 0.5 < nid < 1.0 and b < 1e-8
    assert np.all(np.abs(grad) <= GRAD_ZERO), grad
