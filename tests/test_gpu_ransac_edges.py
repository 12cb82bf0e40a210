"""GPU edge suite of the RANSAC scoring and mask launches of initial_guess_auto (csrc/pose_estimation.cu), held to the CPU
checker tests/cpp/pose_oracle.c: its rotation (pose_oracle.rotation, pinned to the reference's SVD in
test_ransac_rotation_host.py) and its squared reprojection errors e_j (pose_oracle.errors), both in the kernel's
operation order.

Bar: plumb_bob, omnidir and rational_polynomial project with + - * / sqrt only, so every e_j is bit-identical to the
kernel's: counts, degenerate flags and the winner's inlier mask (e_j < pow(thresh, 2)) must equal the checker's exactly.
fisheye, atan and equirectangular call transcendental functions whose device and host results may differ in the last
ulp: there a count may differ by the correspondences within 1e-9 px^2 of the threshold, and the mask only at those."""
import math

import numpy as np
import pytest

import pose_oracle
import util
from direct_visual_lidar_calibration_b200 import pose_estimation as PE
from direct_visual_lidar_calibration_b200 import synthetic as S

pytestmark = pytest.mark.gpu
EXACT = ["plumb_bob", "omnidir", "rational_polynomial"]
POSE_THREADS, POSE_TILE = 128, 256  # hypotheses per block, correspondences per shared-memory tile
INVALID = "ransac_error_thresh > 0"


@pytest.fixture(scope="module")
def sms():
    import torch

    return int(torch.cuda.get_device_properties(0).multi_processor_count)


def _problem(O, model, m, seed, outliers=0.3, noise=1.0):
    """Projections of random points under the ground truth, pixel noise, a share of the keypoints replaced by random pixels.
    -> (oracle camera, kp0 (M,2), points (M,3), (intrinsics, distortion))"""
    intr, dist, (W, H) = util.CAMERAS[model]
    rng = np.random.default_rng(seed)
    T = S.gt_T_camera_lidar()
    pts = S.lidar_directions("sphere" if model == "equirectangular" else "avia", m, rng) * rng.uniform(1.0, 30.0, (m, 1))
    pts = pts.astype(np.float32).astype(np.float64)
    ocam = O.create_camera(model, intr, dist)
    kp = O.project(ocam, pts @ T[:3, :3].T + T[:3, 3]).reshape(-1, 2) + (rng.normal(0.0, noise, (m, 2)) if noise else 0.0)
    out = rng.random(m) < outliers
    kp[out] = rng.uniform([0, 0], [W, H], (int(out.sum()), 2))
    return ocam, np.ascontiguousarray(kp), pts, (intr, dist)


def _cam(V, model, cd):
    return V.create_camera(model, *cd)


def _check_counts(model, counts, degenerate, ref_counts, ref_degenerate, ref_near):
    assert np.array_equal(degenerate, ref_degenerate)
    assert np.all(counts[degenerate] == 0)
    if model in EXACT:
        bad = counts != ref_counts
        assert not bad.any(), (int(bad.sum()), np.nonzero(bad)[0][:5], counts[bad][:5], ref_counts[bad][:5])
    else:
        assert np.all(np.abs(counts.astype(np.int64) - ref_counts) <= ref_near)


def _check_mask(model, mask, e, thresh_sq):
    want = e < thresh_sq
    if model in EXACT:
        assert np.array_equal(mask, want), np.nonzero(mask != want)[0][:10]
    else:
        assert np.all((mask == want) | (np.abs(e - thresh_sq) <= 1e-9))


# ---- 1. every model: counts, flags and the winner's mask ------------------------------------------------------------------


@pytest.mark.parametrize("model", util.MODELS)
def test_counts_and_the_winners_mask(gpu, oracle, model):
    ocam, kp, pts, cd = _problem(oracle, model, 2000, seed=21)
    cam = _cam(gpu, model, cd)
    pairs = PE.sample_pairs(len(kp), 8192)
    dc, dl = pose_oracle.bearings(ocam, kp, pts)
    counts, degenerate = PE.score_pairs(cam, kp, pts, pairs, 5.0)
    ref = pose_oracle.score_bearings(ocam, kp, dc, dl, pairs, 5.0)
    _check_counts(model, counts, degenerate, *ref)
    est = PE.PoseEstimation()
    _, mask = est.estimate(cam, kp, pts)
    best = est.stats["best_index"]
    assert best == int(np.argmax(counts)) and est.stats["best_inliers"] == counts[best]
    if model in EXACT:
        assert best == int(np.argmax(ref[0]))
    e = pose_oracle.errors(ocam, pose_oracle.pair_rotation(dc, dl, pairs[best]), kp, dl)
    _check_mask(model, mask, e, math.pow(5.0, 2))
    assert est.stats["degenerate"] == int(degenerate.sum())


# ---- 2. threshold edges ----------------------------------------------------------------------------------------------------


def _thresholds_on_errors(e, limit):
    """thresh with pow(thresh, 2) == e_j exactly, for inliers e_j below limit^2 (nextafter around sqrt(e_j))."""
    out = []
    for j in np.argsort(np.abs(e - 0.5 * limit * limit)):
        if not e[j] < limit * limit:
            continue
        s = math.sqrt(e[j])
        for t in (math.nextafter(s, 0.0), s, math.nextafter(s, math.inf)):
            if math.pow(t, 2) == e[j]:
                out.append((int(j), t))
                break
        if len(out) == 3:
            break
    return out


@pytest.mark.parametrize("model", EXACT)
def test_threshold_equal_to_an_error(gpu, oracle, model):
    """thresh^2 == e_j exactly and one ulp of thresh either side, through score_pairs and through estimate with one
    hypothesis (the winner, so the mask launch decides e_j == thresh^2): e_j is not an inlier at thresh, it is one ulp above."""
    ocam, kp, pts, cd = _problem(oracle, model, 3000, seed=22, outliers=0.0)
    cam = _cam(gpu, model, cd)
    pair = PE.sample_pairs(len(kp), 1)
    dc, dl = pose_oracle.bearings(ocam, kp, pts)
    R = pose_oracle.pair_rotation(dc, dl, pair[0])
    assert R is not None
    e = pose_oracle.errors(ocam, R, kp, dl)
    found = _thresholds_on_errors(e, 5.0)
    assert found, "no error with an exact square root neighbour"
    for j, t in found:
        lo, hi = math.nextafter(t, 0.0), math.nextafter(t, math.inf)
        got = {}
        for thr in (lo, t, hi):
            sq = math.pow(thr, 2)
            counts, degenerate = PE.score_pairs(cam, kp, pts, pair, thr)
            assert not degenerate[0] and counts[0] == int((e < sq).sum())
            got[thr] = int(counts[0])
            est = PE.PoseEstimation(PE.PoseEstimationParams(ransac_iterations=1, ransac_error_thresh=thr))
            _, mask = est.estimate(cam, kp, pts)
            assert est.stats["best_index"] == 0 and est.stats["best_inliers"] == got[thr]
            assert np.array_equal(mask, e < sq), np.nonzero(mask != (e < sq))[0][:10]
            assert mask[j] == (thr == hi)
        ties = int((e == math.pow(t, 2)).sum())
        assert ties >= 1
        assert got[hi] - got[t] == ties + int(((e > math.pow(t, 2)) & (e < math.pow(hi, 2))).sum())
        assert got[t] - got[lo] == int(((e >= math.pow(lo, 2)) & (e < math.pow(t, 2))).sum())


def test_thresholds_score_pairs_does_not_validate(gpu, oracle):
    """0 -> no inliers, +inf -> every finite error, NaN -> none, -t like t (pow(-t, 2) == pow(t, 2), as in the reference)."""
    model = "plumb_bob"
    ocam, kp, pts, cd = _problem(oracle, model, 700, seed=23)
    cam = _cam(gpu, model, cd)
    pairs = PE.sample_pairs(len(kp), 64)
    pairs[5] = [3, 3]
    dc, dl = pose_oracle.bearings(ocam, kp, pts)
    finite = np.array([0 if R is None else int(np.isfinite(pose_oracle.errors(ocam, R, kp, dl)).sum()) for R in (pose_oracle.pair_rotation(dc, dl, p) for p in pairs)])
    assert finite.max() == len(kp)
    for thr, want in ((0.0, np.zeros(64)), (-0.0, np.zeros(64)), (math.inf, finite), (-math.inf, finite), (math.nan, np.zeros(64))):
        counts, degenerate = PE.score_pairs(cam, kp, pts, pairs, thr)
        assert np.array_equal(counts, want), thr
        assert degenerate[5] and degenerate.sum() == (finite == 0).sum()
    for t in (0.75, 3.0, 5.0, 17.25):
        pos, _ = PE.score_pairs(cam, kp, pts, pairs, t)
        neg, _ = PE.score_pairs(cam, kp, pts, pairs, -t)
        assert np.array_equal(pos, neg)
        assert np.array_equal(pos, pose_oracle.score_bearings(ocam, kp, dc, dl, pairs, t)[0])


def test_estimate_validates_the_threshold(gpu, oracle):
    model = "plumb_bob"
    ocam, kp, pts, cd = _problem(oracle, model, 400, seed=24)
    cam = _cam(gpu, model, cd)
    for thr in (0.0, -0.0, -5.0, -math.inf, math.nan):
        with pytest.raises(gpu.VlcalError, match=INVALID):
            PE.PoseEstimation(PE.PoseEstimationParams(ransac_error_thresh=thr)).estimate(cam, kp, pts)
    est = PE.PoseEstimation(PE.PoseEstimationParams(ransac_iterations=256, ransac_error_thresh=math.inf))
    _, mask = est.estimate(cam, kp, pts)
    dc, dl = pose_oracle.bearings(ocam, kp, pts)
    rotations = [pose_oracle.pair_rotation(dc, dl, p) for p in PE.sample_pairs(len(kp), 256)]
    first = next(i for i, R in enumerate(rotations) if R is not None)
    finite = np.isfinite(pose_oracle.errors(ocam, rotations[first], kp, dl))
    assert est.stats["best_index"] == first and est.stats["best_inliers"] == finite.sum() > 0.9 * len(kp)
    assert np.array_equal(mask, finite)


# ---- 3. launch geometry ----------------------------------------------------------------------------------------------------


def _split(h, m, sms):
    """score_hypotheses: blockIdx.y splits the tiles when there are few hypothesis blocks (about 4 blocks per SM)."""
    hyp_blocks = -(-h // POSE_THREADS)
    tiles = -(-m // POSE_TILE)
    return max(1, min(tiles, -(-4 * sms // hyp_blocks))), tiles


def test_launch_geometry(gpu, oracle, sms):
    """H at the hypothesis-block edges and past 4 * SMs * 128 (split = 1); M at the tile edges, and M with split == tiles
    and a ragged last tile, and with 1 < split < tiles (several tiles per y block, the last ragged)."""
    model = "plumb_bob"
    ragged = (4 * sms * 2 // 3) * POSE_TILE + 77  # tiles <= 4 SMs: split == tiles for H <= 128
    ocam, kp_all, pts_all, cd = _problem(oracle, model, ragged, seed=25)
    cam = _cam(gpu, model, cd)
    big_h = 4 * sms * POSE_THREADS + 5
    cases = [(h, m) for h in (1, 127, 128, 129, big_h) for m in (2, 255, 256, 257, 511, 513)]
    cases += [(1, ragged), (128, ragged), (129, ragged), (3 * POSE_THREADS, ragged)]
    rng = np.random.default_rng(26)
    seen = set()
    bearings = {}
    for h, m in cases:
        split, tiles = _split(h, m, sms)
        seen.add("one" if split == 1 else "all" if split == tiles else "some")
        kp, pts = kp_all[:m], pts_all[:m]
        if m not in bearings:
            bearings[m] = pose_oracle.bearings(ocam, kp, pts)
        pairs = rng.integers(0, m, (h, 2)).astype(np.int32)
        pairs[0] = [0, 1]
        counts, degenerate = PE.score_pairs(cam, kp, pts, pairs, 5.0)
        ref = pose_oracle.score_bearings(ocam, kp, *bearings[m], pairs, 5.0)
        _check_counts(model, counts, degenerate, *ref)
        if m > 256 and h > 100:
            assert ref[0].max() > 0
    assert seen == {"one", "all", "some"}
    split, tiles = _split(1, ragged, sms)
    assert split == tiles > 1 and ragged % POSE_TILE
    split, tiles = _split(3 * POSE_THREADS, ragged, sms)
    assert 1 < split < tiles
    assert _split(big_h, 513, sms)[0] == 1


# ---- 4. the degenerate rule ------------------------------------------------------------------------------------------------


def _near_one_e_minus_18(anti):
    """LiDAR points (0, 0, 1) and (d, 0, +-1) whose bearings' |l1 -+ l2|^2 = d * d lies just below and just at or above
    1e-18 (d found by nextafter from 1e-9)."""
    d = 1e-9
    while d * d >= 1e-18:
        d = math.nextafter(d, 0.0)
    below = d
    while d * d < 1e-18:
        d = math.nextafter(d, 1.0)
    return [np.array([[0.0, 0.0, 1.0], [dd, 0.0, -1.0 if anti else 1.0]]) for dd in (below, d)]


def _sq3(v):
    return (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]


@pytest.mark.parametrize("model", ["plumb_bob", "equirectangular"])
def test_degenerate_rule(gpu, oracle, model):
    """The same index twice, two identical keypoints (equal camera bearings, b = 0), equirectangular keypoints half a turn
    apart (antiparallel camera bearings, as far as estimate_direction resolves them), and LiDAR pairs with |l1 - l2|^2 and
    |l1 + l2|^2 just below and at 1e-18: the flags equal the checker's, a degenerate hypothesis counts 0."""
    ocam, kp, pts, cd = _problem(oracle, model, 600, seed=27)
    intr, dist, (W, H) = util.CAMERAS[model]
    cam = _cam(gpu, model, cd)
    kp, pts = kp.copy(), pts.copy()
    kp[21] = kp[20]
    rows = {}
    at = 30
    for anti in (False, True):
        for which, pair in zip(("below", "above"), _near_one_e_minus_18(anti)):
            pts[at], pts[at + 1] = pair
            rows[(anti, which)] = at
            at += 2
    pairs = [[5, 5], [599, 599], [20, 21], [21, 20]] + [[i, i + 1] for i in rows.values()] + [[i + 1, i] for i in rows.values()]
    if model == "equirectangular":
        kp[40] = [100.25, 90.5]
        kp[41] = [100.25 + W / 2, H - 90.5]
        pairs += [[40, 41], [41, 40]]
    pairs += PE.sample_pairs(600, 64).tolist()
    pairs = np.array(pairs, dtype=np.int32)
    dc, dl = pose_oracle.bearings(ocam, kp, pts)
    counts, degenerate = PE.score_pairs(cam, kp, pts, pairs, 5.0)
    ref = pose_oracle.score_bearings(ocam, kp, dc, dl, pairs, 5.0)
    _check_counts(model, counts, degenerate, *ref)
    assert degenerate[:4].all()
    for (anti, which), i in rows.items():
        v = dl[i] + dl[i + 1] if anti else dl[i] - dl[i + 1]
        assert (_sq3(v) < 1e-18) == (which == "below") and abs(_sq3(v) / 1e-18 - 1.0) < 1e-6
        k = 4 + list(rows).index((anti, which))
        assert degenerate[k] == degenerate[k + len(rows)] == (which == "below")
    if model == "equirectangular":
        assert np.abs(dc[40] + dc[41]).max() < 1e-2  # antiparallel to the resolution of estimate_direction


# ---- 5. ties between winners -----------------------------------------------------------------------------------------------


@pytest.mark.parametrize("model", EXACT)
def test_winner_ties(gpu, oracle, model):
    """Noise-free correspondences: many hypotheses reach the maximum count.  The winner is the lowest index among them, its
    mask the checker's; (i, j) and (j, i) give the same R bit for bit, hence the same count."""
    ocam, kp, pts, cd = _problem(oracle, model, 600, seed=28, outliers=0.0, noise=0.0)
    cam = _cam(gpu, model, cd)
    pairs = PE.sample_pairs(len(kp), 8192)
    counts, degenerate = PE.score_pairs(cam, kp, pts, pairs, 5.0)
    top = np.nonzero(counts == counts.max())[0]
    assert len(top) >= 2
    est = PE.PoseEstimation()
    _, mask = est.estimate(cam, kp, pts)
    assert est.stats["best_index"] == int(top[0]) and est.stats["best_inliers"] == counts.max()
    dc, dl = pose_oracle.bearings(ocam, kp, pts)
    e = pose_oracle.errors(ocam, pose_oracle.pair_rotation(dc, dl, pairs[top[0]]), kp, dl)
    _check_mask(model, mask, e, 25.0)
    rev, rev_degenerate = PE.score_pairs(cam, kp, pts, pairs[:, ::-1], 5.0)
    assert np.array_equal(rev, counts) and np.array_equal(rev_degenerate, degenerate)
    for i, j in pairs[:200]:
        a, b = pose_oracle.pair_rotation(dc, dl, (i, j)), pose_oracle.pair_rotation(dc, dl, (j, i))
        assert (a is None and b is None) or a.tobytes() == b.tobytes()
