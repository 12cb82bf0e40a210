"""The exact-sum mode-B reference (tests/mode_b_reference.py) against the oracle's NIDCost::operator()<double>, on the CPU:
before the GPU suite (tests/test_gpu_mode_b_edges.py) holds K2 / K3 to it, it must itself be the reference's operation.

- histograms: the oracle sums each bin serially in double, so it is within gamma_(m-1) sum |w| of the exact sum of the
  same m taps (Higham, Accuracy and Stability, eq. 4.4), plus the rounding of the fsum result;
- NID within 1e-12; ok flags equal; inlier counts exact.
Inputs: random clouds of all six camera models, float32-representable and general doubles, the edge-adversarial clouds
(decision edges, clamped corners, tiny images) and the invalid inputs (NaN / Inf coordinates, camera centre, intensities
outside [0, 1) and NaN)."""
import numpy as np
import pytest

import mode_b_reference as R
import util
from direct_visual_lidar_calibration_b200 import synthetic as _S

util.S = _S
U = R.U


def _gamma(m):
    m = np.asarray(m, dtype=np.float64)
    return m * U / (1.0 - m * U)


def _compare(oracle, model, intr, dist, image, pts, ins, bins, tp):
    cam = oracle.create_camera(model, intr, dist)
    ex = R.Exact(oracle, cam, image, pts, ins, bins, tp)
    ok, nid, hist = oracle.nid_cost_bspline(cam, image, pts, ins, bins, tp)
    bound = _gamma(np.maximum(ex.taps - 1, 0)) * ex.abs_sum + np.abs(ex.hist) * U
    assert np.all(np.abs(hist - ex.hist) <= bound), np.max(np.abs(hist - ex.hist) - bound)
    assert np.array_equal(ex.taps == 0, hist == 0) or np.all(hist[ex.taps == 0] == 0)
    assert ok == bool(np.isfinite(ex.nid))
    if ok:
        assert abs(nid - float(ex.nid)) <= 1e-12, (nid, float(ex.nid))
    # the inlier count is exact: each point's 16 weights sum to 1 (to ~1e-15), so the lidar marginal rounds to it
    assert np.array_equal(np.rint(hist.sum(axis=0)), ex.points)
    return ex


@pytest.mark.parametrize("f32", [True, False])
@pytest.mark.parametrize("model", util.MODELS)
def test_random_clouds(oracle, model, f32):
    pr = util.random_problem(model, n=6000, seed=91, f32=f32)
    Ts = util.random_poses(pr["T"], 3, seed=5)
    for bins, T in zip((16, 5, 17), Ts):
        ex = _compare(oracle, model, pr["intrinsics"], pr["distortion"], pr["image"], pr["points"], pr["intensities"], bins, R.sophus_params(T))
        assert ex.n_inliers > 1000


@pytest.mark.parametrize("size", [None, (1, 1), (2, 3), (5, 2), (3, 5)])
@pytest.mark.parametrize("model", util.MODELS)
def test_edge_clouds(oracle, model, size):
    for f32 in (False, True):
        pr = R.edge_problem(oracle, model, size=size, seed=7, f32=f32)
        ex = _compare(oracle, model, pr["intrinsics"], pr["distortion"], pr["image"], pr["points"], pr["intensities"], 16, pr["tp"])
        assert ex.n_inliers > (100 if size is None else 20)
        if size is None and not f32 and model != "equirectangular":  # equirectangular u never goes below 0
            # the strip u in (-1, 0) truncates to -1 under floor(): rejected in mode B (mode A's int() cast accepts it)
            strip = (ex.u > -1.0) & (ex.u < 0.0) & (ex.v > 0.0) & (ex.v < pr["H"])
            assert strip.any() and not ex.inlier[strip].any()


@pytest.mark.parametrize("model", util.MODELS)
def test_invalid_inputs(oracle, model):
    pr = R.invalid_problem(model, seed=3)
    for tp in pr["tps"]:
        ex = _compare(oracle, model, pr["intrinsics"], pr["distortion"], pr["image"], pr["points"], pr["intensities"], 16, tp)
        assert not ex.inlier[np.r_[0:8, 9]].any()  # NaN / Inf coordinates never pass the bounds test (floor -> INT_MIN)


def test_fixed_point_scale():
    """min(40, 62 - ceil(log2 n)): 40 fraction bits up to 2^22 points, fewer above, so n * 2^F <= 2^62."""
    assert [R.fixed_bits(n) for n in (0, 1, 2, 255, 100003, 2**22)] == [40] * 6
    assert R.fixed_bits(2**22 + 1) == 39 and R.fixed_bits(2**24 + 2**20) == 37 and R.fixed_bits(2**31 - 1) == 31
    for n in (2**22 + 1, 2**24 + 2**20, 2**31 - 1):
        assert n * 2 ** R.fixed_bits(n) <= 2**62


def test_exact_sum_is_not_the_serial_sum():
    """The reference sums exactly: a bin of many tiny weights next to a large one is not the serial double sum."""
    w = np.array([1.0] + [2.0**-54] * 1000)
    assert R._fsum_by(np.zeros(w.size, dtype=np.int64), w, 1)[0] == 1.0 + 1000 * 2.0**-54
    assert float(np.cumsum(w)[-1]) == 1.0
