"""GPU suite of the fp32 filters' DECISIONS at their edges: the FoV cone, each camera model's guards, the filter's enable
threshold and the pixel edges of the distorted models, against the CPU oracle.

For float32 clouds every point-pose is first classified in fp32 (classify_lean / classify_lean2 of the persistent kernel,
the equirectangular delta step, classify_fast of the round-1 kernels); a verdict is kept only when it is provably the
reference's.  Random clouds almost never put a point inside a decision's uncertain band (about 1e-6 relative wide on the
cone), so a wrong margin there would pass every other test.  Here the points are placed on the host, in double, with the
oracle as the arbiter: a point is rounded to float32 and then moved to the float32 neighbour (+-k ulps per coordinate)
whose oracle quantity (angle to the optical axis, pixel coordinate, guard value) is closest to the target.

Every case checks
  1. the verify kernels: debug_filter_check reports no verdict that contradicts the exact path, and the fp32 error of
     the accepted verdicts inside the bound (lean classifier, round-1 classifier, and the delta step for equirectangular);
  2. histograms bit-identical to oracle.nid_calculate at the same max_fov (NID within 1e-12) through the persistent
     kernel, the filter kernel variants 2, 3, 4, the exact kernel (variant 1) and the pose sweep kernel (K1s, whose
     scores must also equal the persistent kernel's bit for bit);
  3. that the edge was reached: the oracle confirms the targeted points on the intended side, and the filters defer
     more than a stated share of the targeted point-poses to the exact path.  The count is the cloud's deferred
     point-poses minus those of the same cloud without the targeted points, so the ordinary points' natural deferrals
     (a few per cent) cannot meet the floor on their own."""
import math

import numpy as np
import pytest

import util
from direct_visual_lidar_calibration_b200 import _lib
from direct_visual_lidar_calibration_b200 import initial_guess as ig
from direct_visual_lidar_calibration_b200 import synthetic as _S

pytestmark = pytest.mark.gpu
NID_TOL = 1e-12


# ---- placement ---------------------------------------------------------------------------------------------------------


def _camera_frame(T, p):
    """T p in Eigen's operation order (as tests/viewer_oracle.py)."""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], axis=1)


def _to_cloud(T, pc):
    """Inverse of _camera_frame in double (the float32 rounding comes after)."""
    return (pc - T[:3, 3]) @ T[:3, :3]


def _nz(T, p):
    """z / |p| of the camera-frame point: the reference's FoV quantity (cost_calculator_nid.cpp:32)."""
    pc = _camera_frame(T, p)
    n2 = (pc[:, 0] * pc[:, 0] + pc[:, 1] * pc[:, 1]) + pc[:, 2] * pc[:, 2]
    return pc[:, 2] / np.sqrt(n2)


def _refine(pts, q, target, k=3):
    """Round pts (M, 3) to float32, then pick among the float32 neighbours (+-k ulps per coordinate) the one whose q is
    closest to target.  -> (float32-representable points as float64, their q)."""
    p32 = np.asarray(pts, dtype=np.float64).astype(np.float32)
    sp = np.spacing(np.abs(p32))
    best = p32.astype(np.float64)
    qb = q(best)
    err = np.abs(qb - target)
    err = np.where(np.isfinite(err), err, np.inf)
    steps = np.arange(-k, k + 1, dtype=np.float32)
    for dx in steps:
        for dy in steps:
            for dz in steps:
                cand = (p32 + np.stack([dx * sp[:, 0], dy * sp[:, 1], dz * sp[:, 2]], axis=1)).astype(np.float32).astype(np.float64)
                qc = q(cand)
                e = np.abs(qc - target)
                m = e < err
                best[m], qb[m], err[m] = cand[m], qc[m], e[m]
    return best, qb


def _cone_points(rng, n, fov, eps, T, near=None, rg_range=(0.5, 25.0)):
    """n float32 points at angle fov (1 + eps) from the optical axis at pose T (relative offset, oracle's arithmetic).
    near = (camera-frame point c on the cone, radius): the points lie within about radius of c instead."""
    a = fov * (1.0 + eps)
    if near is None:
        az = rng.uniform(0.0, 2.0 * math.pi, 4 * n)
        rg = rng.uniform(*rg_range, 4 * n)
    else:
        c = near[0] + rng.uniform(-near[1], near[1], (4 * n, 3))
        az, rg = np.arctan2(c[:, 1], c[:, 0]), np.linalg.norm(c, axis=1)
    pc = np.stack([rg * math.sin(a) * np.cos(az), rg * math.sin(a) * np.sin(az), rg * math.cos(a)], axis=1)
    q = lambda p: np.arccos(np.clip(_nz(T, p), -1.0, 1.0)) / fov - 1.0
    pts, got = _refine(_to_cloud(T, pc), q, eps)
    keep = np.argsort(np.abs(got - eps), kind="stable")[:n]  # the best quarter of the candidates
    return pts[keep], got[keep]


def _assert_placed(got, eps):
    """The oracle puts every targeted point where the case says: on the side of the cone eps says, close to the target."""
    tol = max(0.3 * abs(eps), 5e-10)
    assert np.abs(got - eps).max() <= tol, (eps, np.abs(got - eps).max())
    if eps != 0.0:
        assert np.all(np.sign(got) == np.sign(eps)), eps


def _problem(model, targets, n_plain=20_000, seed=0, intr=None, dist=None, size=None):
    """A random problem of this model whose cloud also holds the targeted points, scattered over random indices (both
    parities, next to ordinary points: both halves of classify_lean2's pairs see them).  -> (problem, target indices)."""
    rng = np.random.default_rng(seed)
    pr = util.random_problem(model, n=n_plain + len(targets), seed=seed, size=size)
    if intr is not None:
        pr["intrinsics"], pr["distortion"] = intr, dist
    at = rng.permutation(len(pr["points"]))[: len(targets)]
    pr["points"][at, :3] = targets
    assert np.all(pr["points"][:, :3] == pr["points"][:, :3].astype(np.float32))
    assert {0, 1} <= set((at % 2).tolist())
    return pr, at


def _cost(V, pr, max_fov=None):
    cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    return V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]), V.NIDCostParams(16), max_fov=max_fov)


def _oracle_fov(O, pr, max_fov=None):
    cam = O.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
    return cam, (O.estimate_camera_fov(cam, pr["W"], pr["H"]) if max_fov is None else max_fov)


def _oracle_eval(O, pr, Ts, fov):
    cam, _ = _oracle_fov(O, pr, fov)
    out = [O.nid_calculate(cam, pr["image"], pr["points"], pr["intensities"], 16, fov, T) for T in Ts]
    return np.array([o[0] for o in out]), np.stack([o[1] for o in out])


def _assert_nid(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    m = ~np.isnan(a)
    assert np.all(np.abs(a[m] - b[m]) < NID_TOL), np.abs(a[m] - b[m]).max()


def _in_image(O, pr, T, pts):
    """Share of pts that land in the image at pose T when the FoV test is left out (oracle projection, truncation)."""
    cam, _ = _oracle_fov(O, pr)
    uv = O.project(cam, _camera_frame(T, pts))
    with np.errstate(invalid="ignore"):
        ok = (np.trunc(uv[:, 0]) >= 0) & (np.trunc(uv[:, 0]) < pr["W"]) & (np.trunc(uv[:, 1]) >= 0) & (np.trunc(uv[:, 1]) < pr["H"])
    return float(np.mean(ok))


def _deferred(V, pr, Ts, max_fov, delta):
    """Deferred point-poses of the verify kernels (lean, round-1, delta step) and of one persistent pose-list call."""
    cost = _cost(V, pr, max_fov)
    out = {}
    for key, variant, dl in [("lean", 0, False), ("round1", 4, False)] + ([("delta", 0, True)] if delta else []):
        cost.set_kernel_variant(variant)
        out[key] = cost.debug_filter_check(Ts, delta=dl)[1]
    cost.set_kernel_variant(0)
    cost.reset_profile()
    cost.calculate_batch(Ts)
    prof = cost.profile()
    out["persistent"] = prof["deferred_plain"] + prof["deferred_delta"]
    out["sweep"] = _sweep(cost, Ts)[2]
    return out


def _sweep(cost, Ts):
    """The pose sweep kernel on Ts whatever the cloud size: (NID, histograms, (point, pose) pairs it deferred)."""
    nid, hist = ig.sweep_poses([cost], Ts, return_hist=True, kernel_only=True)
    deferred = int(_lib.load_library().vlcal_nid_debug_sweep_last_deferred())
    assert deferred >= 0
    return nid, hist, deferred


def _check(V, O, pr, Ts, max_fov=None, at=None, n_band=0, floor=0.5, name=""):
    """Checks 1-3 of the module docstring.  at: indices of the targeted points; n_band: targeted point-poses that sit in
    an uncertain band -- the lean and round-1 classifiers, the persistent kernel and (equirectangular) the delta step must
    each defer more than floor * n_band point-poses beyond what the cloud without the targets defers.  Equirectangular
    cases also run the delta step's verify kernel.  -> deferred point-poses per path, and the delta passes."""
    delta = pr["model"] == "equirectangular"
    cost = _cost(V, pr, max_fov)
    assert cost.filter_enabled and cost.points_are_f32, name
    fov = cost.max_fov
    if max_fov is not None:
        assert fov == max_fov
    ref_nid, ref_hist = _oracle_eval(O, pr, Ts, fov)
    n_pp = len(pr["points"]) * len(Ts)
    out = {}
    # 1. verify kernels: lean classifier (packed pairs), round-1 classifier, delta step (each group of 8 poses anchored
    # at its central pose)
    checks = [("lean", 0, False), ("round1", 4, False)] + ([("delta", 0, True)] if delta else [])
    for key, variant, dl in checks:
        cost.set_kernel_variant(variant)
        got_pp, deferred, mismatches, ratio = cost.debug_filter_check(Ts, delta=dl)
        assert got_pp == n_pp and mismatches == 0 and ratio < 1.0, (name, key, got_pp, deferred, mismatches, ratio)
        out[key] = deferred
    # 2. histograms: persistent kernel (pose list), filter variants 2 / 3 / round-1 4, exact 1
    cost.set_kernel_variant(0)
    cost.reset_profile()
    nid, hist = cost.calculate_batch(Ts, return_hist=True)
    prof = cost.profile()
    assert prof["kernel_launches"] == 1, (name, prof)
    assert np.array_equal(hist, ref_hist), (name, int(np.abs(hist.astype(np.int64) - ref_hist).sum()))
    _assert_nid(nid, ref_nid)
    out["persistent"] = prof["deferred_plain"] + prof["deferred_delta"]
    out["delta_passes"] = prof["delta_passes"]
    pk_nid = nid
    for variant in (2, 3, 4, 1):
        cost.set_kernel_variant(variant)
        nid, hist = cost.calculate_batch(Ts, return_hist=True)
        assert np.array_equal(hist, ref_hist), (name, variant, int(np.abs(hist.astype(np.int64) - ref_hist).sum()))
        _assert_nid(nid, ref_nid)
    cost.set_kernel_variant(0)
    # K1s: groups of 4 poses, its own copy of the bound and its own deferral queue
    nid, hist, out["sweep"] = _sweep(cost, Ts)
    assert np.array_equal(hist, ref_hist), (name, "sweep", int(np.abs(hist.astype(np.int64) - ref_hist).sum()))
    _assert_nid(nid, ref_nid)
    assert np.array_equal(nid, pk_nid, equal_nan=True), name
    # 3. the edge was reached: deferrals of the targeted points, over those of the same cloud without them
    keys = ("lean", "round1", "persistent", "sweep") + (("delta",) if delta else ())
    if n_band:
        base = _deferred(V, dict(pr, points=np.delete(pr["points"], at, axis=0), intensities=np.delete(pr["intensities"], at)), Ts, max_fov, delta)
        for key in keys:
            out[key + "_targets"] = out[key] - base[key]
            assert out[key + "_targets"] > floor * n_band, (name, key, out[key], base[key], n_band)
    print(f"{name}: {n_band} targeted point-poses in the band; deferred " + ", ".join(
        f"{k} {out[k]}" + (f" ({out[k + '_targets']} by the targets)" if n_band else "") for k in keys) + f" of {n_pp}")
    return out


def _second_pose(T):
    return _S.perturb(T, (1.5, -1.0, 2.0), (0.05, -0.03, 0.02))


# ---- 1. the FoV cone at an explicit max_fov ----------------------------------------------------------------------------

# model -> max_fov values (rad) at which the cone crosses the image interior of util.CAMERAS; the second value of fisheye,
# omnidir and equirectangular is beyond 90 degrees (cos_fov < 0; fisheye: the cone's points project through |z|)
CONE_FOVS = {
    "plumb_bob": [0.6],
    "rational_polynomial": [0.6],
    "atan": [0.6],
    "fisheye": [0.9, 2.1],
    "omnidir": [1.2, 1.9],
    "equirectangular": [1.0, 2.2],
}
CONE_OFFSETS = [0.0, 1e-9, -1e-9, 1e-7, -1e-7, 1e-5, -1e-5]  # relative, in angle
IN_BAND = 1e-7  # every offset up to this one lies inside every model's uncertain band


@pytest.mark.parametrize("model,fov", [(m, f) for m, fs in CONE_FOVS.items() for f in fs])
def test_fov_cone_at_an_explicit_max_fov(gpu, oracle, model, fov):
    rng = np.random.default_rng(int(fov * 1000) + len(model))
    T0 = util.random_problem(model, n=16)["T"]
    Ts = np.stack([T0, _second_pose(T0)])
    groups, n_band = [], 0
    for T in Ts:
        for eps in CONE_OFFSETS:
            pts, got = _cone_points(rng, 800, fov, eps, T)
            _assert_placed(got, eps)
            groups.append(pts)
            n_band += len(pts) if abs(eps) <= IN_BAND else 0
            if eps == 0.0:
                share = _in_image(oracle, {"model": model, **_cam_dict(model)}, T, pts)
                assert share > 0.2, (model, fov, share)  # the cone crosses the image interior
    pr, at = _problem(model, np.concatenate(groups), seed=11)
    _check(gpu, oracle, pr, Ts, max_fov=fov, at=at, n_band=n_band, name=f"{model} cone {fov}")


def _cam_dict(model):
    intr, dist, (W, H) = util.CAMERAS[model]
    return {"intrinsics": intr, "distortion": dist, "W": W, "H": H}


def test_fov_cone_through_the_estimated_fov_of_a_folding_lens(gpu, oracle):
    """A C2-like plumb_bob (1920 x 1080, f = 1000, distortion that folds back): the reference's own max_fov estimate
    lies beyond the image corner's angle, and the cone still crosses the image."""
    intr, dist = [1000.0, 1000.0, 960.0, 540.0], [-0.04, 0.08, 1e-4, -3e-4, -0.04]
    pr0 = util.random_problem("plumb_bob", n=16, size=(1920, 1080))
    pr0["intrinsics"], pr0["distortion"] = intr, dist
    cam, fov = _oracle_fov(oracle, pr0)
    corner = math.atan(math.hypot(960.0, 540.0) / 1000.0)
    assert fov > corner + 0.1, (fov, corner)
    rng = np.random.default_rng(12)
    T0 = pr0["T"]
    Ts = np.stack([T0, _second_pose(T0)])
    groups, n_band = [], 0
    for T in Ts:
        for eps in CONE_OFFSETS:
            pts, got = _cone_points(rng, 800, fov, eps, T)
            _assert_placed(got, eps)
            groups.append(pts)
            n_band += len(pts) if abs(eps) <= IN_BAND else 0
    pr, at = _problem("plumb_bob", np.concatenate(groups), seed=13, intr=intr, dist=dist, size=(1920, 1080))
    # the cone cuts through the image: with the FoV test left out, some of the points placed on it at T0 land in it
    on_cone = np.concatenate(groups[: len(CONE_OFFSETS)])
    n_in = round(_in_image(oracle, pr, T0, on_cone) * len(on_cone))
    assert n_in >= 20, n_in
    _check(gpu, oracle, pr, Ts, at=at, n_band=n_band, name="C2-like cone")


# ---- 2. the filter enable threshold cos(max_fov) >= 0.05 ----------------------------------------------------------------


def _threshold_fovs():
    """(fov - 1 ulp, fov, fov + 1 ulp) with fov the largest double whose libm cosine is >= 0.05."""
    f = math.acos(0.05)
    while math.cos(f) < 0.05:
        f = math.nextafter(f, 0.0)
    while math.cos(math.nextafter(f, 4.0)) >= 0.05:
        f = math.nextafter(f, 4.0)
    return math.nextafter(f, 0.0), f, math.nextafter(f, 4.0)


@pytest.mark.parametrize("model", ["plumb_bob", "rational_polynomial", "atan"])
def test_filter_enable_threshold(gpu, oracle, model):
    below, at, above = _threshold_fovs()
    assert math.cos(at) >= 0.05 > math.cos(above)
    rng = np.random.default_rng(20)
    T0 = util.random_problem(model, n=16)["T"]
    groups = [_cone_points(rng, 500, at, eps, T0)[0] for eps in (0.0, 1e-9, -1e-9, 1e-7)]
    pr, _ = _problem(model, np.concatenate(groups), seed=21)
    Ts = np.stack([T0, _second_pose(T0)])
    for fov in (below, at):
        _check(gpu, oracle, pr, Ts, max_fov=fov, n_band=0, name=f"{model} threshold fov {fov!r}")
    cost = _cost(gpu, pr, above)
    assert not cost.filter_enabled
    ref_nid, ref_hist = _oracle_eval(oracle, pr, Ts, above)
    for variant in (0, 1):
        cost.set_kernel_variant(variant)
        nid, hist = cost.calculate_batch(Ts, return_hist=True)
        assert np.array_equal(hist, ref_hist) and hist.sum() > 1000
        _assert_nid(nid, ref_nid)


# ---- 3. pixel edges of the distorted models ----------------------------------------------------------------------------

# px from an integer column / row.  A float32 ulp of a coordinate moves the projection by ~1e-5 px; the neighbour search
# reaches ~1e-6 px for most points, and every offset from 1e-4 px down lies inside the filters' pixel band
EDGE_OFFSETS = [1e-3, -1e-4, 1e-5, -1e-6]
EDGE_IN_BAND = 1e-5


def _direction_for_pixel(O, cam, uv, z):
    """Camera-frame points at depth-like scale z whose oracle projection is uv: Newton on the normalised plane."""
    xy = np.full((len(uv), 2), 0.01)  # off the axis (fisheye: 0 / 0 there)
    for _ in range(30):
        p = np.c_[xy * z[:, None], z]
        f = O.project(cam, p) - uv
        J = np.empty((len(uv), 2, 2))
        h = 1e-7
        for k in range(2):
            d = np.zeros_like(xy)
            d[:, k] = h
            J[:, :, k] = (O.project(cam, np.c_[(xy + d) * z[:, None], z]) - uv - f) / h
        det = J[:, 0, 0] * J[:, 1, 1] - J[:, 0, 1] * J[:, 1, 0]
        ok = np.isfinite(det) & (np.abs(det) > 1e-30) & np.isfinite(f).all(axis=1)
        det = np.where(ok, det, 1.0)
        step = np.stack([J[:, 1, 1] * f[:, 0] - J[:, 0, 1] * f[:, 1], J[:, 0, 0] * f[:, 1] - J[:, 1, 0] * f[:, 0]], axis=1) / det[:, None]
        xy -= np.where(ok[:, None], step, 0.0)
    return np.c_[xy * z[:, None], z]


def _equirect_points(W, H, uv, rng, rg_range=(0.5, 25.0)):
    """Inverse of equirectangular.hpp:21-27: lon = atan2(x, z), lat = -asin(y / |p|)."""
    lon = (uv[:, 0] / W - 0.5) * 2.0 * math.pi
    lat = (0.5 - uv[:, 1] / H) * math.pi
    rg = rng.uniform(*rg_range, len(uv))
    return np.stack([rg * np.cos(lat) * np.sin(lon), -rg * np.sin(lat), rg * np.cos(lat) * np.cos(lon)], axis=1)


def _edge_points(O, cam, pr0, T, axis, off, n, tol, rng, strips=True, z_range=(1.0, 20.0), near=None):
    """n float32 points whose oracle coordinate `axis` at pose T lies within tol of an integer edge + off: interior
    edges, and with strips=True also 0 and -1 (the (-1, 0) truncation strip) and W / H.  Depth (equirectangular: range)
    in z_range; near = (pixel, spread): only edges and pixels within spread px of it.  -> (points, their edges)."""
    W, H = pr0["W"], pr0["H"]
    m = 4 * n  # candidates
    if near is None:
        edge = rng.integers(1, (W if axis == 0 else H), m).astype(np.float64)
        if strips:
            edge[:20], edge[20:40], edge[40:60] = 0.0, -1.0, (W if axis == 0 else H)
        uv = np.stack([rng.uniform(5.0, W - 5.0, m), rng.uniform(5.0, H - 5.0, m)], axis=1)
    else:
        s = int(near[1])
        edge = np.floor(near[0][axis]) + rng.integers(-s, s + 2, m)
        uv = near[0] + rng.uniform(-near[1], near[1], (m, 2))
    uv[:, axis] = edge + off
    if pr0["model"] == "equirectangular":
        pc = _equirect_points(W, H, uv, rng, z_range)
    else:
        pc = _direction_for_pixel(O, cam, uv, rng.uniform(*z_range, m))
    q = lambda p: O.project(cam, _camera_frame(T, p))[:, axis] - (edge + off)
    pts, got = _refine(_to_cloud(T, pc), q, 0.0)
    ok = np.abs(got) <= tol  # got: distance from the targeted offset, px (NaN: Newton did not converge)
    assert ok.sum() >= n, (pr0["model"], axis, off, ok.sum())
    keep = np.nonzero(ok)[0][:n]
    return pts[keep], edge[keep]


@pytest.mark.parametrize("model", util.MODELS)
def test_pixel_edges_of_every_model(gpu, oracle, model):
    """Points within 1e-3 ... 1e-6 px of interior columns (and, in a second group, rows), in the (-1, 0) truncation strip
    and at u = W, v = H."""
    rng = np.random.default_rng(30)
    pr0 = util.random_problem(model, n=16)
    cam, _ = _oracle_fov(oracle, pr0)
    T0 = pr0["T"]
    Ts = np.stack([T0, T0])  # the same pose twice: both halves of a pass see the same edges
    groups, n_band = [], 0
    for axis in (0, 1):
        for off in EDGE_OFFSETS:
            pts, _ = _edge_points(oracle, cam, pr0, T0, axis, off, 400, 0.3 * abs(off), rng)
            groups.append(pts)
            if abs(off) <= EDGE_IN_BAND:
                n_band += 2 * len(pts)
    pr, at = _problem(model, np.concatenate(groups), seed=31)
    _check(gpu, oracle, pr, Ts, at=at, n_band=n_band, floor=0.5, name=f"{model} pixel edges")


def _shift_onto_edge(O, cam, T0, p, axis, target, upper):
    """Pose T0 with its translation moved along camera axis `axis` by a sub-ulp double amount s, bisected until the
    oracle coordinate of point p is at the target: the first double s with coordinate >= target (upper) or the last one
    below it.  -> (pose, achieved coordinate)."""
    def coord(s):
        T = T0.copy()
        T[axis, 3] += s
        return T, float(O.project(cam, _camera_frame(T, p[None]))[0, axis])

    lo, hi = -1e-6, 1e-6  # moves the projection by >= 2e-5 px, against a residual below 1e-6 px
    assert coord(lo)[1] < target <= coord(hi)[1]
    while True:
        mid = 0.5 * (lo + hi)
        if mid in (lo, hi):
            break
        if coord(mid)[1] >= target:
            hi = mid
        else:
            lo = mid
    return coord(hi if upper else lo)


@pytest.mark.parametrize("model", ["plumb_bob", "omnidir", "rational_polynomial"])
def test_pixel_edges_at_1e_12_px_by_sub_ulp_pose_shifts(gpu, oracle, model):
    """The distorted models whose exact path uses + - * / sqrt only: the exact path must round as the reference does,
    down to 1e-12 px.  A float32 ulp of a coordinate moves the projection by ~1e-5 px, so these cases shift the pose
    instead: for each of 24 poses (three batches of 8), a double translation bisected so that one chosen point lies
    exactly on an interior column or row edge, 1e-12 px above or below it.  The other edge points stay within ~1e-6 px
    of their edges at every pose."""
    rng = np.random.default_rng(35)
    pr0 = util.random_problem(model, n=16)
    cam, _ = _oracle_fov(oracle, pr0)
    T0 = pr0["T"]
    per_axis = [_edge_points(oracle, cam, pr0, T0, axis, 0.0, 300, 1e-6, rng, strips=False) for axis in (0, 1)]
    Ts, hits = [], []
    for k in range(24):
        axis, j = k % 2, k // 2
        off = (0.0, 1e-12, -1e-12)[j % 3]
        p, edge = per_axis[axis][0][j], per_axis[axis][1][j]
        T, c = _shift_onto_edge(oracle, cam, T0, p, axis, edge + off, upper=off >= 0.0)
        d = c - edge
        # the oracle puts the chosen point where the case says: on the edge (at most a double ulp of the coordinate
        # above it), or 1e-12 px above / below it
        if off == 0.0:
            assert 0.0 <= d < 2.5e-13, (k, d)
        else:
            assert np.sign(d) == np.sign(off) and abs(d - off) < 2.5e-13, (k, d)
        Ts.append(T)
        hits.append(d)
    Ts = np.stack(Ts)
    assert np.abs(Ts[:, :3, 3] - T0[:3, 3]).max() < 1e-6
    pts = np.concatenate([per_axis[0][0], per_axis[1][0]])
    pr, at = _problem(model, pts, seed=36)
    pr["T"] = T0
    out = _check(gpu, oracle, pr, Ts, at=at, n_band=len(pts) * len(Ts), floor=0.9, name=f"{model} edges at 1e-12 px")
    print(f"{model}: chosen points at {', '.join(f'{h:.1e}' for h in hits[:6])} ... px from their edges; {out['lean_targets']} deferred")


# ---- 4. model guards ---------------------------------------------------------------------------------------------------


def _guard_points(rng, n, T, q, target, make):
    pc = make(4 * n)
    pts, got = _refine(_to_cloud(T, pc), q, target)
    keep = np.argsort(np.abs(got - target), kind="stable")[:n]
    return pts[keep], got[keep]


def _normalised_radius(T, p):
    pc = _camera_frame(T, p)
    x, y = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
    return np.sqrt(x * x + y * y)


@pytest.mark.parametrize("d0", [0.9, 1e-7, "below"])
def test_atan_branch_at_r_1e_3(gpu, oracle, d0):
    """atan.hpp switches from the identity to the atan factor at r = 1e-3 (a 0.03 px step with d0 = 0.9): points at
    r = 1e-3 and a float32 ulp or a small offset either side.  d0 = 1e-7 turns the distortion on, one double below off."""
    d0 = math.nextafter(1e-7, 0.0) if d0 == "below" else d0
    intr = [400.0, 400.0, 320.0, 240.0]
    rng = np.random.default_rng(40)
    T0 = np.eye(4)
    ulp_r = float(np.spacing(np.float32(1e-3)))
    offsets = [0.0, ulp_r, -ulp_r, 1e-8, -1e-8, 1e-6, -1e-6]

    groups, n_band = [], 0
    for off in offsets:
        def make(m, r=1e-3 + off):
            az = rng.uniform(0.0, 2.0 * math.pi, m)
            z = rng.uniform(1.0, 20.0, m)
            return np.stack([r * z * np.cos(az), r * z * np.sin(az), z], axis=1)

        pts, got = _guard_points(rng, 600, T0, lambda p: _normalised_radius(T0, p), 1e-3 + off, make)
        assert np.abs(got - (1e-3 + off)).max() <= max(0.2 * abs(off), 2e-11), off
        if off != 0.0:
            assert np.all(np.sign(got - 1e-3) == np.sign(off))
        groups.append(pts)
        n_band += len(pts) if abs(off) <= 1e-8 else 0
    pr, at = _problem("atan", np.concatenate(groups), seed=41, intr=intr, dist=[d0])
    pr["T"] = T0
    Ts = np.stack([T0, _S.perturb(T0, (0.0, 0.0, 0.5), (0.0, 0.0, 0.0))])  # pose 2: rotation about the axis keeps r
    assert np.allclose(_normalised_radius(Ts[1], groups[0]), 1e-3, rtol=1e-6)
    # the step only exists while the distortion is on; the guard only defers then
    _check(gpu, oracle, pr, Ts, at=at, n_band=2 * n_band if d0 >= 1e-7 else 0, name=f"atan r = 1e-3, d0 = {d0!r}")


def test_rational_polynomial_denominator_guards(gpu, oracle):
    """den = 1 - r^2 (k4 = -1): crosses den_lb's 0.1 at r^2 = 0.9 and the reference's 1e-8 branch (rational_polynomial.hpp:33)
    at r^2 = 1 - 1e-8, where the projection jumps from far outside the image (r_coeff = 1e8) into it (r_coeff = 1)."""
    intr, dist = [200.0, 200.0, 320.0, 240.0], [0.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0]  # r = 1 lands inside the image
    rng = np.random.default_rng(50)
    T0 = np.eye(4)
    fov = 0.9  # tan^2 = 1.59: the whole crossing lies inside the FoV

    def den(p):
        pc = _camera_frame(T0, p)
        x, y = pc[:, 0] / pc[:, 2], pc[:, 1] / pc[:, 2]
        return 1.0 + -1.0 * ((x * x) + (y * y))

    groups, n_band, jump = [], 0, []
    for target, offs in ((0.1, (0.0, 1e-7, -1e-7, 1e-5)), (1e-8, (0.0, 3e-9, -3e-9, 1e-7))):
        for off in offs:
            r = math.sqrt(1.0 - (target + off))

            def make(m, r=r):
                az = rng.uniform(0.0, 2.0 * math.pi, m)
                z = rng.uniform(1.0, 20.0, m)
                return np.stack([r * z * np.cos(az), r * z * np.sin(az), z], axis=1)

            pts, got = _guard_points(rng, 600, T0, den, target + off, make)
            assert np.abs(got - (target + off)).max() <= max(0.3 * abs(off), 1e-9 if target == 1e-8 else 1e-8), (target, off)
            if off != 0.0:
                assert np.all(np.sign(got - target) == np.sign(off))
            groups.append(pts)
            n_band += len(pts)
            if target == 1e-8 and off != 0.0:
                jump.append((off, _in_image(oracle, {"model": "rational_polynomial", "intrinsics": intr, "distortion": dist, "W": 640, "H": 480}, T0, pts)))
    # in the image just below 1e-8 (r_coeff = numerator), far outside just above it (r_coeff = 1 / den)
    assert [s > 0.3 for o, s in jump if o < 0] == [True] and all(s == 0.0 for o, s in jump if o > 0), jump
    pr, at = _problem("rational_polynomial", np.concatenate(groups), seed=51, intr=intr, dist=dist)
    pr["T"] = T0
    _check(gpu, oracle, pr, np.stack([T0, T0]), max_fov=fov, at=at, n_band=2 * n_band, floor=0.9, name="rational denominator")


def test_omnidir_guard_sz_plus_xi(gpu, oracle):
    """xi = 0.6: sz + xi = 0.1 at 120 degrees from the axis, inside a 132-degree FoV."""
    intr, dist = [300.0, 300.0, 320.0, 240.0, 0.6], [-0.1, 0.02, 1e-3, -2e-3]
    rng = np.random.default_rng(60)
    T0 = np.eye(4)
    q = lambda p: _nz(T0, p) + 0.6
    groups, n_band = [], 0
    for off in (0.0, 1e-9, -1e-9, 1e-7, -1e-7, 1e-5, -1e-5):
        a = math.acos(0.1 + off - 0.6)

        def make(m, a=a):
            az = rng.uniform(0.0, 2.0 * math.pi, m)
            rg = rng.uniform(0.5, 25.0, m)
            return np.stack([rg * math.sin(a) * np.cos(az), rg * math.sin(a) * np.sin(az), rg * math.cos(a)], axis=1)

        pts, got = _guard_points(rng, 600, T0, q, 0.1 + off, make)
        assert np.abs(got - (0.1 + off)).max() <= max(0.3 * abs(off), 5e-10), off
        if off != 0.0:
            assert np.all(np.sign(got - 0.1) == np.sign(off))
        groups.append(pts)
        n_band += len(pts) if abs(off) <= 1e-7 else 0
    pr, at = _problem("omnidir", np.concatenate(groups), seed=61, intr=intr, dist=dist)
    pr["T"] = T0
    _check(gpu, oracle, pr, np.stack([T0, T0]), max_fov=2.3, at=at, n_band=2 * n_band, name="omnidir sz + xi")


def test_fisheye_optical_axis(gpu, oracle):
    """r -> 0: on the axis the reference computes theta_d / r = 0 / 0 (NaN, the point is skipped); next to it the point
    lands on the principal point.  Both fall within the guard r > 8 delta."""
    rng = np.random.default_rng(70)
    T0 = np.eye(4)
    m = 600
    z = rng.choice([0.5, 1.0, 3.0, 17.0], m) * rng.choice([1.0, -1.0], m, p=[0.8, 0.2])
    on_axis = np.stack([np.zeros(m), np.zeros(m), z], axis=1)
    tiny = np.stack([rng.choice([1e-30, 1e-20, 1e-10, 1e-7], m) * rng.choice([1.0, -1.0], m), np.zeros(m), np.abs(z)], axis=1)
    tiny[::2, [0, 1]] = tiny[::2, [1, 0]]
    pts = np.concatenate([on_axis, tiny]).astype(np.float32).astype(np.float64)
    cam, _ = _oracle_fov(oracle, {"model": "fisheye", **_cam_dict("fisheye")})
    uv = oracle.project(cam, on_axis)
    assert np.isnan(uv).all()
    uv = oracle.project(cam, pts[m:])
    assert np.isfinite(uv).all() and np.abs(uv - [320.0, 240.0]).max() < 1e-3
    pr, at = _problem("fisheye", pts, seed=71)
    # on-axis points behind the camera (z < 0) are certain FoV rejects at both max_fov values; all others sit in the band
    n_front = int(np.sum(pts[:, 2] > 0.0))
    pr["T"] = T0
    Ts = np.stack([T0, _S.perturb(T0, (0.0, 0.0, 1.0), (0.0, 0.0, 0.0))])  # rotation about the axis keeps both groups
    _check(gpu, oracle, pr, Ts, at=at, n_band=2 * n_front, floor=0.9, name="fisheye axis")
    _check(gpu, oracle, pr, Ts, max_fov=2.0, at=at, n_band=2 * n_front, floor=0.9, name="fisheye axis, fov 2.0")


def test_equirectangular_centre_branch_and_poles(gpu, oracle):
    """|p|^2 < 1e-3 returns the image centre (equirectangular.hpp:15): points at |p|^2 = 1e-3 and a float32 ulp or a
    small offset either side; and points next to the poles in a batch the delta step takes."""
    rng = np.random.default_rng(80)
    T0 = np.eye(4)

    def n2(p):
        pc = _camera_frame(T0, p)
        return (pc[:, 0] * pc[:, 0] + pc[:, 1] * pc[:, 1]) + pc[:, 2] * pc[:, 2]

    groups, n_band = [], 0
    for off in (0.0, 1e-10, -1e-10, 1e-9, -1e-9, 1e-7, -1e-7):
        make = lambda m, off=off: _S.lidar_directions("sphere", m, rng) * math.sqrt(1e-3 + off)
        pts, got = _guard_points(rng, 600, T0, n2, 1e-3 + off, make)
        assert np.abs(got - (1e-3 + off)).max() <= max(0.3 * abs(off), 2e-11), off
        if off != 0.0:
            assert np.all(np.sign(got - 1e-3) == np.sign(off))
        groups.append(pts)
        n_band += len(pts)
    # poles: r_xz tiny against |y| at every pose of the batch
    m = 2000
    pole = np.stack([rng.uniform(-1e-4, 1e-4, m), rng.choice([-1.0, 1.0], m) * rng.uniform(1.0, 20.0, m), rng.uniform(-1e-4, 1e-4, m)], axis=1)
    groups.append(pole.astype(np.float32).astype(np.float64))
    n_band += m
    pr, at = _problem("equirectangular", np.concatenate(groups), seed=81)
    pr["T"] = T0
    Ts = np.stack([T0] + [_S.perturb(T0, (0.0, 0.0, 0.0), (0.0, 1e-3 * k, 0.0)) for k in range(1, 8)])  # inside the delta gate
    out = _check(gpu, oracle, pr, Ts, at=at, n_band=8 * n_band, floor=0.9, name="equirectangular centre + poles")
    assert out["delta_passes"] == 1, out


# ---- 5. the equirectangular delta step at the cone ----------------------------------------------------------------------


def test_delta_step_at_the_cone(gpu, oracle):
    """Explicit max_fov < pi; a batch of 8 poses inside the delta gate; at every pose k >= 1 a group of points sits on the
    cone (offsets 0 and +-1e-9 ... 1e-7): the delta step's pass and reject radii 0.49 (g~0 - mf) must defer them."""
    fov = 1.3
    rng = np.random.default_rng(90)
    T0 = util.random_problem("equirectangular", n=16)["T"]
    Ts = np.stack([T0] + [_S.perturb(T0, (0.0, 0.0, 0.02 * k), (1e-3 * k, 0.0, -1e-3 * k)) for k in range(1, 8)])
    groups, n_band = [], 0
    for T in Ts[1:]:
        for eps in (0.0, 1e-9, -1e-9, 1e-7, -1e-7):
            pts, got = _cone_points(rng, 300, fov, eps, T)
            _assert_placed(got, eps)
            groups.append(pts)
            n_band += len(pts)
    pr, at = _problem("equirectangular", np.concatenate(groups), seed=91)
    pr["T"] = T0
    out = _check(gpu, oracle, pr, Ts, max_fov=fov, at=at, n_band=n_band, name="delta step at the cone")
    assert out["delta_passes"] == 1, out


# ---- 6. large translations: the max|t| term of the bound -------------------------------------------------------------------
#
# Every fp32 filter bounds the transform error of a point by delta = 5.25 u (|x| + |y| + |z| + max|t|), max|t| over the
# poses that share the bound (a K1p pass, a K1s group, a round-1 pose).  Two geometries make that term matter:
#   (a) a far camera over a near cloud: |t| of 30 and 300 m, the points within about 1 m of the LiDAR origin, so
#       max|t| is nearly all of delta;
#   (b) the map frame (preprocess_map keeps the map's coordinates): points 60 and 450 m from the origin and the camera
#       among them, where R p and t cancel.
# Each translation is moved to about half a float32 ulp from its float32 value, on the side where that rounding pushes
# the targeted points down across their edges.  The pose of largest |t| stands first, in the middle and last of a K1p
# pass and a round-1 launch of 8 poses and of a K1s group of 4, the other one in other slots, among ordinary poses.

FAR_SLOTS = ((0, 0), (13, 0), (23, 0), (5, 1), (18, 1))  # (index in a list of 24 poses, which large-|t| pose)
FAR_DIST = (300.0, 30.0)  # (a): distance of the LiDAR origin from the camera, largest first
MAP_DIST = (450.0, 60.0)  # (b): distance of the camera from the map origin, largest first
FAR_EDGE_OFFSETS = [1e-5, 3e-6, 1e-6, -1e-6]  # px
MAP_EDGE_OFFSETS = {450.0: [1e-3, -1e-3], 60.0: [1e-4, -1e-4]}  # px: the float32 grid of the cloud is coarser there
MAP_CONE_OFFSETS = {450.0: [1e-5, -1e-5, 3e-6], 60.0: [3e-6, -3e-6, 1e-6]}  # relative, in angle


def _push_translation(T, qc, pc0):
    """T with every translation component set to about half a float32 ulp from its float32 value, on the side where
    float32(t) lowers the camera-frame quantity qc at pc0."""
    T = T.copy()
    for k in range(3):
        e = np.zeros((1, 3))
        e[0, k] = 1e-4 * np.linalg.norm(pc0)
        g = float(qc(pc0[None] + e)[0] - qc(pc0[None] - e)[0])
        f = np.float32(T[k, 3])
        T[k, 3] = float(f) + math.copysign(0.49, g) * float(np.spacing(np.abs(f)))
        assert np.float32(T[k, 3]) == f
    return T


def _with_large_poses(T0, large, seed):
    """24 poses around T0 with the large-|t| poses at FAR_SLOTS."""
    Ts = util.random_poses(T0, 24, seed=seed)
    for i, k in FAR_SLOTS:
        Ts[i] = large[k]
    return Ts


def _n_slots(k):
    return sum(1 for _, j in FAR_SLOTS if j == k)


def _angle_q(fov):
    return lambda pc: np.arccos(np.clip(pc[:, 2] / np.linalg.norm(pc, axis=1), -1.0, 1.0)) / fov - 1.0


def _cone_direction_in_image(O, cam, pr0, fov):
    """A unit camera-frame direction at angle fov from the axis that lands in the image (the FoV test left out)."""
    for az in np.linspace(0.0, 2.0 * math.pi, 97)[:-1]:
        d = np.array([math.sin(fov) * math.cos(az), math.sin(fov) * math.sin(az), math.cos(fov)])
        uv = O.project(cam, d[None])[0]
        if np.all(np.isfinite(uv)) and 0.0 <= uv[0] < pr0["W"] and 0.0 <= uv[1] < pr0["H"]:
            return d
    raise AssertionError("the cone misses the image")


def _pixel_direction(O, cam, pr0, uv, dist):
    """The camera-frame point of pixel uv at depth dist (equirectangular: range), as _edge_points places them."""
    if pr0["model"] == "equirectangular":
        return _equirect_points(pr0["W"], pr0["H"], uv[None], np.random.default_rng(0), (dist, dist))[0]
    return _direction_for_pixel(O, cam, uv[None], np.array([dist]))[0]


def _large_pose(T0, pc_origin):
    """T0's rotation with the LiDAR origin at camera-frame point pc_origin."""
    T = T0.copy()
    T[:3, 3] = pc_origin
    return T


def _map_pose(T0, C):
    """T0's rotation with the camera at LiDAR-frame (map) position C."""
    T = T0.copy()
    T[:3, 3] = -T0[:3, :3] @ C
    return T


@pytest.mark.parametrize("model", util.MODELS)
def test_far_camera_near_cloud_at_the_cone(gpu, oracle, model):
    """(a) at the cone: the LiDAR origin on the cone of the widest max_fov of the model, 300 and 30 m away; the targeted
    points within about 1 m of it, at the offsets of section 1."""
    rng = np.random.default_rng(200 + len(model))
    pr0 = util.random_problem(model, n=16)
    cam, _ = _oracle_fov(oracle, pr0)
    fov = CONE_FOVS[model][-1]
    d = _cone_direction_in_image(oracle, cam, pr0, fov)
    groups, n_band, large = [], 0, []
    for k, dist in enumerate(FAR_DIST):
        T = _push_translation(_large_pose(pr0["T"], dist * d), _angle_q(fov), dist * d)
        large.append(T)
        for eps in CONE_OFFSETS:
            pts, got = _cone_points(rng, 300, fov, eps, T, near=(T[:3, 3], 1.0))
            _assert_placed(got, eps)
            assert np.abs(pts).max() < 2.0
            groups.append(pts)
            n_band += _n_slots(k) * len(pts) if abs(eps) <= IN_BAND else 0
    pr, at = _problem(model, np.concatenate(groups), seed=201)
    _check(gpu, oracle, pr, _with_large_poses(pr0["T"], large, seed=202), max_fov=fov, at=at, n_band=n_band, name=f"{model} far cone")


@pytest.mark.parametrize("model", util.MODELS)
def test_far_camera_near_cloud_at_pixel_edges(gpu, oracle, model):
    """(a) at the pixel edges: the LiDAR origin 300 and 30 m away in front of the image centre; targeted points within
    1e-5 ... 1e-6 px of the columns and rows about its pixel, within about 1 m of it."""
    rng = np.random.default_rng(210 + len(model))
    pr0 = util.random_problem(model, n=16)
    cam, _ = _oracle_fov(oracle, pr0)
    uv_c = np.array([0.5 * pr0["W"] + 37.3, 0.5 * pr0["H"] - 23.7])
    groups, n_band, large = [], 0, []
    for k, dist in enumerate(FAR_DIST):
        pc0 = _pixel_direction(oracle, cam, pr0, uv_c, dist)
        spread = float(np.abs(oracle.project(cam, pc0[None] + [0.5, 0.0, 0.0]) - uv_c).max())  # px of 0.5 m there
        T = _push_translation(_large_pose(pr0["T"], pc0), lambda pc, a=k % 2: oracle.project(cam, pc)[:, a], pc0)
        large.append(T)
        for axis in (0, 1):
            for off in FAR_EDGE_OFFSETS:
                pts, _ = _edge_points(oracle, cam, pr0, T, axis, off, 150, 0.3 * abs(off), rng, z_range=(dist - 0.7, dist + 0.7), near=(uv_c, spread))
                assert np.abs(pts).max() < 3.0
                groups.append(pts)
                n_band += _n_slots(k) * len(pts)
    pr, at = _problem(model, np.concatenate(groups), seed=211)
    _check(gpu, oracle, pr, _with_large_poses(pr0["T"], large, seed=212), at=at, n_band=n_band, name=f"{model} far pixel edges")


@pytest.mark.parametrize("model", util.MODELS)
def test_map_frame_cone_and_pixel_edges(gpu, oracle, model):
    """(b): the camera 450 and 60 m from the map origin, the targeted points 15-25 m from it: on the cone (its widest
    max_fov) in one case, on pixel edges (the estimated max_fov) in the other.  Then a whole map-frame cloud: the
    share of point-poses the filters defer there."""
    rng = np.random.default_rng(220 + len(model))
    pr0 = util.random_problem(model, n=16)
    cam, _ = _oracle_fov(oracle, pr0)
    fov = CONE_FOVS[model][-1]
    direction = np.array([0.48, -0.6, 0.64])
    uv_c = np.array([0.5 * pr0["W"] + 37.3, 0.5 * pr0["H"] - 23.7])
    d = _cone_direction_in_image(oracle, cam, pr0, fov)
    for kind in ("cone", "pixel"):
        groups, n_band, large = [], 0, []
        for k, dist in enumerate(MAP_DIST):
            T = _map_pose(pr0["T"], dist * direction)
            if kind == "cone":
                T = _push_translation(T, _angle_q(fov), 20.0 * d)
            else:
                pc0 = _pixel_direction(oracle, cam, pr0, uv_c, 20.0)
                T = _push_translation(T, lambda pc, a=k % 2: oracle.project(cam, pc)[:, a], pc0)
            large.append(T)
            if kind == "cone":
                for eps in MAP_CONE_OFFSETS[dist]:
                    pts, got = _cone_points(rng, 300, fov, eps, T, rg_range=(15.0, 25.0))
                    _assert_placed(got, eps)
                    groups.append(pts)
                    n_band += _n_slots(k) * len(pts)
            else:
                for axis in (0, 1):
                    for off in MAP_EDGE_OFFSETS[dist]:
                        pts, _ = _edge_points(oracle, cam, pr0, T, axis, off, 150, 0.3 * abs(off), rng, z_range=(15.0, 25.0), near=(uv_c, 100.0))
                        groups.append(pts)
                        n_band += _n_slots(k) * len(pts)
            assert np.median(np.linalg.norm(groups[-1], axis=1)) > 0.5 * dist
        pr, at = _problem(model, np.concatenate(groups), seed=221)
        _check(gpu, oracle, pr, _with_large_poses(pr0["T"], large, seed=222), max_fov=fov if kind == "cone" else None, at=at, n_band=n_band,
               name=f"{model} map frame {kind}")
    # a whole cloud in the map frame, seen from its own camera: no targets, the deferred share is reported
    pr = util.random_problem(model, n=20_000, seed=223)
    C = MAP_DIST[0] * direction
    pr["points"][:, :3] = (pr["points"][:, :3] + C).astype(np.float32).astype(np.float64)
    Ts = util.random_poses(pr["T"], 8, seed=224)
    Ts[:, :3, 3] -= np.einsum("nij,j->ni", Ts[:, :3, :3], C)  # the same cameras relative to the moved cloud
    out = _check(gpu, oracle, pr, Ts, name=f"{model} map-frame cloud")
    n_pp = len(pr["points"]) * len(Ts)
    print(f"{model} map-frame cloud at {MAP_DIST[0]:g} m: deferred share lean {out['lean'] / n_pp:.4f}, persistent {out['persistent'] / n_pp:.4f}, "
          f"sweep {out['sweep'] / n_pp:.4f}")
