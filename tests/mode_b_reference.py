"""Exact-sum reference of the mode-B (B-spline soft histogram) NID, NIDCost::operator()<double>
(include/vlcal/costs/nid_cost.hpp:36-107), and the certified bounds the GPU kernels are held to.

Per point, in the reference's operation order and in float64 (numpy never contracts a*b+c):
  camera point  uv = 2 (q x p);  pc = ((p + w uv) + q x uv) + t          (Sophus SO3 action, :47)
  projection    oracle.project (tests/test_reference_pin.py ties it bit for bit to the reference's functors, :51)
  knot          k = int(floor(u)), s = u - k; rejected unless 0 <= kx < W and 0 <= ky < H   (:52-58)
  weights       beta_r = ((C[r][0] * 1 + C[r][1] s) + C[r][2] s^2) + C[r][3] s^3,  w_ij = beta_x[i] * beta_y[j]   (:62-77)
  bins          image bin of the clamped knot pixel, min(int(u8 * (1/255.0) * bins), bins - 1)          (:72-79)
                lidar bin max(0, min(bins - 1, int(intensity * bins))), x86 truncation (NaN -> INT_MIN -> 0)  (:49)
Each joint bin is the math.fsum (correctly rounded) of its taps, i.e. the exact sum of the reference's per-tap doubles;
the inlier count per lidar bin is an exact integer; the NID is evaluated from those in np.longdouble.

A kernel that rounds every tap once to a multiple of 2^-F and sums the integers exactly is then within

    |hist_gpu[b] - fsum[b]| <= taps[b] * (2^-(F+1) + tap_uv) + (|hist_gpu[b]| + |fsum[b]|) * 2^-53

where the last term is the two conversions to double and tap_uv covers a projection that is not bit-identical to the
oracle's (see PROJ_TOL)."""
from __future__ import annotations

import math

import numpy as np

U = 2.0**-53  # unit roundoff of double
EPS_LOG = 1e-6  # the + 1e-6 inside the entropy logs (:92-94)
C6 = np.array([[1.0, -3.0, 3.0, -1.0], [4.0, 0.0, -6.0, 3.0], [1.0, 3.0, 3.0, -3.0], [0.0, 0.0, 0.0, 1.0]])
COEFFS = C6 / 6.0  # :29-33

# Largest |u_gpu - u_oracle| (and the same for v), in pixels, allowed per camera model.  plumb_bob, rational_polynomial
# and omnidir use + - * / and sqrt only: the kernels evaluate them uncontracted in the same order, so their projections
# are the oracle's bits (0).  fisheye (atan2, pow), atan (tan, atan) and equirectangular (asin, atan2) call
# transcendentals: CUDA's are within 2 ulp and glibc's within 1 ulp of the true value, so the two differ by <= 3 ulp per
# call.  Each functor composes at most five such calls, the worst amplification being theta^8 in fisheye (x8), so the
# relative difference of u - c stays below (3 + 8 * 3 + 13) ulp = 40 ulp = 4.4e-15; inliers of these test cameras have
# |u - c|, |v - c| < 2000 px, so |du| < 9e-12 px < 2^-36 px = 1.5e-11 px.
PROJ_TOL = {"plumb_bob": 0.0, "rational_polynomial": 0.0, "omnidir": 0.0, "fisheye": 2.0**-36, "atan": 2.0**-36, "equirectangular": 2.0**-36}
# |d beta_r / d s| <= 2/3 and |beta_r| <= 2/3 on [0, 1), so |d w_ij| <= (4/9) (|du| + |dv|) per tap.  Moving the knot
# across an integer leaves the clamped pixel weights continuous (the spline is C2), so a flip adds nothing beyond this.
TAP_PER_UV = 8.0 / 9.0


def fixed_bits(n: int) -> int:
    """Fraction bits of the kernels' fixed-point tap weights for a cloud of n points: min(40, 62 - ceil(log2 n))."""
    return min(40, 62 - (max(int(n), 1) - 1).bit_length())


def cast_int(x):
    """static_cast<int>(double) as x86-64 cvttsd2si: truncation, NaN / out of range -> INT_MIN."""
    x = np.asarray(x, dtype=np.float64)
    ok = (x > -2147483649.0) & (x < 2147483648.0)
    return np.where(ok, np.trunc(np.where(ok, x, 0.0)), -2147483648.0).astype(np.int64)


def camera_points(points_xyzw, tp):
    """Sophus SE3 action on the (N, 3) lidar points in the reference's operation order (oracle/vlcal_oracle.c :47)."""
    p = np.asarray(points_xyzw, dtype=np.float64)[:, :3]
    qx, qy, qz, qw = (float(v) for v in tp[:4])
    X, Y, Z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(invalid="ignore"):  # Inf coordinates give NaN, as in the reference
        ux, uy, uz = qy * Z - qz * Y, qz * X - qx * Z, qx * Y - qy * X
        ux, uy, uz = ux + ux, uy + uy, uz + uz
        cx, cy, cz = qy * uz - qz * uy, qz * ux - qx * uz, qx * uy - qy * ux
        return np.stack([((X + qw * ux) + cx) + tp[4], ((Y + qw * uy) + cy) + tp[5], ((Z + qw * uz) + cz) + tp[6]], axis=1)


def image_bin_lut(bins):
    pix = np.arange(256, dtype=np.float64) * (1.0 / 255.0)  # convertTo(CV_64FC1, 1.0 / 255.0)
    return np.minimum(cast_int(pix * bins), bins - 1)  # :79, std::min only


def beta(s):
    se = (np.ones_like(s), s, s * s, (s * s) * s)
    return np.stack([((COEFFS[r, 0] * se[0] + COEFFS[r, 1] * se[1]) + COEFFS[r, 2] * se[2]) + COEFFS[r, 3] * se[3] for r in range(4)], axis=-1)


def project(oracle, cam, pc):
    return oracle.project(cam, pc) if pc.shape[0] else np.zeros((0, 2))


def taps(oracle, cam, image, points_xyzw, intensities, bins, tp):
    """The reference's taps at pose tp: (inlier mask, lidar bin per point, joint index per tap, weight per tap, u, v).
    Joint index = image_bin * bins + lidar_bin, i.e. the [image_bin, lidar_bin] layout of NIDCost.evaluate."""
    image = np.ascontiguousarray(image, dtype=np.uint8)
    H, W = image.shape
    ins = np.asarray(intensities, dtype=np.float64)
    uv = project(oracle, cam, camera_points(points_xyzw, tp))
    u, v = uv[:, 0], uv[:, 1]
    bp = np.maximum(0, np.minimum(bins - 1, cast_int(ins * bins)))
    with np.errstate(invalid="ignore"):
        kx, ky = cast_int(np.floor(u)), cast_int(np.floor(v))
    inl = (kx >= 0) & (ky >= 0) & (kx < W) & (ky < H)
    kx, ky, su, sv = kx[inl], ky[inl], u[inl] - kx[inl].astype(np.float64), v[inl] - ky[inl].astype(np.float64)
    bx, by = beta(su), beta(sv)  # (n_in, 4)
    w = (bx[:, :, None] * by[:, None, :]).reshape(-1)  # [i (x), j (y)] as the loop at :75-77
    off = np.arange(-1, 3)
    xs = np.clip(kx[:, None] + off, 0, W - 1)
    ys = np.clip(ky[:, None] + off, 0, H - 1)
    ib = image_bin_lut(bins)[image[ys[:, None, :], xs[:, :, None]]].reshape(-1)
    joint = ib * bins + np.repeat(bp[inl], 16)
    return inl, bp, joint, w, u, v


def _fsum_by(index, values, size):
    out = np.zeros(size)
    if index.size == 0:
        return out
    order = np.argsort(index, kind="stable")
    idx, vals = index[order], values[order]
    starts = np.flatnonzero(np.r_[True, idx[1:] != idx[:-1]])
    ends = np.r_[starts[1:], idx.size]
    for a, b in zip(starts, ends):
        out[idx[a]] = math.fsum(vals[a:b].tolist())
    return out


class Exact:
    """Exact mode-B histograms of one pose.  hist / taps / abs_sum are [image_bin, lidar_bin]."""

    def __init__(self, oracle, cam, image, points_xyzw, intensities, bins, tp):
        inl, bp, joint, w, u, v = taps(oracle, cam, image, points_xyzw, intensities, bins, tp)
        nb = bins * bins
        self.bins = bins
        self.u, self.v, self.inlier = u, v, inl
        self.hist = _fsum_by(joint, w, nb).reshape(bins, bins)
        self.hist_image = _fsum_by(joint // bins, w, bins)  # exact row sums (the reference's hist_image, :81)
        self.taps = np.bincount(joint, minlength=nb).reshape(bins, bins)
        self.taps_image = self.taps.sum(axis=1)
        self.abs_sum = np.bincount(joint, weights=np.abs(w), minlength=nb).reshape(bins, bins)
        self.points = np.bincount(bp[inl], minlength=bins)  # hist_points (:60), exact
        self.n_inliers = int(inl.sum())
        self.Hi, self.Hp, self.Hip, self.nid = entropies(self.hist, self.hist_image, self.points)

    def decision_margin(self, W, H):
        """Distance of the inlier decision (floor(u) in [0, W), floor(v) in [0, H)) from flipping, over all points with a
        finite projection: min over |u|, |u - W|, |v|, |v - H| (the edges where the verdict changes)."""
        u, v = self.u, self.v
        m = np.isfinite(u) & np.isfinite(v)
        if not m.any():
            return np.inf
        d = np.minimum(np.minimum(np.abs(u[m]), np.abs(u[m] - W)), np.minimum(np.abs(v[m]), np.abs(v[m] - H)))
        return float(d.min())


def entropies(hist, hist_image, hist_points):
    """(Hi, Hp, Hip, NID) of :86-96 in np.longdouble."""
    h = np.asarray(hist, dtype=np.longdouble)
    hi = np.asarray(hist_image, dtype=np.longdouble)
    hp = np.asarray(hist_points, dtype=np.longdouble)
    s = hp.sum()
    with np.errstate(invalid="ignore", divide="ignore"):
        f = lambda p: -np.sum(p * np.log(p + np.longdouble(EPS_LOG)))  # noqa: E731
        Hi, Hp, Hip = f(hi / s), f(hp / s), f(h / s)
        MI = Hi + Hp - Hip
        nid = (Hip - MI) / Hip
    return Hi, Hp, Hip, nid


def hist_bound(ex: Exact, hist_gpu, F, proj_tol):
    """Per-bin certified bound |hist_gpu - fsum| (module docstring)."""
    per_tap = 2.0 ** -(F + 1) + TAP_PER_UV * proj_tol
    return ex.taps * per_tap + (np.abs(hist_gpu) + np.abs(ex.hist)) * U


def nid_bound(ex: Exact, F, proj_tol, extra_per_tap=0.0):
    """Certified bound on |NID_gpu - NID_exact| for a kernel whose histogram obeys hist_bound.

    With S inliers, p = h / S.  The kernel's p_b is within e_b = d_b / S + u p_b of the exact one, d_b the bin bound (the
    u p_b is the division).  phi(p) = p ln(p + 1e-6) has |phi'| <= |ln 1e-6| + 1 = L on [0, 1 + 1e-6], so an entropy moves
    by at most L sum_b e_b; evaluating it in double adds at most (n + 4) u sum_b |phi(p_b)| (n terms summed in any order,
    log within 2 ulp).  The lidar marginal is exact, only its evaluation error counts.  NID = 2 - (Hi + Hp) / Hip, so
      |dNID| <= (|dHi| + |dHp|) / h + (|Hi| + |Hp|) |dHip| / (|Hip| h) + 4 u (|NID| + 2),   h = |Hip| - |dHip|."""
    S = float(ex.points.sum())
    if S == 0:
        return np.inf
    L = abs(math.log(EPS_LOG)) + 1.0
    per_tap = 2.0 ** -(F + 1) + TAP_PER_UV * proj_tol + extra_per_tap
    p = ex.hist.reshape(-1) / S
    pi = ex.hist_image / S
    pp = ex.points / S
    d_joint = (ex.taps.reshape(-1) * per_tap + 2 * np.abs(ex.hist.reshape(-1)) * U * (1 + 1e-9)) / S + U * p
    d_image = (ex.taps_image * per_tap + 2 * np.abs(ex.hist_image) * U * (1 + 1e-9)) / S + U * pi
    phi = lambda q: np.abs(q * np.log(q + EPS_LOG))  # noqa: E731
    nb = ex.bins * ex.bins
    dHip = L * d_joint.sum() + (nb + 4) * U * phi(p).sum() * (1 + 1e-6)
    dHi = L * d_image.sum() + (ex.bins + 4) * U * phi(pi).sum() * (1 + 1e-6)
    dHp = (ex.bins + 4) * U * phi(pp).sum() * (1 + 1e-6)
    Hi, Hp, Hip = abs(float(ex.Hi)), abs(float(ex.Hp)), abs(float(ex.Hip))
    h = Hip - dHip
    if h <= 0:
        return np.inf
    return (dHi + dHp) / h + (Hi + Hp) * dHip / (Hip * h) + 4 * U * (abs(float(ex.nid)) + 2.0)


def nid_from_gpu_hist(hist_gpu):
    """The NID formula (:86-96) in np.longdouble on a kernel's own histogram: image marginal = row sums, lidar marginal =
    column sums rounded to the integer inlier counts they are (each point's 16 weights sum to 1)."""
    h = np.asarray(hist_gpu, dtype=np.longdouble)
    points = np.rint(np.asarray(hist_gpu, dtype=np.float64).sum(axis=0))
    return entropies(h, h.sum(axis=1), points)


def nid_rounding_bound(Hi, Hp, Hip, nid, bins):
    """Rounding of the double entropy tail alone (nid_bound with exact histograms): what separates a kernel's NID from
    nid_from_gpu_hist of its own histogram."""
    Hi, Hp, Hip = abs(float(Hi)), abs(float(Hp)), abs(float(Hip))
    L = abs(math.log(EPS_LOG)) + 1.0
    # |phi| summed is the entropy itself up to the sign of the terms with p + 1e-6 > 1 (at most one, |phi| < 1e-6)
    dHip = (bins * bins + 4) * U * (Hip + 1e-6) + L * (bins * bins) * U
    dHi = (bins + 4) * U * (Hi + 1e-6) + L * bins * U
    dHp = (bins + 4) * U * (Hp + 1e-6) + L * bins * U
    h = Hip - dHip
    if not np.isfinite(h) or h <= 0:
        return np.inf
    return (dHi + dHp) / h + (Hi + Hp) * dHip / (Hip * h) + 4 * U * (abs(float(nid)) + 2.0)


# ---------------------------------------------------------------------------------------------------------------------
# inputs that put the reference's decisions on edge (shared by the host and the GPU tests)
# ---------------------------------------------------------------------------------------------------------------------


def sophus_params(T):
    from scipy.spatial.transform import Rotation

    q = Rotation.from_matrix(np.asarray(T)[:3, :3]).as_quat()  # x y z w
    return np.concatenate([q, np.asarray(T)[:3, 3]])


def _inverse_action(tp, pc):
    """Lidar point whose camera point at tp is (approximately) pc, for a unit quaternion."""
    from scipy.spatial.transform import Rotation

    R = Rotation.from_quat(tp[:4]).as_matrix()
    return (pc - tp[4:]) @ R


def place_points(oracle, cam, tp, targets, depth, iters=8):
    """Lidar points whose reference projection at pose tp lands on targets (M, 2) in pixels.  Seed: the nearest of a
    0.5-degree grid of camera-frame directions, by its oracle projection; then Newton steps on the full pipeline
    (camera_points + oracle.project) along the two tangents of the seed direction, with a finite-difference Jacobian and
    steps capped at 5 % of the depth.  Returns (points (M, 3), achieved uv (M, 2)); unreachable targets (beyond the
    equirectangular seam or a pole) end wherever the steps leave them."""
    from scipy.spatial import cKDTree
    from scipy.spatial.transform import Rotation

    targets = np.asarray(targets, dtype=np.float64)
    M = targets.shape[0]
    th, ph = np.meshgrid(np.radians(np.arange(0.5, 180.0, 0.5)), np.radians(np.arange(-180.0, 180.0, 0.5)), indexing="ij")
    grid = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], axis=-1).reshape(-1, 3)
    guv = project(oracle, cam, grid)
    fin = np.isfinite(guv).all(axis=1)
    grid, guv = grid[fin], guv[fin]
    d0 = grid[cKDTree(guv).query(targets)[1]]
    e1 = np.cross(d0, np.eye(3)[np.argmin(np.abs(d0), axis=1)])  # tangent from the axis least aligned with d0
    e1 /= np.linalg.norm(e1, axis=1, keepdims=True)
    e2 = np.cross(d0, e1)
    R = Rotation.from_quat(tp[:4]).as_matrix()
    ab = np.zeros((M, 2))

    def lidar(ab_):
        pc = depth[:, None] * (d0 + ab_[:, :1] * e1 + ab_[:, 1:] * e2)
        return (pc - tp[4:]) @ R

    def uv_of(ab_):
        return project(oracle, cam, camera_points(np.c_[lidar(ab_), np.ones(M)], tp))

    for _ in range(iters):
        uv = uv_of(ab)
        h = 1e-7
        J = np.empty((M, 2, 2))
        for k in range(2):
            d = np.zeros((M, 2))
            d[:, k] = h
            J[:, :, k] = (uv_of(ab + d) - uv) / h
        r = targets - uv
        ok = np.isfinite(r).all(axis=1) & np.isfinite(J).all(axis=(1, 2)) & (np.abs(np.linalg.det(J)) > 1e-30)
        step = np.zeros((M, 2))
        step[ok] = np.linalg.solve(J[ok], r[ok][:, :, None])[:, :, 0]
        n = np.linalg.norm(step, axis=1, keepdims=True)
        step *= np.minimum(1.0, 0.05 / np.maximum(n, 1e-300))
        r0 = np.where(np.isfinite(r), np.abs(r), np.inf).max(axis=1)
        for _ in range(30):  # halve the steps that do not reduce the residual (the seam, the poles)
            r1 = np.abs(targets - uv_of(ab + step)).max(axis=1)
            worse = ~(r1 <= r0)
            if not worse.any():
                break
            step[worse] *= 0.5
        ab += np.where((r1 <= r0)[:, None], step, 0.0)
    return lidar(ab), uv_of(ab)


def edge_targets(W, H, rng, offsets=(1e-3, 1e-5, 1e-7, 1e-9)):
    """Pixel targets within the given offsets of the decision edges u = 0, -1, W, v = 0, -1, H, of interior integers (the
    knot flip of floor), plus footprints clamped at the four corners; the other coordinate is random inside."""
    out = []
    interior_u = [1.0, float(W // 2), float(max(W - 1, 1))]
    interior_v = [1.0, float(H // 2), float(max(H - 1, 1))]
    for d in offsets:
        for sgn in (-1.0, 1.0):
            for e in [0.0, -1.0, float(W)] + interior_u:
                out.append((e + sgn * d, rng.uniform(0.0, H)))
            for e in [0.0, -1.0, float(H)] + interior_v:
                out.append((rng.uniform(0.0, W), e + sgn * d))
            for cu in (0.0, float(W)):
                for cv in (0.0, float(H)):
                    out.append((cu + sgn * d, cv + sgn * d))
    for cu in (0.0, W - 1.0):  # footprints clamped at each corner (knot at the first / last column and row)
        for cv in (0.0, H - 1.0):
            for _ in range(4):
                out.append((cu + rng.uniform(0.0, 1.0), cv + rng.uniform(0.0, 1.0)))
    return np.array(out)


def edge_problem(oracle, model, size=None, seed=0, f32=False):
    """A cloud whose projections at the problem's pose sit on the decision edges and clamp the footprint (edge_targets),
    mixed with random points, for the camera of util.CAMERAS[model]; size=(W, H) overrides the image (tiny images)."""
    import util

    intr, dist, (W, H) = util.CAMERAS[model]
    if size is not None:
        W, H = size
        if model == "equirectangular":
            intr = [float(W), float(H)]  # its intrinsics are the image size: the tiny image still spans the sphere
    rng = np.random.default_rng(seed)
    cam = oracle.create_camera(model, intr, dist)
    T = util.S.gt_T_camera_lidar()
    tp = sophus_params(T)
    targets = edge_targets(W, H, rng)
    # tiny images are the pixels around (0, 0) of the full camera's frame
    depth = rng.uniform(1.0, 20.0, targets.shape[0])
    pts, uv = place_points(oracle, cam, tp, targets, depth)
    # some targets cannot be reached (u < 0 or u > W across the equirectangular seam, v beyond a pole): keep the points,
    # except any that ended within 1e-10 px of a verdict edge, closer than the GPU/oracle projection tolerance allows
    m = np.minimum(np.minimum(np.abs(uv[:, 0]), np.abs(uv[:, 0] - W)), np.minimum(np.abs(uv[:, 1]), np.abs(uv[:, 1] - H)))
    pts = pts[~(m < 1e-10)]
    base = util.random_problem(model, n=4000, seed=seed, size=(W, H))
    base["intrinsics"] = intr
    pts = np.concatenate([pts, base["points"][:, :3]])
    if f32:
        pts = pts.astype(np.float32).astype(np.float64)
        inten = rng.integers(0, 256, pts.shape[0]) / 256.0
    else:
        inten = rng.uniform(0.0, 1.0, pts.shape[0])
    image = rng.integers(0, 256, (H, W), dtype=np.uint8)
    return {"model": model, "intrinsics": intr, "distortion": dist, "W": W, "H": H, "image": image, "points": np.c_[pts, np.ones(pts.shape[0])], "intensities": inten, "tp": tp}


def invalid_problem(model, seed=0):
    """NaN / +-Inf coordinates, a point at the camera centre of the identity pose, intensities outside [0, 1) and NaN,
    among ordinary points.  Evaluate it at the problem's pose and at the identity pose [0 0 0 1 0 0 0]."""
    import util

    pr = util.random_problem(model, n=3000, seed=seed, f32=False)
    pts = pr["points"].copy()
    inten = pr["intensities"].copy()
    bad = np.array([[np.nan, 1.0, 5.0], [1.0, np.nan, 5.0], [1.0, 1.0, np.nan], [np.inf, 0.0, 5.0], [-np.inf, 0.0, 5.0],
                    [0.0, np.inf, 5.0], [0.0, 0.0, np.inf], [0.0, 0.0, -np.inf], [0.0, 0.0, 0.0], [np.inf, np.inf, np.inf]])
    n_bad = bad.shape[0]
    pts[:n_bad, :3] = bad
    vals = np.array([-0.5, 1.0, 1.7, np.nan])
    inten[n_bad : n_bad + 40] = np.tile(vals, 10)  # on ordinary points: these reach the histogram
    inten[:n_bad] = np.resize(vals, n_bad)
    pr.update(points=pts, intensities=inten)
    pr["tps"] = np.stack([sophus_params(pr["T"]), np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])])
    return pr
