"""GPU edge suite of view culling (K4, csrc/view_cull.cu), held to oracle.view_cull: the per-pixel minimum of the
float-rounded ranges, the keep rule !(range > double(float cell) + 0.1), the FoV test on the normalised 4-vector, the
truncation and bounds tests, the block scan and both compactions.

Bar: on the public path (vlcal_view_cull) the index list identical to the oracle's; on the internal paths (the
tile-ordered counting sort the solver's cost objects score, and the keep_all reorder behind reorder_for_pose), read back
through vlcal_debug_view_cull_points, exactly the oracle's points as a multiset, grouped by 32 x 8-pixel tile."""
import math

import numpy as np
import pytest

import util
from test_gpu_persistent_edges import DYADIC_PINHOLE, _special_points

pytestmark = pytest.mark.gpu
FLT_MAX = float(np.finfo(np.float32).max)
PINHOLE = ("plumb_bob", [500.0, 500.0, 320.0, 240.0], [], 640, 480)  # distortion-free: the optical axis is pixel (320, 240)
DYADIC = ("plumb_bob", DYADIC_PINHOLE[0], DYADIC_PINHOLE[1], 640, 480)  # u = 512 x / z + 320 exact for dyadic x, z
EQUI = ("equirectangular", util.CAMERAS["equirectangular"][0], [], 640, 320)
CULL_THREADS = 256


def _spec(model, size=None):
    intr, dist, (W, H) = util.CAMERAS[model]
    if size is not None:
        W, H = size
    return model, intr, dist, W, H


def _xyzw(p):
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    return np.concatenate([p, np.ones((p.shape[0], 1))], axis=1)


def _oracle(O, spec, pts, T, depth, fov=None):
    model, intr, dist, W, H = spec
    ocam = O.create_camera(model, intr, dist)
    if fov is None:
        fov = O.estimate_camera_fov(ocam, W, H)
    return O.view_cull(ocam, W, H, fov, depth, pts, T)


def _culling(V, spec, depth):
    model, intr, dist, W, H = spec
    return V.ViewCulling(V.create_camera(model, intr, dist), (W, H), V.ViewCullingParams(depth))


def _pixels(O, spec, pts, T, ids):
    """The oracle's pixel (ix, iy) of points ids at T: pt_camera = ((T0 x + T1 y) + T2 z) + T3, projected, truncated."""
    model, intr, dist, W, H = spec
    p = pts[ids]
    pc = np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], axis=1)
    uv = O.project(O.create_camera(model, intr, dist), pc).reshape(-1, 2)
    ix, iy = np.trunc(uv[:, 0]).astype(np.int64), np.trunc(uv[:, 1]).astype(np.int64)
    assert np.all((ix >= 0) & (ix < W) & (iy >= 0) & (iy < H))
    return ix, iy


def check_cull(V, O, spec, pts, T, depth, fov=None, internal=True):
    """Public path == oracle; tile path and keep_all reorder == oracle as multisets, grouped by tile.  Returns the
    oracle's kept indices."""
    model, intr, dist, W, H = spec
    pts = np.ascontiguousarray(pts)
    n = pts.shape[0]
    ref = _oracle(O, spec, pts, T, depth, fov)
    vc = _culling(V, spec, depth)
    idx = vc.cull_indices(pts, T, max_fov=fov)
    assert np.array_equal(idx, ref), (len(idx), len(ref), np.setxor1d(idx, ref)[:10])
    if not internal:
        return ref
    with np.errstate(over="ignore"):
        f32 = bool(np.all((pts[:, :3].astype(np.float32).astype(np.float64) == pts[:, :3]) | np.isnan(pts[:, :3])))
    ids_value = np.arange(n, dtype=np.float64)  # carried in the intensity slot (exact in float32 below 2^24 points)
    tiles_x = (W + 31) // 32
    n_tiles = tiles_x * ((H + 7) // 8) + 1
    in_view = _oracle(O, spec, pts, T, False, fov)
    for keep_all in (False, True):
        rows, on_f32 = vc.debug_culled_points(pts, ids_value, T, max_fov=fov, keep_all=keep_all)
        assert on_f32 == f32
        ids = rows[:, 3].astype(np.int64)
        want = np.arange(n) if keep_all else ref
        assert np.array_equal(np.sort(ids), want), (keep_all, len(ids), len(want))
        assert np.array_equal(rows[:, :3], pts[ids, :3], equal_nan=True)
        tile = np.full(len(ids), n_tiles - 1)
        seen = np.isin(ids, in_view) if keep_all else np.ones(len(ids), bool)
        ix, iy = _pixels(O, spec, pts, T, ids[seen])
        tile[seen] = (iy >> 3) * tiles_x + (ix >> 5)
        assert np.all(np.diff(tile) >= 0), "not grouped by tile"
        rx, ry = _pixels(O, spec, pts, T, in_view if keep_all else ref)
        want_counts = np.bincount((ry >> 3) * tiles_x + (rx >> 5), minlength=n_tiles)
        if keep_all:
            want_counts[n_tiles - 1] = n - len(in_view)  # out of view: last
        assert np.array_equal(np.bincount(tile, minlength=n_tiles), want_counts)
    return ref


# ---- 1. the keep threshold ---------------------------------------------------------------------------------------------


def _axis(z):
    return _xyzw(np.stack([np.zeros(len(z)), np.zeros(len(z)), np.asarray(z, dtype=np.float64)], axis=1))


@pytest.mark.parametrize("z0", [10.3, 7.0 + 0.75 * 2.0**-21, 2.0 + 0.25 * 2.0**-22, 123.456])
def test_keep_threshold_in_the_double_layout(gpu, oracle, z0):
    """Ranges exactly double(float(min)) + 0.1 and one double ulp either side, on the optical axis (range = z exactly);
    z0 rounds up to its float in two of the cases, so that a cell rounded toward zero would move the threshold."""
    cell = float(np.float32(z0))
    t = cell + 0.1
    z = [z0, t, np.nextafter(t, 0.0), np.nextafter(t, 1e9), t + 1e-6, z0 + 1e-12, np.nextafter(z0, 1e9)]
    pts = _axis(z)
    for depth in (True, False):
        ref = check_cull(gpu, oracle, PINHOLE, pts, np.eye(4), depth)
        assert list(ref) == ([0, 1, 2, 5, 6] if depth else list(range(7))), ref
    # several pixels, each with its own minimum: the threshold cases repeated at 64 points of a row
    rng = np.random.default_rng(2000)
    rows = []
    for k in range(64):
        zk = z0 * (1.0 + rng.uniform(0, 0.5))
        tk = float(np.float32(zk)) + 0.1
        u = 100 + 7 * k + 0.5
        for zz in (zk, tk, np.nextafter(tk, 0.0), np.nextafter(tk, 1e9)):
            rows.append([(u - 320.0) / 512.0 * zz, 0.5 / 512.0 * zz, zz])
    pts = _xyzw(np.array(rows))
    check_cull(gpu, oracle, DYADIC, pts, np.eye(4), True)


@pytest.mark.parametrize("z0", [10.3, 7.0, 2.0 + 3 * 2.0**-22])
def test_keep_threshold_in_the_float4_layout(gpu, oracle, z0):
    """float4 layout: the nearest float ranges below and above double(float(min)) + 0.1, and points on one pixel whose
    ranges round to the same float."""
    f = np.float32
    cell = f(z0)
    t = float(cell) + 0.1
    below = f(t) if float(f(t)) <= t else np.nextafter(f(t), f(0))
    above = np.nextafter(below, f(1e9))
    assert float(below) <= t < float(above)
    z = np.array([cell, below, above, np.nextafter(below, f(0)), cell, np.nextafter(cell, f(1e9))], dtype=f).astype(np.float64)
    pts = _axis(z)
    for depth in (True, False):
        ref = check_cull(gpu, oracle, PINHOLE, pts, np.eye(4), depth)
        assert list(ref) == ([0, 1, 3, 4, 5] if depth else list(range(6))), ref


# ---- 2. rounding of the ranges ----------------------------------------------------------------------------------------------


def test_ranges_around_flt_max_and_infinite(gpu, oracle):
    """Ranges that round to FLT_MAX, to +inf (ties with the +inf initial cell), and an infinite range (z ~ 1e200, z^2
    overflows; max_fov 2.0 so that the 4-vector FoV test, nz = 0, passes)."""
    half_ulp = 2.0**103
    sets = [
        [FLT_MAX, FLT_MAX + 0.5 * half_ulp, FLT_MAX + half_ulp, FLT_MAX * 1.5],  # min FLT_MAX: the rest within + 0.1 or not
        [FLT_MAX + half_ulp, FLT_MAX * 2.0, FLT_MAX + 0.99 * half_ulp],          # rounds to +inf; one that rounds to FLT_MAX
        [FLT_MAX * 1.5, 1e200, 1e300],                                           # every cell +inf
        [1e200, 1e200 * (1 + 2**-50), 1e30],
    ]
    for zs in sets:
        pts = _axis(zs)
        for depth in (True, False):
            ref = check_cull(gpu, oracle, PINHOLE, pts, np.eye(4), depth, fov=2.0)
            if not depth:
                assert len(ref) == len(zs)
    # off the axis: the pinhole's u = fx x / z + cx stays finite at 1e200
    pts = _xyzw([[0.5e200, 0.0, 1e200], [-0.5e200, 0.4e200, 1e200], [0.0, 1e199, 1e200], [0.25e200, -0.25e200, 1e200]])
    for depth in (True, False):
        assert len(check_cull(gpu, oracle, PINHOLE, pts, np.eye(4), depth, fov=2.0)) == 4


def test_zero_range_at_the_camera_centre_equirectangular(gpu, oracle):
    """The camera centre projects (equirectangular) to the pixel of the +z axis with range 0: its cell is 0 and the
    axis points at ranges 0.05 and 0.1 are kept, the one a double ulp beyond 0.1 is not."""
    z = [0.0, 0.05, 0.1, np.nextafter(0.1, 1.0), 0.2, 0.1 + 2.0**-40]
    pts = _axis(z)
    ref = check_cull(gpu, oracle, EQUI, pts, np.eye(4), True)
    assert list(ref) == [0, 1, 2]
    check_cull(gpu, oracle, EQUI, pts, np.eye(4), False)


# ---- 3. the FoV cone ---------------------------------------------------------------------------------------------------------


def _bisect_edge(inside, lo, hi):
    """(a, b) adjacent values with inside(a) != inside(b), lo and hi on opposite sides; floats of any dtype."""
    assert inside(lo) != inside(hi)
    while True:
        mid = lo + (hi - lo) / 2
        if mid == lo or mid == hi:
            return lo, hi
        if inside(mid) == inside(lo):
            lo = mid
        else:
            hi = mid


def _cone_points(O, spec, fov, direction, r, dtype):
    """Points r (cos a direction_xy, sin a ...) straddling the FoV decision, found by bisection on the oracle (depth off):
    the last angle kept and the first one culled, in doubles or in float32 coordinates."""
    dx, dy = direction
    def pt(a):
        a = float(a)
        p = np.array([[math.sin(a) * dx * r, math.sin(a) * dy * r, math.cos(a) * r]]).astype(dtype).astype(np.float64)
        return p
    inside = lambda a: len(_oracle(O, spec, _xyzw(pt(a)), np.eye(4), False, fov)) == 1
    lo, hi = _bisect_edge(inside, 0.01, 3.0)
    # adjacent angles: the two points differ by at most one ulp (of double or float32) in each coordinate
    assert inside(lo) and not inside(hi)
    return np.concatenate([pt(lo), pt(hi)])


@pytest.mark.parametrize("case", ["given", "estimated", "above_half_pi"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_fov_cone_edge_found_by_bisection(gpu, oracle, case, dtype):
    if case == "given":
        spec, fov, direction = PINHOLE, 0.4, (1.0, 0.0)
    elif case == "estimated":  # towards the corner pixel (0, 0), where the estimated FoV comes from
        spec, fov, direction = PINHOLE, None, (-0.8, -0.6)
    else:
        spec, fov, direction = EQUI, 2.0, (0.6, 0.8)
    rows = []
    for r in ((0.5, 3.0, 10.0, 40.0) if spec is EQUI else (3.0, 10.0, 25.0)):  # the pinhole's cone edge stays inside the image
        rows.append(_cone_points(oracle, spec, fov, direction, r, dtype))
    pts = _xyzw(np.concatenate(rows))
    ocam = oracle.create_camera(*spec[:3])
    min_z = math.cos(fov if fov is not None else oracle.estimate_camera_fov(ocam, spec[3], spec[4]))
    assert (min_z < 0) == (case == "above_half_pi")
    # the decision is the FoV test itself: the normalised 4-vector's z straddles cos(max_fov)
    nz = pts[:, 2] / np.sqrt((pts[:, 0] ** 2 + pts[:, 1] ** 2) + (pts[:, 2] ** 2 + 1.0))
    assert np.all(nz[0::2] >= min_z - 1e-15) and np.all(nz[1::2] < min_z + 1e-15), (nz - min_z)
    for depth in (False, True):
        ref = check_cull(gpu, oracle, spec, pts, np.eye(4), depth, fov)
        if not depth:
            assert list(ref) == list(range(0, len(pts), 2))


# ---- 4. truncation and bounds ------------------------------------------------------------------------------------------------


def _truncation_points(W, H, f32):
    s = 2.0**-20
    rows = []
    for z in (16.0, 32.0, 64.0):  # far enough for the 4-vector FoV test to pass up to the image border
        us = [-1.0, np.nextafter(-1.0, 0.0), -1.0 + s, -0.5, -s, -1e-300, 0.0, 0.5, W - 1 + (1 - s), np.nextafter(float(W), 0.0), float(W), W + s]
        for k in (1, 17, 319, 320, 321, W - 1):
            us += [k - 1e-9, float(k), k + 1e-9]
        for u in us:
            rows.append([(u - 320.0) / 512.0 * z, 0.5 / 512.0 * z, z])
        vs = [-1.0, np.nextafter(-1.0, 0.0), -0.5, -s, 0.0, H - 1 + (1 - 1e-7), H - 1 + (1 - s), np.nextafter(float(H), 0.0), float(H)]
        for k in (1, 8, 239, 240, H - 1):
            vs += [k - 1e-9, float(k), k + 1e-9]
        for v in vs:
            rows.append([0.5 / 512.0 * z, (v - 240.0) / 512.0 * z, z])
    pts = np.array(rows)
    if f32:
        pts = pts.astype(np.float32).astype(np.float64)
    nan, inf = math.nan, math.inf
    special = [[nan, 0, 1], [0, nan, 1], [0, 0, nan], [inf, 0, 1], [-inf, 0, 1], [0, inf, 1], [0, -inf, 1], [0, 0, inf], [0, 0, -inf],
               [inf, inf, inf], [nan, nan, nan]]
    return np.concatenate([pts, np.array(special, dtype=np.float64)])


@pytest.mark.parametrize("f32", [False, True])
def test_truncation_and_bounds(gpu, oracle, f32):
    W, H = DYADIC[3], DYADIC[4]
    pts = _xyzw(_truncation_points(W, H, f32))
    for depth in (False, True):
        ref = check_cull(gpu, oracle, DYADIC, pts, np.eye(4), depth)
        assert len(ref) > 30
    # the same rows and columns from the reference's exact values: u in (-1, 0) kept (column 0), -1 and W not
    ocam = oracle.create_camera(*DYADIC[:3])
    kept = set(_oracle(oracle, DYADIC, pts, np.eye(4), False).tolist())
    uv = oracle.project(ocam, pts[:, :3])
    with np.errstate(invalid="ignore"):
        strip = (uv[:, 0] > -1.0) & (uv[:, 0] < 0.0) & (uv[:, 1] >= 0) & (uv[:, 1] < H)
        at_w = uv[:, 0] == float(W)
    assert strip.sum() >= 3 and all(i in kept for i in np.flatnonzero(strip))
    assert at_w.sum() >= 3 and not any(i in kept for i in np.flatnonzero(at_w))


@pytest.mark.parametrize("model", util.MODELS)
def test_special_values_among_random_points_all_models(gpu, oracle, model):
    pr = util.random_problem(model, n=20_000, seed=2100)
    spec = _spec(model)
    sp = _xyzw(_truncation_points(spec[3], spec[4], True))
    pts = pr["points"].copy()
    pts[7_001 : 7_001 + sp.shape[0]] = sp
    for depth in (False, True):
        check_cull(gpu, oracle, spec, pts, np.eye(4), depth)
        check_cull(gpu, oracle, spec, pts, pr["T"], depth)
    pts64 = util.random_problem(model, n=20_000, seed=2101, f32=False)["points"]
    pts64[9_001 : 9_001 + sp.shape[0]] = sp
    for depth in (False, True):
        check_cull(gpu, oracle, spec, pts64, pr["T"], depth)


# ---- 5. sizes -------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 1024 * CULL_THREADS - 1, 1024 * CULL_THREADS, 1024 * CULL_THREADS + 1, 1_000_000])
def test_sizes_around_the_scan_chunk(gpu, oracle, n):
    """N = 1024 x 256 +- 1 puts the block count at the single-block scan's chunk edge (1024 entries)."""
    model = "plumb_bob" if n % 2 else "fisheye"
    pr = util.random_problem(model, n=max(n, 16), seed=2200 + n % 1000)
    pts = pr["points"][:n]
    for depth in (True, False):
        ref = check_cull(gpu, oracle, _spec(model), pts, pr["T"], depth)
        if n > 1000:
            assert len(ref) > 0.2 * n


def test_five_million_points_both_layouts(gpu, oracle):
    pr = util.random_problem("rational_polynomial", n=5_000_000, seed=2300)
    spec = _spec("rational_polynomial")
    ref = check_cull(gpu, oracle, spec, pr["points"], pr["T"], True, internal=False)
    assert len(ref) > 100_000
    pts = pr["points"].copy()
    pts[::3, :3] += 1e-9  # double layout
    check_cull(gpu, oracle, spec, pts, pr["T"], True, internal=False)


@pytest.mark.parametrize("n", [1, 300, 1024 * CULL_THREADS + 1])
def test_every_point_or_no_point_survives(gpu, oracle, n):
    """All points on distinct pixels in front of the camera (depth culling keeps every one), or all behind it (kept = 0,
    no scatter)."""
    rng = np.random.default_rng(2400)
    W, H = DYADIC[3], DYADIC[4]
    pix = rng.choice(W * H, size=n, replace=False)
    assert n <= W * H
    z = np.full(n, 2.0)
    u, v = pix % W + 0.5, pix // W + 0.5
    front = np.stack([(u - 320.0) / 512.0 * z, (v - 240.0) / 512.0 * z, z], axis=1)
    for depth in (True, False):
        ref = check_cull(gpu, oracle, DYADIC, _xyzw(front), np.eye(4), depth, fov=1.2)  # the whole image inside the FoV
        assert len(ref) == n
        ref = check_cull(gpu, oracle, DYADIC, _xyzw(front * [1.0, 1.0, -1.0]), np.eye(4), depth, fov=1.2)
        assert len(ref) == 0


# ---- 6. the internal orders ----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("model,size", [("plumb_bob", (637, 479)), ("omnidir", (641, 483)), ("atan", (100, 9)), ("equirectangular", (1920, 960))])
def test_tile_order_and_keep_all_permutation(gpu, oracle, model, size):
    """Image sizes that are not multiples of 32 x 8 (partial tiles on the right and bottom), and a 1920 x 960
    equirectangular camera: 60 x 120 tiles + 1 = 7201 buckets, so the tile path's scan runs over eight 1024-entry chunks."""
    intr, dist, (W0, H0) = util.CAMERAS[model]
    W, H = size
    if model == "equirectangular":
        intr = [float(W), float(H)]
    else:  # the same field of view on the other image size
        intr = list(intr)
        intr[0], intr[1], intr[2], intr[3] = intr[0] * W / W0, intr[1] * H / H0, W / 2.0, H / 2.0
    spec = (model, intr, dist, W, H)
    n = 300_000 if model == "equirectangular" else 60_000
    pr = util.random_problem(model, n=n, seed=2500)
    for depth in (True, False):
        ref = check_cull(gpu, oracle, spec, pr["points"], pr["T"], depth)
        assert len(ref) > (0 if depth else 0.1 * n)
    if model == "equirectangular":
        assert ((W + 31) // 32) * ((H + 7) // 8) + 1 == 7201
