"""GPU edge suite of generate_lidar_image (K5, csrc/lidar_image.cu), held to oracle.generate_lidar_image: per pixel the
point with the smallest squared range (x^2 + y^2) + z^2 wins, of equal ones the last; a pixel keeps DBL_MAX until a point
beats it with `stored < sq` false, so a squared range of exactly DBL_MAX is written and +inf never is.

Bar: the index map identical to the oracle's, the intensity image bit-identical (compared as uint64), except a NaN
intensity in the float4 layout, where only NaN-ness is compared (float(NaN) may change the payload).  Every case runs in
both layouts the upload chooses from (float32-representable points with float-exact intensities -> float4, otherwise
double4), and checks the layout through vlcal_debug_view_cull_points, which uploads with the same rule."""
import ctypes as C

import numpy as np
import pytest

import util
from test_gpu_persistent_edges import DYADIC_PINHOLE, _special_points

pytestmark = pytest.mark.gpu
DBL_MAX = float(np.finfo(np.float64).max)
PIN = ("plumb_bob", DYADIC_PINHOLE[0], DYADIC_PINHOLE[1], 640, 480)  # identity pose: u = 512 x / z + 320, exact for dyadic points
EQUI = ("equirectangular", [640.0, 320.0], [], 640, 320)  # FoV pi: points at range +inf reach the range compare


def _xyzw(p):
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    return np.concatenate([p, np.ones((p.shape[0], 1))], axis=1)


def _is_f32(pts, inten):
    with np.errstate(over="ignore", invalid="ignore"):
        v = np.concatenate([pts[:, :3].reshape(-1), inten])
        return bool(np.all((v.astype(np.float32).astype(np.float64) == v) | np.isnan(v)))


def _double_layout(inten):
    """The same values with every finite intensity moved off float32 (1e-9 is not a float), so that the upload takes the
    double layout with the points unchanged."""
    out = np.array(inten, dtype=np.float64)
    fin = np.isfinite(out)
    out[fin] += 1e-9
    return out


def check(V, O, spec, pts, inten, T=None, layout=None):
    """generate_lidar_image == oracle; `layout` "f32" / "f64" asserts which layout the cloud took.  Returns the oracle's
    index map."""
    model, intr, dist, W, H = spec
    T = np.eye(4) if T is None else T
    pts = np.ascontiguousarray(pts, dtype=np.float64)
    inten = np.ascontiguousarray(inten, dtype=np.float64)
    cam = V.create_camera(model, intr, dist)
    img, idx = V.generate_lidar_image(cam, (W, H), T, pts, inten)
    ref_img, ref_idx = O.generate_lidar_image(O.create_camera(model, intr, dist), W, H, T, pts, inten)
    bad = idx != ref_idx
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5], idx[bad][:5], ref_idx[bad][:5])
    f32 = _is_f32(pts, inten)
    if layout is not None:
        assert f32 == (layout == "f32")
        if pts.shape[0] > 0:  # the upload rule as the library reports it (large clouds: on a prefix, against the same rule)
            sub = slice(0, min(len(pts), 1 << 16))
            _, on_f32 = V.ViewCulling(cam, (W, H)).debug_culled_points(pts[sub], inten[sub], T, keep_all=True)
            assert on_f32 == (f32 if len(pts) <= 1 << 16 else _is_f32(pts[sub], inten[sub]))
    nan = np.isnan(ref_img)
    assert np.array_equal(np.isnan(img), nan)
    if f32:
        assert np.array_equal(img[~nan].view(np.uint64), ref_img[~nan].view(np.uint64))
    else:
        assert np.array_equal(img.view(np.uint64), ref_img.view(np.uint64))
    return ref_idx


def check_both(V, O, spec, pts, inten_f32, T=None):
    """The case in the float4 layout (inten_f32 float-exact, points float32-representable) and in the double layout."""
    a = check(V, O, spec, pts, inten_f32, T, layout="f32")
    b = check(V, O, spec, pts, _double_layout(inten_f32), T, layout="f64")
    assert np.array_equal(a, b)
    return a


def _at_pixel(ix, iy, z, du=0.5, dv=0.5):
    """Points of PIN at pixel (ix + du, iy + dv), range z (dyadic du, dv, z: exact)."""
    z = np.asarray(z, dtype=np.float64)
    return np.stack([(ix + du - 320.0) / 512.0 * z, (iy + dv - 240.0) / 512.0 * z, z], axis=-1)


def _sq(p):
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    return (p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]


def _ramp(n):
    return (np.arange(n) % (1 << 20)) / float(1 << 20)  # distinct below 2^20 points, float-exact


# ---- 1. ties -------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("k", [2, 33, 1024, 1_000_000])
def test_copies_of_one_point(gpu, oracle, k):
    """k copies of one point with distinct intensities, shuffled among points of other pixels: the largest index wins."""
    rng = np.random.default_rng(k)
    ix, iy = rng.integers(0, 640, 3000), rng.integers(0, 480, 3000)
    keep = (ix != 100) | (iy != 200)
    other = _at_pixel(ix[keep], iy[keep], rng.choice([1.0, 2.0, 4.0, 8.0], int(keep.sum())))
    pts = np.concatenate([other, np.repeat(_at_pixel(100, 200, 4.0)[None], k, axis=0)])
    order = rng.permutation(len(pts))
    ref = check_both(gpu, oracle, PIN, _xyzw(pts[order]), _ramp(len(pts)))
    assert ref[200, 100] == int(np.nonzero(order >= len(other))[0].max())


def _diagonal(k, z, swap=False):
    """(a, b, z) with a = (k + 1/4) z / 512, b = a + z / 4096, or (b, a, z): both land in pixel (320 + k, 240 + k) of PIN,
    and their squared ranges (a^2 + b^2) + z^2 and (b^2 + a^2) + z^2 are equal bit for bit."""
    a = (k + 0.25) / 512.0 * z
    b = (k + 0.375) / 512.0 * z
    return np.array([b, a, z] if swap else [a, b, z])


def test_distinct_points_with_bit_equal_ranges(gpu, oracle):
    """(a, b, z) and (b, a, z) in one pixel, in either order, two to five at a time: the last one wins."""
    rng = np.random.default_rng(7)
    rows, last = [], {}
    for k in range(-230, 230):
        z = float(rng.choice([0.5, 2.0, 4.0, 8.0]))
        group = [bool(x) for x in rng.integers(0, 2, rng.integers(2, 6))]
        group[0], group[1] = False, True  # at least one of each
        rng.shuffle(group)
        for sw in group:
            rows.append(_diagonal(k, z, sw))
        last[k] = len(rows) - 1
    pts = np.array(rows)
    ref = check_both(gpu, oracle, PIN, _xyzw(pts), _ramp(len(pts)))
    for k, j in last.items():
        assert ref[240 + k, 320 + k] == j
    assert _sq(_diagonal(3, 4.0))[0] == _sq(_diagonal(3, 4.0, True))[0]


@pytest.mark.parametrize("k", range(-3, 5))
def test_ranges_one_ulp_apart(gpu, oracle, k):
    """(0, 0, z) and (2^(k-26), 0, z) for z = 2^k, squared ranges z^2 and nextafter(z^2), in pixel (320, 240) among points
    of other pixels: the nearer wins whatever the order."""
    z, x = 2.0**k, 2.0**(k - 26)
    assert (x * x + 0.0 * 0.0) + z * z == np.nextafter(z * z, np.inf)
    rng = np.random.default_rng(40 + k)
    other = _at_pixel(rng.integers(0, 300, 500), rng.integers(0, 480, 500), rng.choice([1.0, 2.0], 500))
    for near_first in (True, False):
        pair = [[0.0, 0.0, z], [x, 0.0, z]] if near_first else [[x, 0.0, z], [0.0, 0.0, z]]
        pts = np.concatenate([other[:250], pair, other[250:]])
        ref = check_both(gpu, oracle, PIN, _xyzw(pts), _ramp(len(pts)))
        assert ref[240, 320] == (250 if near_first else 251)


def test_a_pixel_of_ties_interleaved_with_nearer_points(gpu, oracle):
    """Per diagonal pixel a run of tied points at range z (copies and (a, b) / (b, a) swaps) interleaved with nearer points
    at z / 2 arriving before, between and after them, and farther ones at 2 z; without nearer points the last tie wins."""
    rng = np.random.default_rng(11)
    rows, want = [], {}
    for k in range(-230, 230):
        z = float(rng.choice([2.0, 4.0, 8.0]))
        kinds = list(rng.choice(["tie", "swap", "far"], rng.integers(3, 30)))
        if k % 2 == 0:  # nearer points: first, somewhere between, last or all three
            where = rng.integers(0, 4)
            spots = {0: [0], 1: [len(kinds) // 2], 2: [len(kinds)], 3: [0, len(kinds) // 2, len(kinds)]}[int(where)]
            for s in sorted(spots, reverse=True):
                kinds.insert(s, "near")
        w = None
        for kind in kinds:
            zz = {"tie": z, "swap": z, "far": 2 * z, "near": z / 2}[kind]
            rows.append(_diagonal(k, zz, kind == "swap"))
            if kind == "near" or (kind in ("tie", "swap") and "near" not in kinds):
                w = len(rows) - 1
        want[k] = w
    pts = np.array(rows)
    ref = check_both(gpu, oracle, PIN, _xyzw(pts), _ramp(len(pts)))
    for k, w in want.items():
        if w is not None:
            assert ref[240 + k, 320 + k] == w


# ---- 2. range extremes (double layout) ---------------------------------------------------------------------------------


def _dbl_max_point():
    """(x, 0, z) with z*z one ulp below DBL_MAX and (x*x + 0) + z*z == DBL_MAX exactly, found on the host."""
    below = np.nextafter(DBL_MAX, 0.0)
    z = float(np.sqrt(below))
    with np.errstate(over="ignore"):
        for _ in range(64):
            if z * z == below:
                break
            z = float(np.nextafter(z, 0.0 if z * z > below else np.inf))
        assert z * z == below
        for x in 2.0**485 * np.array([1.0625, 1.125, 1.25, 1.375]):
            if (x * x + 0.0 * 0.0) + z * z == DBL_MAX:
                return np.array([x, 0.0, z])
    raise AssertionError("no point with squared range DBL_MAX")


def _reaches_range_compare(O, spec, p):
    """The oracle's decisions before the range compare (FoV on the normalised z, projection, truncation, bounds)."""
    model, intr, dist, W, H = spec
    cam = O.create_camera(model, intr, dist)
    with np.errstate(over="ignore", invalid="ignore"):
        n2 = _sq(p)[0]
        nz = p[2] / np.sqrt(n2) if n2 > 0 else p[2]
        if not nz >= np.cos(O.estimate_camera_fov(cam, W, H)):
            return False
        u, v = O.project(cam, p)
    return bool(0 <= np.trunc(u) < W and 0 <= np.trunc(v) < H)


def test_squared_ranges_of_dbl_max_and_infinity(gpu, oracle):
    dm = _dbl_max_point()
    with np.errstate(over="ignore"):
        assert _sq(dm)[0] == DBL_MAX
        infs = [np.array([0.0, 0.0, 1e200]), np.array([1e200, 0.0, 1e200]), np.array([3e160, -1e-3, 2e200])]
        assert all(_sq(p)[0] == np.inf for p in infs)
    for spec in (EQUI, PIN):
        assert _reaches_range_compare(oracle, spec, dm)
    for p in infs:  # pinhole: z / sqrt(inf) = 0 < cos(fov); equirectangular (FoV pi): the centre pixel
        assert _reaches_range_compare(oracle, EQUI, p)
        assert not _reaches_range_compare(oracle, PIN, p)
    fin = np.array([1e-3, 1e-3, 1.0])  # the same pixel of EQUI, (320, 160)
    cam = oracle.create_camera(*EQUI[:3])
    assert np.array_equal(np.trunc(oracle.project(cam, fin)), np.trunc(oracle.project(cam, dm)))
    assert np.array_equal(np.trunc(oracle.project(cam, infs[0])), np.trunc(oracle.project(cam, dm)))
    cases = [
        ([dm], 0), ([infs[0]], -1), ([infs[1]], -1), (infs, -1),
        ([dm, dm], 1), ([dm, infs[0]], 0), ([infs[0], dm, infs[1]], 1),
        ([fin, dm], 0), ([dm, fin], 1), ([fin, infs[0]], 0), ([infs[0], fin, infs[2]], 1),
        ([infs[0], dm, fin, infs[1], dm], 2),
    ]
    for spec in (EQUI, PIN):
        for rows, want in cases:
            pts = _xyzw(np.array(rows))
            inten = np.linspace(0.1, 0.9, len(rows)) + 1e-9
            ref = check(gpu, oracle, spec, pts, inten, layout="f64")
            if spec is EQUI:
                assert ref[160, 320] == want, (rows, ref[160, 320])
                assert (ref >= 0).sum() == (want >= 0)


# ---- 3. special input ----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("spec", [PIN, EQUI], ids=["pinhole", "equirectangular"])
def test_special_points_and_intensities(gpu, oracle, spec):
    """NaN and +-Inf in each coordinate, the camera centre, points behind the camera, the (-1, 0) truncation strip, the last
    row and column, beside ordinary points of the same pixels; intensities NaN, negative and above 1."""
    sp = _special_points(640, 480).astype(np.float32).astype(np.float64)
    rng = np.random.default_rng(5)
    base = _at_pixel(rng.integers(0, 640, 400), rng.integers(0, 480, 400), rng.choice([0.5, 1.0, 2.0, 4.0], 400))
    pts = np.concatenate([base[:200], sp, base[200:], sp[::-1], -base[:50]])  # -base: behind the camera
    n = len(pts)
    inten = _ramp(n)
    inten[::7] = np.nan
    inten[1::7] = -0.5 - inten[1::7]
    inten[2::7] = 1.5 + inten[2::7]
    inten[3::7] = -0.0
    ref = check_both(gpu, oracle, spec, _xyzw(pts), inten)
    assert (ref >= 0).sum() > 100


def test_nan_intensities_in_both_layouts(gpu, oracle):
    """NaN intensities win pixels: NaN-ness in the float4 layout, the exact payload in the double layout."""
    rng = np.random.default_rng(6)
    pts = _at_pixel(rng.integers(0, 64, 5000), rng.integers(0, 64, 5000), rng.choice([1.0, 2.0], 5000))
    inten = _ramp(len(pts))
    inten[rng.random(len(pts)) < 0.5] = np.nan
    payload = np.array([0x7FF8000000000123, 0xFFF0000000000001], dtype=np.uint64).view(np.float64)
    inten[::3] = payload[np.arange(len(inten[::3])) % 2]
    check(gpu, oracle, PIN, _xyzw(pts), inten, layout="f32")
    check(gpu, oracle, PIN, _xyzw(pts), _double_layout(inten), layout="f64")


# ---- 4. sizes ------------------------------------------------------------------------------------------------------------


def _targeted(spec, n, rng, margin=2.0):
    """n float32 points of a distortion-free pinhole spec aimed uniformly at pixels in [-margin, W + margin) x ..."""
    model, intr, dist, W, H = spec
    fx, fy, cx, cy = intr
    z = rng.choice([0.5, 1.0, 2.0, 4.0, 8.0], n) * (1.0 + rng.integers(0, 64, n) / 64.0)
    u, v = rng.uniform(-margin, W + margin, n), rng.uniform(-margin, H + margin, n)
    p = np.stack([(u - cx) / fx * z, (v - cy) / fy * z, z], 1).astype(np.float32).astype(np.float64)
    return p


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 4097])
def test_point_counts_at_the_block_edges(gpu, oracle, n):
    rng = np.random.default_rng(n)
    pts = _targeted(PIN, n, rng)
    if n > 3:
        pts[-1] = pts[0]  # a tie with the last index
        pts[-2] = pts[n // 2]
    if n == 0:
        check(gpu, oracle, PIN, np.zeros((0, 4)), np.zeros(0))
        return
    check_both(gpu, oracle, PIN, _xyzw(pts), _ramp(n))


def test_indices_above_float_precision(gpu, oracle):
    """2^24 + 3 points (float4 layout): indices 2^24 ... 2^24 + 2 are not all floats, the winners must still be exact.  The
    last 2^16 + 3 points are the nearest of their pixels, each tied with a copy at a random earlier index: they win by
    index, the last three in pixels of their own."""
    n = (1 << 24) + 3
    rng = np.random.default_rng(24)
    pts = _targeted(PIN, n, rng)  # ranges from z >= 0.5
    tail = (1 << 16) + 3
    ix, iy = rng.integers(0, 640, tail), rng.integers(0, 480, tail)
    ix[-3:], iy[-3:] = [5, 6, 7], [470, 470, 470]
    ix[:-3][(iy[:-3] == 470) & (ix[:-3] >= 5) & (ix[:-3] <= 7)] = 0
    near = _at_pixel(ix, iy, np.full(tail, 0.25))
    pts[-tail:] = near
    pts[rng.choice(n - tail, tail, replace=False)] = near
    inten = rng.integers(0, 256, n) / 256.0
    ref = check(gpu, oracle, PIN, _xyzw(pts), inten, layout="f32")
    assert list(ref[470, 5:8]) == [1 << 24, (1 << 24) + 1, (1 << 24) + 2]
    assert (ref >= n - tail).sum() > 50_000


def test_contention_on_sixteen_pixels(gpu, oracle):
    """2*10^7 points on 16 pixels: every atomicMin / atomicMax of a pixel contended by ~10^6 threads, with ties among
    the nearest."""
    n = 20_000_000
    rng = np.random.default_rng(16)
    pix = rng.integers(0, 16, n)
    z = np.array([2.0, 4.0, 8.0, 16.0])[rng.integers(0, 4, n)]
    z[rng.random(n) < 1e-5] = 1.0  # a few nearer points per pixel, scattered through the order
    pts = _at_pixel(300 + (pix % 4) * 3, 200 + (pix // 4) * 5, z, 0.5, 0.5)
    inten = rng.integers(0, 256, n) / 256.0
    ref = check(gpu, oracle, PIN, _xyzw(pts), inten, layout="f32")
    assert (ref >= 0).sum() == 16


@pytest.mark.parametrize("size", [(1, 1), (1, 4097), (4097, 1), (15, 17), (16, 16), (257, 1), (255, 257), (256, 256), (65537, 1)])
def test_image_sizes_at_the_grid_edges(gpu, oracle, size):
    """1 x 1, single rows and columns, and W*H = 256k - 1, 256k, 256k + 1 (the init and gather grids)."""
    W, H = size
    spec = ("plumb_bob", [512.0, 512.0, W / 2.0, H / 2.0], [], W, H)
    rng = np.random.default_rng(W * 7 + H)
    n = max(min(20 * W * H, 400_000), 1000) + 37
    pts = _targeted(spec, n, rng)
    pts[n // 2 : n // 2 + 4, :2] = 0.0  # on the optical axis: inside the FoV estimated for any size
    pts[-5:] = pts[:5]
    ref = check_both(gpu, oracle, spec, _xyzw(pts), _ramp(n))
    assert (ref >= 0).sum() >= (1 if W * H == 1 else 0.5 * W * H)


def test_large_images(gpu, oracle):
    """1920 x 960 equirectangular (points all around) and 4096 x 4096 pinhole."""
    rng = np.random.default_rng(1920)
    spec = ("equirectangular", [1920.0, 960.0], [], 1920, 960)
    d = rng.normal(size=(2_000_000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = (d * rng.choice([1.0, 2.0, 4.0], (len(d), 1))).astype(np.float32).astype(np.float64)
    pts[-1000:] = pts[:1000]
    check_both(gpu, oracle, spec, _xyzw(pts), _ramp(len(pts)))
    spec = ("plumb_bob", [2048.0, 2048.0, 2048.0, 2048.0], [], 4096, 4096)
    pts = _targeted(spec, 3_000_000, rng)
    pts[-1000:] = pts[:1000]
    check_both(gpu, oracle, spec, _xyzw(pts), _ramp(len(pts)))


@pytest.mark.parametrize("model", util.MODELS)
def test_every_model_at_a_pose_with_translation(gpu, oracle, model):
    pr = util.random_problem(model, n=200_000, seed=31)
    pts = pr["points"].copy()
    pts[-2000:] = pts[:2000]
    spec = (model, pr["intrinsics"], pr["distortion"], pr["W"], pr["H"])
    T = pr["T"]
    assert np.abs(T[:3, 3]).max() > 0 and not np.allclose(T[:3, :3], np.eye(3))
    ref = check_both(gpu, oracle, spec, pts, pr["intensities"], T)
    assert (ref >= 0).sum() > 1000


# ---- 5. refusals ---------------------------------------------------------------------------------------------------------


def _raw(V, W, H, n, pts=True, inten=True, T=True, out=True):
    L = V._lib.load_library()
    intr = np.array(DYADIC_PINHOLE[0])
    p, i, t = np.ones(4 * max(n, 1)), np.zeros(max(n, 1)), np.eye(4).reshape(-1)
    img, idx = np.zeros(4), np.zeros(4, np.int32)
    dp = C.POINTER(C.c_double)
    rc = L.vlcal_generate_lidar_image(
        -1, 0, intr.ctypes.data_as(dp), 4, None, 0, W, H, t.ctypes.data_as(dp) if T else None, p.ctypes.data if pts else None,
        i.ctypes.data if inten else None, n, img.ctypes.data if out else None, idx.ctypes.data if out else None)
    return rc, L.vlcal_nid_last_error().decode() if rc else ""


def test_refusals(gpu):
    """Negative n, zero sizes, null pointers, and more than 2^31 - 1 pixels (pixel indices are int): refused with
    VLCAL_ERR_INVALID_ARGUMENT before anything is allocated; the output buffers here hold 4 pixels."""
    ERR = gpu._lib.ERR_INVALID_ARGUMENT
    assert _raw(gpu, 2, 2, 0)[0] == 0
    assert _raw(gpu, 2, 2, 1)[0] == 0
    assert _raw(gpu, 2, 2, -1)[0] == ERR
    assert _raw(gpu, 0, 2, 0)[0] == ERR
    assert _raw(gpu, 2, 0, 0)[0] == ERR
    assert _raw(gpu, -2, -2, 0)[0] == ERR
    assert _raw(gpu, 2, 2, 1, pts=False)[0] == ERR
    assert _raw(gpu, 2, 2, 1, inten=False)[0] == ERR
    assert _raw(gpu, 2, 2, 0, T=False)[0] == ERR
    assert _raw(gpu, 2, 2, 0, out=False)[0] == ERR
    for W, H in ((65536, 65536), (46341, 46341), (2147483647, 2), (2, 1 << 30 | 1 << 29 | 1)):
        rc, msg = _raw(gpu, W, H, 0)
        assert rc == ERR and "2^31-1 pixels" in msg, (W, H, rc, msg)
    rc, msg = _raw(gpu, 65536, 65536, 1)
    assert rc == ERR and "2^31-1 pixels" in msg
