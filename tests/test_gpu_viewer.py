"""GPU suite of the headless viewer (csrc/viewer.cu, the radius of csrc/lidar_image.cu, viewer.py), held to the numpy
checker of tests/viewer_oracle.py.

Bar: PointsColorUpdater.update bit-equal to the checker (float32 compared as uint32); the overlay's index map and BGR
image equal to the checker's, and at radius 0 its index map equal to generate_lidar_image's.  Every case runs in both
layouts the upload chooses from (float-exact values -> float4, otherwise double4)."""
import json
import os

import numpy as np
import pytest

import util
import viewer_oracle as VO
from direct_visual_lidar_calibration_b200 import synthetic as S

pytestmark = pytest.mark.gpu
WEIGHTS = [0.0, float(np.float32(0.7)), 1.0]
PIN = ("plumb_bob", [512.0, 512.0, 320.0, 240.0], [], 640, 480)  # identity pose: u = 512 x / z + 320, exact for dyadic points


def _xyzw(p):
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    return np.concatenate([p, np.ones((p.shape[0], 1))], axis=1)


def _is_f32(pts, inten):
    with np.errstate(over="ignore", invalid="ignore"):
        v = np.concatenate([pts[:, :3].reshape(-1), inten])
        return bool(np.all((v.astype(np.float32).astype(np.float64) == v) | np.isnan(v)))


def _double_layout(inten):
    """The same intensities moved off float32 (1e-9 is not a float), so that the upload takes the double layout."""
    out = np.array(inten, dtype=np.float64)
    fin = np.isfinite(out)
    out[fin] += 1e-9
    return out


def _layouts(V, cam, size, pts, inten):
    """(name, intensities) of the two layouts, each confirmed through the upload rule as the library reports it."""
    out = [("f32", inten), ("f64", _double_layout(inten))]
    for name, ins in out:
        assert _is_f32(pts, ins) == (name == "f32")
        if len(pts):
            sub = slice(0, min(len(pts), 1 << 16))
            _, on_f32 = V.ViewCulling(cam, size).debug_culled_points(pts[sub], ins[sub], np.eye(4), keep_all=True)
            assert on_f32 == _is_f32(pts[sub], ins[sub])
    return out


def _assert_colors(got, ref):
    assert got.dtype == np.float32 and got.shape == ref.shape
    bad = (got.view(np.uint32) != ref.view(np.uint32)).any(axis=1)
    assert not bad.any(), (int(bad.sum()), np.nonzero(bad)[0][:5], got[bad][:3], ref[bad][:3])


def check_update(V, O, spec, image, pts, inten, T, weights=WEIGHTS):
    """update() == checker in both layouts and for every weight; returns the checker's colours of the float4 layout at the first weight."""
    model, intr, dist, W, H = spec
    cam, ocam = V.create_camera(model, intr, dist), O.create_camera(model, intr, dist)
    first = None
    for _, ins in _layouts(V, cam, (W, H), pts, inten):
        upd = V.PointsColorUpdater(cam, image, pts, ins)
        for w in weights:
            ref = VO.colorize(O, ocam, image, T, pts, ins, w)
            _assert_colors(upd.update(T, w), ref)
            first = ref if first is None else first
    return first


def check_overlay(V, O, spec, image, pts, inten, T, radius, w=0.7):
    """render_overlay == checker in both layouts; returns the checker's (bgr, index) of the float4 layout."""
    model, intr, dist, W, H = spec
    cam, ocam = V.create_camera(model, intr, dist), O.create_camera(model, intr, dist)
    first = None
    for _, ins in _layouts(V, cam, (W, H), pts, inten):
        bgr, index = V.render_overlay(cam, image, T, pts, ins, point_radius=radius, blend_weight=w)
        ref_bgr, ref_index = VO.overlay(O, ocam, image, T, pts, ins, radius, np.float32(w))
        bad = index != ref_index
        assert not bad.any(), (radius, int(bad.sum()), np.argwhere(bad)[:5], index[bad][:5], ref_index[bad][:5])
        bad = (bgr != ref_bgr).any(axis=2)
        assert not bad.any(), (radius, int(bad.sum()), np.argwhere(bad)[:5], bgr[bad][:3], ref_bgr[bad][:3])
        if radius == 0:
            _, k5 = V.generate_lidar_image(cam, (W, H), T, pts, ins)
            assert np.array_equal(index, k5)
        first = (ref_bgr, ref_index) if first is None else first
    return first


def _image(W, H, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (H, W), dtype=np.uint8)


def _ramp(n):
    return (np.arange(n) % 4096) / 4096.0 * 1.25 - 0.125  # float-exact, below 0 and above 1 at the ends


def _at(u, v, z):
    z = np.asarray(z, dtype=np.float64)
    return np.stack([(np.asarray(u) - 320.0) / 512.0 * z, (np.asarray(v) - 240.0) / 512.0 * z, z + 0.0 * np.asarray(u)], axis=-1)


NONFINITE = np.array([
    [np.nan, 0.0, 1.0], [0.0, np.nan, 1.0], [0.0, 0.0, np.nan], [np.inf, 0.0, 1.0], [-np.inf, 0.0, 1.0], [0.0, np.inf, 1.0], [0.0, 0.0, np.inf], [0.0, 0.0, -np.inf],
    [np.inf, np.inf, np.inf], [0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 2.0**-10], [-(2.0**-7), 0.0, -(2.0**-7)],
])


# ---- 1. update() ---------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("model", util.MODELS)
def test_update_every_model(gpu, oracle, model):
    """A random cloud at a pose with rotation and translation, NaN / +-inf coordinates and the camera centre among it,
    intensities below 0, above 1 and NaN."""
    pr = util.random_problem(model, n=100_000, seed=51)
    pts = pr["points"].copy()
    pts[1000 : 1000 + len(NONFINITE), :3] = NONFINITE
    inten = _ramp(len(pts))
    inten[::97] = np.nan
    spec = (model, pr["intrinsics"], pr["distortion"], pr["W"], pr["H"])
    ref = check_update(gpu, oracle, spec, pr["image"], pts, inten, pr["T"])
    coloured = ref[:, 3] != 0
    assert coloured.mean() > 0.3 and not coloured.all()


@pytest.mark.parametrize("model", [m for m in util.MODELS if m != "equirectangular"])
def test_update_colours_the_band_the_cost_rejects(gpu, oracle, model):
    """Points between the cost's FoV and the viewer's, 0.5 degrees wider.  The FoV is estimated from the pixels (0, 0),
    (W/2, 0) and (0, H/2), so with the principal point towards that corner the band lies inside the image on the far side."""
    intr, dist, (W, H) = util.CAMERAS[model]
    intr = list(intr)
    intr[2], intr[3] = 200.0, 150.0
    ocam = oracle.create_camera(model, intr, dist)
    fov = oracle.estimate_camera_fov(ocam, W, H)
    rng = np.random.default_rng(52)
    th = fov + np.deg2rad(rng.uniform(-0.25, 0.75, 40_000))
    az = rng.uniform(-np.pi, np.pi, th.size)
    pts = np.stack([np.sin(th) * np.cos(az), np.sin(th) * np.sin(az), np.cos(th)], 1) * rng.uniform(1.0, 8.0, (th.size, 1))
    pts = _xyzw(pts.astype(np.float32).astype(np.float64))
    image = _image(W, H, 52)
    ref = check_update(gpu, oracle, (model, intr, dist, W, H), image, pts, _ramp(len(pts)), np.eye(4), weights=[WEIGHTS[1]])
    by_cost, _ = VO.classify(oracle, ocam, W, H, VO.cost_cos_fov(oracle, ocam, W, H), np.eye(4), pts)
    band = (ref[:, 3] != 0) & (by_cost < 0)
    assert band.sum() > 100, int(band.sum())
    assert ((ref[:, 3] == 0) & (th > fov + np.deg2rad(0.6))).sum() > 100  # beyond the viewer's threshold: skipped


def test_update_on_the_image_borders(gpu, oracle):
    """u and v on each border of the image, one ulp either side of it and in the (-1, 0) strip that truncates to 0."""
    rows = []
    for z in (1.0, 2.0):
        for edge, other in ((0.0, 100.5), (-1.0, 100.5), (640.0, 100.5), (639.0, 100.5)):
            rows += [_at(edge, other, z), _at(-0.5 if edge <= 0 else edge - 0.5, other, z)]
        for edge, other in ((0.0, 100.5), (-1.0, 100.5), (480.0, 100.5), (479.0, 100.5)):
            rows += [_at(other, edge, z), _at(other, -0.5 if edge <= 0 else edge - 0.5, z)]
    base = np.array(rows)
    image = _image(640, 480, 53)
    for dtype in (np.float32, np.float64):  # an ulp of the layout the cloud travels in
        b = base.astype(dtype)
        pts = np.concatenate([b, np.nextafter(b, dtype(np.inf)), np.nextafter(b, dtype(-np.inf))]).astype(np.float64)
        inten = _ramp(len(pts)) if dtype is np.float32 else _double_layout(_ramp(len(pts)))
        cam = gpu.create_camera(*PIN[:3])
        ocam = oracle.create_camera(*PIN[:3])
        assert _is_f32(pts, inten) == (dtype is np.float32)
        for w in WEIGHTS:
            ref = VO.colorize(oracle, ocam, image, np.eye(4), _xyzw(pts), inten, w)
            _assert_colors(gpu.PointsColorUpdater(cam, image, _xyzw(pts), inten).update(np.eye(4), w), ref)
        n = len(base)
        coloured = ref[:, 3] != 0
        assert coloured[:n].tolist() == [e for z in (1, 2) for e in (True, True, False, True, False, True, True, True) * 2]
        assert 0 < coloured[n:].sum() < 2 * n  # an ulp decides on either side of the borders


def test_update_of_an_empty_cloud(gpu, oracle):
    cam = gpu.create_camera(*PIN[:3])
    out = gpu.PointsColorUpdater(cam, _image(640, 480), np.zeros((0, 4)), np.zeros(0)).update(np.eye(4), 0.7)
    assert out.shape == (0, 4) and out.dtype == np.float32


# ---- 2. overlay ------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("radius", [0, 1, 2])
@pytest.mark.parametrize("model", ["plumb_bob", "equirectangular", "fisheye"])
def test_overlay_of_a_random_cloud(gpu, oracle, model, radius):
    pr = util.random_problem(model, n=150_000, seed=61)
    pts = pr["points"].copy()
    pts[-3000:] = pts[:3000]  # ties: the last index wins
    pts[500 : 500 + len(NONFINITE), :3] = NONFINITE
    inten = _ramp(len(pts))
    inten[::89] = np.nan
    spec = (model, pr["intrinsics"], pr["distortion"], pr["W"], pr["H"])
    bgr, index = check_overlay(gpu, oracle, spec, pr["image"], pts, inten, pr["T"], radius)
    assert (index >= 0).sum() > 10_000
    assert (index >= len(pts) - 3000).sum() > 100


@pytest.mark.parametrize("radius", [1, 2])
def test_overlay_squares_are_clipped_at_the_borders(gpu, oracle, radius):
    """One point in each corner and on each border: the squares lose the part outside the image and nothing wraps."""
    uv = [(0.5, 0.5), (639.5, 0.5), (0.5, 479.5), (639.5, 479.5), (320.5, 0.5), (320.5, 479.5), (0.5, 240.5), (639.5, 240.5), (1.5, 1.5), (300.5, 200.5)]
    pts = _xyzw(np.array([_at(u, v, 2.0) for u, v in uv]))
    image = _image(640, 480, 62)
    _, index = check_overlay(gpu, oracle, PIN, image, pts, np.linspace(0.0, 1.0, len(uv)).astype(np.float32).astype(np.float64), np.eye(4), radius)
    side = 2 * radius + 1
    assert (index == 9).sum() == side * side and (index == 3).sum() == (radius + 1) ** 2
    assert (index == 4).sum() == side * (radius + 1) and (index == 7).sum() == side * (radius + 1)
    assert index[0, 639 - radius] == 1 and index[0, 0] in (0, 8) and index[radius + 2 : 240 - radius, 0].max() == -1


@pytest.mark.parametrize("radius", [0, 1, 2])
def test_overlay_ties_go_to_the_last_index(gpu, oracle, radius):
    """Two points with equal squared range whose squares share pixels, in either order, and copies of one point."""
    a = np.array([5.25 / 512.0 * 4.0, 5.375 / 512.0 * 4.0, 4.0])  # pixel (325, 245), and so is (y, x, z)
    b = a[[1, 0, 2]]
    c = _at(300.5, 300.5, 2.0)
    pts = _xyzw(np.array([a, b, c, c, b, a, c]))
    assert (a[0] * a[0] + a[1] * a[1]) + a[2] * a[2] == (b[0] * b[0] + b[1] * b[1]) + b[2] * b[2]
    _, index = check_overlay(gpu, oracle, PIN, _image(640, 480, 63), pts, np.arange(7) / 8.0, np.eye(4), radius)
    assert index[300, 300] == 6 and index[245, 325] == 5 and set(np.unique(index)) == {-1, 5, 6}


def test_overlay_radius_closes_the_gaps_of_a_near_wall(gpu, oracle):
    """A near wall sampled at every second pixel in front of a far wall sampled at every pixel: at radius 0 the far wall
    shows through the gaps, at radius 1 and 2 it is hidden wherever the near wall stands."""
    u, v = np.meshgrid(np.arange(100, 300), np.arange(100, 250))
    far = _at(u.reshape(-1) + 0.5, v.reshape(-1) + 0.5, 8.0)
    un, vn = np.meshgrid(np.arange(150, 250, 2), np.arange(120, 220, 2))
    near = _at(un.reshape(-1) + 0.5, vn.reshape(-1) + 0.5, 1.0)
    pts = _xyzw(np.concatenate([far, near]))
    inten = np.concatenate([np.full(len(far), 0.25), np.full(len(near), 0.75)])
    image = _image(640, 480, 64)
    n_far = len(far)
    shown = {}
    for radius in (0, 1, 2):
        _, index = check_overlay(gpu, oracle, PIN, image, pts, inten, np.eye(4), radius)
        wall = index[120:219, 150:249]
        shown[radius] = int(((wall >= 0) & (wall < n_far)).sum())
        assert (wall >= 0).all()
    assert shown[0] > 7000 and shown[1] == 0 and shown[2] == 0


def test_overlay_of_an_empty_cloud_is_the_image(gpu, oracle):
    image = _image(640, 480, 65)
    bgr, index = gpu.render_overlay(gpu.create_camera(*PIN[:3]), image, np.eye(4), np.zeros((0, 4)), np.zeros(0))
    assert (index == -1).all() and np.array_equal(bgr, np.repeat(image[:, :, None], 3, axis=2))


# ---- 3. full size --------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("config", ["C2", "C3"])
def test_full_size(gpu, oracle, config):
    """The C2 cloud (10^6 points, 1920 x 1080 plumb_bob) and the C3 cloud (5 * 10^6, 3840 x 1920 equirectangular) against
    the checker; a second run is byte-identical (the atomics are order independent)."""
    camera_key, pattern, n = {"C2": ("pinhole_1920x1080", "os1_64", 1_000_000), "C3": ("equirect_3840x1920", "avia", 5_000_000)}[config]
    model, intr, dist, W, H = S.CAMERAS[camera_key]
    pts, inten = S.make_cloud(pattern, n, scene_seed=71, seed=72)
    image = _image(W, H, 73)
    T = S.gt_T_camera_lidar()
    cam, ocam = gpu.create_camera(model, intr, dist), oracle.create_camera(model, intr, dist)
    w = float(np.float32(0.7))
    upd = gpu.PointsColorUpdater(cam, image, pts, inten)
    colors = upd.update(T, w)
    _assert_colors(colors, VO.colorize(oracle, ocam, image, T, pts, inten, w))
    assert (colors[:, 3] != 0).mean() > 0.5
    assert np.array_equal(upd.update(T, w).view(np.uint32), colors.view(np.uint32))
    bgr, index = gpu.render_overlay(cam, image, T, pts, inten, point_radius=1, blend_weight=w)
    ref_bgr, ref_index = VO.overlay(oracle, ocam, image, T, pts, inten, 1, np.float32(w))
    assert np.array_equal(index, ref_index) and np.array_equal(bgr, ref_bgr)
    bgr2, index2 = gpu.render_overlay(cam, image, T, pts, inten, point_radius=1, blend_weight=w)
    assert np.array_equal(index2, index) and np.array_equal(bgr2, bgr)


# ---- 4. the tool ---------------------------------------------------------------------------------------------------------


def test_cli_end_to_end(gpu, oracle, tmp_path):
    """Two synthetic bags, init_T_lidar_camera = ground truth with a perturbation, T_lidar_camera = ground truth."""
    import cv2

    from direct_visual_lidar_calibration_b200 import io as vio
    from direct_visual_lidar_calibration_b200 import viewer

    data, dst = tmp_path / "data", tmp_path / "out"
    data.mkdir()
    bags = [S.make_bag("pinhole_640x480", "frustum", 40_000, config_index=9, bag_index=b) for b in range(2)]
    names = ["bag0", "bag1"]
    for name, bag in zip(names, bags):
        cv2.imwrite(str(data / (name + ".png")), bag["image"])
        vio.save_ply_binary(str(data / (name + ".ply")), bag["points"][:, :3], bag["intensities"])
    T_gt = bags[0]["T_gt"]
    T_init = S.perturb(T_gt, (1.5, -1.0, 1.0), (0.04, -0.03, 0.02))
    config = {
        "camera": {"camera_model": bags[0]["camera_model"], "intrinsics": bags[0]["intrinsics"], "distortion_coeffs": bags[0]["distortion"]},
        "meta": {"bag_names": names},
        "results": {"init_T_lidar_camera": vio.T_to_tum(vio.invert_isometry(T_init)), "T_lidar_camera": vio.T_to_tum(vio.invert_isometry(T_gt))},
    }
    vio.save_calib_json(str(data), config)
    before = (data / "calib.json").read_bytes()
    assert viewer.main([str(data), "--dst_path", str(dst)]) == 0
    assert (data / "calib.json").read_bytes() == before
    assert sorted(os.listdir(dst)) == sorted([n + s for n in names for s in ("_colored.ply", "_overlay.png")] + ["viewer_report.json"])
    assert sorted(os.listdir(data)) == sorted(["calib.json"] + [n + s for n in names for s in (".png", ".ply")])

    report = json.loads((dst / "viewer_report.json").read_text())
    assert report["labels"] == ["INIT_GUESS (MANUAL)", "CALIBRATION_RESULT"] and report["selected"] == "CALIBRATION_RESULT"
    assert report["bag_names"] == names and len(report["T_lidar_camera"]) == 2
    nid = np.array(report["nid"])
    assert nid.shape == (2, 2) and np.allclose(nid.sum(axis=0), report["nid_sum"], atol=1e-12)
    assert report["nid_sum"][1] < report["nid_sum"][0] and (nid[:, 1] < nid[:, 0]).all()

    proj = gpu.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    ocam = oracle.create_camera(bags[0]["camera_model"], bags[0]["intrinsics"], bags[0]["distortion"])
    labels, T_lc, selected = viewer.find_transformations(config)
    T_sel = vio.invert_isometry(T_lc[selected])
    for b, name in enumerate(names):
        d = vio.load_visual_lidar_data(str(data), name)
        colors = gpu.PointsColorUpdater(proj, d.image, d.points, d.intensities).update(T_sel, 0.7)
        raw = (dst / (name + "_colored.ply")).read_bytes().split(b"end_header\n", 1)[1]
        rec = np.frombuffer(raw, dtype=[("xyzi", "<f4", 4), ("rgba", "u1", 4)])
        assert np.array_equal(rec["rgba"], np.rint(colors.astype(np.float64) * 255.0).astype(np.uint8))
        assert np.array_equal(rec["xyzi"][:, :3].astype(np.float64), d.points[:, :3])
        overlay = cv2.imread(str(dst / (name + "_overlay.png")), cv2.IMREAD_COLOR)
        ref_bgr, _ = VO.overlay(oracle, ocam, d.image, T_sel, d.points, d.intensities, 1, np.float32(0.7))
        assert np.array_equal(overlay, ref_bgr)
        fov = oracle.estimate_camera_fov(ocam, bags[0]["width"], bags[0]["height"])
        for k in range(2):  # the report's numbers are CostCalculatorNID::calculate's, the inlier count the selected pose's
            ref_nid, hist = oracle.nid_calculate(ocam, d.image, d.points, d.intensities, 16, fov, vio.invert_isometry(T_lc[k]))
            assert abs(ref_nid - nid[b, k]) < 1e-9
        assert report["selected_inliers"][b] == int(hist.sum())

    # another transformation on request, into the data directory by default
    assert viewer.main([str(data), "--transformation", "manual", "--point_radius", "0", "--first_n_bags", "1"]) == 0
    report = json.loads((data / "viewer_report.json").read_text())
    assert report["selected"] == "INIT_GUESS (MANUAL)" and report["bag_names"] == ["bag0"] and (data / "calib.json").read_bytes() == before
