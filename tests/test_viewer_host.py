"""CPU suite of the headless viewer: the Turbo table, the numpy checker the GPU tests hold the kernels to
(tests/viewer_oracle.py) on cases with known answers, transformation discovery, the coloured PLY, the C ABI and the
CLI's refusals.  No kernel runs here."""
import ctypes as C
import itertools
import json

import numpy as np
import pytest

import util
import viewer_oracle as VO

PIN = ("plumb_bob", [512.0, 512.0, 320.0, 240.0], [], 640, 480)  # identity pose: u = 512 x / z + 320, exact for dyadic points


def _at(u, v, z=2.0):
    return [(u - 320.0) / 512.0 * z, (v - 240.0) / 512.0 * z, z]


def _image(W=640, H=480, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (H, W), dtype=np.uint8)


def test_turbo_table_is_opencvs(vlcal):
    table = vlcal.turbo_colormap()
    assert table.shape == (256, 3) and table.dtype == np.uint8
    assert np.array_equal(table, VO.turbo_table())
    assert list(table[0]) == [48, 18, 59] and list(table[255]) == [122, 4, 3]  # the ends of the published table


def test_new_abi_symbols_resolve(vlcal):
    lib = C.CDLL(vlcal.library_path())
    for name in ("vlcal_colorize_points", "vlcal_render_overlay", "vlcal_turbo_colormap"):
        assert hasattr(lib, name), name
    for name in ("PointsColorUpdater", "render_overlay", "turbo_colormap"):
        assert name in vlcal.__all__ and hasattr(vlcal, name)


def test_checker_known_answers(oracle):
    cam = oracle.create_camera(*PIN[:3])
    img = _image()
    pts = np.array([
        _at(100.5, 50.5, -2.0),  # behind the camera
        _at(-0.5, 7.5),          # u in (-1, 0): truncates to column 0
        _at(640.0, 7.5),         # u = W: outside
        _at(639.5, 479.5),       # last pixel
        _at(-1.0, 7.5),          # u = -1: outside
    ])
    inten = np.array([0.5, 0.25, 0.25, 1.0, 0.0])
    T = np.eye(4)
    for w in (0.0, np.float32(0.7), 1.0):
        c = VO.colorize(oracle, cam, img, T, pts, inten, w)
        assert c.dtype == np.float32 and c.shape == (5, 4)
        assert not c[0].any() and not c[2].any() and not c[4].any()
        assert c[1, 3] == np.float32(w) + np.float32(1.0 - float(np.float32(w)))
    turbo = VO.turbo_table().astype(np.float32) / np.float32(255)
    pure_turbo = VO.colorize(oracle, cam, img, T, pts, inten, 0.0)
    assert np.array_equal(pure_turbo[1, :3], turbo[63]) and np.array_equal(pure_turbo[3, :3], turbo[255])  # int(0.25 * 255) = 63
    pure_gray = VO.colorize(oracle, cam, img, T, pts, inten, 1.0)
    assert np.array_equal(pure_gray[1, :3], np.full(3, np.float32(img[7, 0]) / np.float32(255)))
    assert np.array_equal(pure_gray[3, :3], np.full(3, np.float32(img[479, 639]) / np.float32(255)))
    assert pure_gray[1, 3] == 1.0 and pure_turbo[1, 3] == 1.0


def test_checker_clamps_intensities():
    got = VO.turbo_index([np.nan, -1.0, -0.0, 0.0, 1.0 / 255, 0.999, 1.0, 7.0, np.inf, -np.inf, 1e300])
    assert list(got) == [0, 0, 0, 0, 1, 254, 255, 255, 255, 0, 255]


def test_checker_keeps_the_viewers_wider_fov(oracle):
    """A point between the cost's FoV and the viewer's (0.5 degrees wider) is coloured by the viewer, skipped by the
    cost's rule.  The FoV is estimated from the pixels (0, 0), (W/2, 0) and (0, H/2) (estimate_fov.cpp:37), so with the
    principal point near a corner the band lies inside the image on the far side."""
    W, H = 640, 480
    cam = oracle.create_camera("plumb_bob", [512.0, 512.0, 100.0, 100.0], [])
    fov = oracle.estimate_camera_fov(cam, W, H)
    assert 0.3 < fov < 0.6
    th = fov + np.deg2rad(0.25)
    p = np.array([[np.sin(th), 0.0, np.cos(th)]]) * 3.0
    assert VO.classify(oracle, cam, W, H, VO.cost_cos_fov(oracle, cam, W, H), np.eye(4), p)[0][0] == -1
    assert VO.classify(oracle, cam, W, H, VO.viewer_cos_fov(oracle, cam, W, H), np.eye(4), p)[0][0] >= 0


@pytest.mark.parametrize("model", ["plumb_bob", "equirectangular"])
def test_checker_overlay_at_radius_0_is_generate_lidar_image(oracle, model):
    pr = util.random_problem(model, n=30_000, seed=3)
    pr["points"][-500:] = pr["points"][:500]  # ties
    cam = oracle.create_camera(model, pr["intrinsics"], pr["distortion"])
    _, ref = oracle.generate_lidar_image(cam, pr["W"], pr["H"], pr["T"], pr["points"], pr["intensities"])
    bgr, index = VO.overlay(oracle, cam, pr["image"], pr["T"], pr["points"], pr["intensities"], 0, 0.7)
    assert np.array_equal(index, ref) and (ref >= 0).sum() > 1000
    blank = index < 0
    assert np.array_equal(bgr[blank], np.repeat(pr["image"][blank][:, None], 3, axis=1))


@pytest.mark.parametrize("radius", [1, 2])
def test_checker_overlay_equals_the_serial_rule(oracle, radius):
    W, H = 48, 40
    cam = oracle.create_camera("plumb_bob", [40.0, 40.0, 24.0, 20.0], [])
    rng = np.random.default_rng(radius)
    z = rng.choice([1.0, 2.0, 4.0], 600)
    pts = np.stack([(rng.integers(-2, W + 2, 600) + 0.5 - 24.0) / 40.0 * z, (rng.integers(-2, H + 2, 600) + 0.5 - 20.0) / 40.0 * z, z], 1)
    pts[-100:] = pts[:100]
    img = _image(W, H)
    _, index = VO.overlay(oracle, cam, img, np.eye(4), pts, rng.random(600), radius, 0.5)
    assert np.array_equal(index, VO.overlay_serial(oracle, cam, img, np.eye(4), pts, None, radius, 0.5))
    _, index0 = VO.overlay(oracle, cam, img, np.eye(4), pts, rng.random(600), 0, 0.5)
    assert (index >= 0).sum() > 2 * (index0 >= 0).sum()
    assert index[0, 0] >= 0 or index[H - 1, W - 1] >= 0 or index[0, W - 1] >= 0 or index[H - 1, 0] >= 0  # squares clipped at a corner


KEYS = ["init_T_lidar_camera_auto", "init_T_lidar_camera", "T_lidar_camera"]
LABELS = ["INIT_GUESS (AUTO)", "INIT_GUESS (MANUAL)", "CALIBRATION_RESULT"]


@pytest.mark.parametrize("present", list(itertools.product([False, True], repeat=3)))
def test_transformation_discovery(vlcal, capsys, present):
    from direct_visual_lidar_calibration_b200 import io as vio
    from direct_visual_lidar_calibration_b200 import viewer

    tums = [[0.1 * (k + 1), 0.2, -0.3, 0.0, 0.0, np.sin(0.1 * (k + 1)), np.cos(0.1 * (k + 1))] for k in range(3)]
    results = {key: tum for key, tum, on in zip(KEYS, tums, present) if on}
    config = {"results": results} if any(present) else {}
    labels, poses, selected = viewer.find_transformations(config)
    err = capsys.readouterr().err
    if not any(present):
        assert labels == ["NONE"] and np.array_equal(poses[0], np.eye(4)) and selected == 0
        assert "error: no transformation found in calib.json!!" in err
        return
    assert err == ""
    assert labels == [lab for lab, on in zip(LABELS, present) if on]
    assert selected == len(labels) - 1  # the last one found (viewer.cpp:83)
    for pose, tum in zip(poses, [t for t, on in zip(tums, present) if on]):
        assert np.allclose(pose, vio.tum_to_T(tum), atol=1e-15)
    for name, on in zip(("auto", "manual", "result"), present):
        if on:
            assert labels[viewer.find_transformations(config, name)[2]] == LABELS[("auto", "manual", "result").index(name)]
        else:
            with pytest.raises(ValueError):
                viewer.find_transformations(config, name)


def test_ply_without_colors_is_byte_identical_to_before(vlcal, tmp_path):
    """The layout of preprocess.cpp:163-169, spelled out byte for byte."""
    from direct_visual_lidar_calibration_b200 import io as vio

    pts = (np.arange(30, dtype=np.float64).reshape(10, 3) - 7.0) / 8.0
    inten = np.arange(10) / 16.0
    vio.save_ply_binary(str(tmp_path / "a.ply"), pts, inten)
    raw = (tmp_path / "a.ply").read_bytes()
    head = b"ply\nformat binary_little_endian 1.0\nelement vertex 10\nproperty float x\nproperty float y\nproperty float z\nproperty float intensity\nend_header\n"
    body = np.concatenate([pts, inten[:, None]], axis=1).astype("<f4").tobytes()
    assert raw == head + body
    vio.save_ply_binary(str(tmp_path / "b.ply"), pts)
    assert (tmp_path / "b.ply").read_bytes() == head.replace(b"property float intensity\n", b"") + pts.astype("<f4").tobytes()


def test_colored_ply_round_trip(vlcal, tmp_path):
    from direct_visual_lidar_calibration_b200 import io as vio

    rng = np.random.default_rng(1)
    pts = rng.normal(size=(100, 3)).astype(np.float32).astype(np.float64)
    inten = rng.integers(0, 256, 100) / 256.0
    colors = rng.random((100, 4)).astype(np.float32)
    colors[0], colors[1], colors[2] = 0.0, 1.0, [0.5 / 255, 1.5 / 255, 2.5 / 255, 254.5 / 255]
    path = str(tmp_path / "c.ply")
    vio.save_ply_binary(path, pts, inten, colors=colors)
    got_pts, got_inten = vio.load_ply(path)  # the colour properties are skipped
    assert np.array_equal(got_pts, pts) and np.array_equal(got_inten, inten)
    raw = open(path, "rb").read()
    head, body = raw.split(b"end_header\n", 1)
    assert head.decode().splitlines()[3:] == [f"property float {n}" for n in ("x", "y", "z", "intensity")] + [f"property uchar {n}" for n in ("red", "green", "blue", "alpha")]
    rec = np.frombuffer(body, dtype=[("xyzi", "<f4", 4), ("rgba", "u1", 4)])
    assert len(rec) == 100
    assert np.array_equal(rec["rgba"], np.rint(colors.astype(np.float64) * 255.0).astype(np.uint8))
    assert list(rec["rgba"][0]) == [0, 0, 0, 0] and list(rec["rgba"][1]) == [255] * 4
    fields = vio._read_ply_fields(path)
    assert [f[0] for f in fields] == ["x", "y", "z", "intensity", "red", "green", "blue", "alpha"]


def test_cli_reports_a_missing_calib_json(vlcal, tmp_path, capsys):
    from direct_visual_lidar_calibration_b200 import viewer

    assert viewer.main([str(tmp_path)]) == 1
    assert f"error: failed to open {tmp_path}/calib.json" in capsys.readouterr().err


def test_cli_refuses_an_absent_transformation_and_bad_options(vlcal, tmp_path, capsys):
    from direct_visual_lidar_calibration_b200 import viewer

    config = {"camera": {"camera_model": "plumb_bob", "intrinsics": PIN[1], "distortion_coeffs": []}, "meta": {"bag_names": []},
              "results": {"init_T_lidar_camera": [0, 0, 0, 0, 0, 0, 1]}}
    (tmp_path / "calib.json").write_text(json.dumps(config))
    before = (tmp_path / "calib.json").read_bytes()
    assert viewer.main([str(tmp_path), "--transformation", "result"]) == 1
    assert "holds no result transformation" in capsys.readouterr().err
    assert viewer.main([str(tmp_path), "--point_radius", "9"]) == 1
    assert viewer.main([str(tmp_path), "--blend_weight", "1.5"]) == 1
    assert (tmp_path / "calib.json").read_bytes() == before


def test_abi_refusals_need_no_device(vlcal):
    """Arguments are checked before a device is looked for, as in vlcal_generate_lidar_image."""
    cam = vlcal.create_camera(*PIN[:3])
    img, pts, inten = _image(), np.array([_at(5.5, 5.5)]), np.array([0.5])
    ERR = vlcal._lib.ERR_INVALID_ARGUMENT
    for kwargs in ({"point_radius": -1}, {"point_radius": 9}, {"blend_weight": -0.1}, {"blend_weight": 1.1}, {"blend_weight": float("nan")}):
        with pytest.raises(vlcal.VlcalError) as e:
            vlcal.render_overlay(cam, img, np.eye(4), pts, inten, **kwargs)
        assert e.value.code == ERR, kwargs
    for w in (-0.1, 1.1, float("nan")):
        with pytest.raises(vlcal.VlcalError) as e:
            vlcal.PointsColorUpdater(cam, img, pts, inten).update(np.eye(4), w)
        assert e.value.code == ERR
    if vlcal.device_count() == 0:
        with pytest.raises(vlcal.VlcalError) as e:
            vlcal.PointsColorUpdater(cam, img, pts, inten).update(np.eye(4), 0.7)
        assert e.value.code == vlcal._lib.ERR_NO_DEVICE and "no CPU fallback" in str(e.value)
