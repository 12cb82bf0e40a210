"""GPU checks of preprocess_map: every stage byte-equal to the sequential checker (tests/cpp/preprocess_oracle.c) at its
edges, the refusals, and the CLI end to end -- its files equal to a CPU pipeline of the checker, the oracle's
generate_lidar_image and cv2, and initial_guess_auto + calibrate run on the dataset it writes."""
import json
import math
import os

import cv2
import numpy as np
import pytest

import preprocess_oracle as PO
from direct_visual_lidar_calibration_b200 import io as vio
from direct_visual_lidar_calibration_b200 import preprocess as P
from direct_visual_lidar_calibration_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _cloud(n, leaf, seed):
    """Points over ~120^3 voxels of the leaf: merges, hash collisions and evictions at every size."""
    rng = np.random.default_rng(seed)
    pts = np.empty((n, 4), np.float32)
    pts[:, :3] = (rng.uniform(-60.0, 60.0, (n, 3)) * leaf).astype(np.float32)
    pts[:, 3] = rng.uniform(0.0, 100.0, n).astype(np.float32)
    return pts


def _same_avg(gpu_pts, leaf):
    got = P.approximate_voxel_grid(gpu_pts, leaf)
    ref = PO.approximate_voxel_grid(gpu_pts, leaf)
    assert got.shape == ref.shape and got.tobytes() == ref.tobytes()
    return got


@pytest.mark.parametrize("leaf", [0.002, 0.05, 1.0])
@pytest.mark.parametrize("n", [0, 1, 511, 512, 513, 100_000, 10_000_000])
def test_voxel_grid_sizes(gpu, n, leaf):
    got = _same_avg(_cloud(n, leaf, seed=n % 1000 + 1), leaf)
    if n >= 100_000:
        assert got.shape[0] < n  # voxels merged


def test_voxel_grid_one_run_of_a_million(gpu):
    rng = np.random.default_rng(2)
    pts = rng.uniform(0.0, 0.0499, (1_000_000, 4)).astype(np.float32)
    assert _same_avg(pts, 0.05).shape[0] == 1


def test_voxel_grid_alternating_colliding_voxels(gpu):
    rng = np.random.default_rng(3)
    pts = rng.uniform(0.0, 0.999, (200_001, 4)).astype(np.float32)
    pts[1::2, 0] += np.float32(512.0)  # voxels (0,0,0) and (512,0,0) share slot 0
    assert _same_avg(pts, 1.0).shape[0] == pts.shape[0]


def test_voxel_grid_edges(gpu):
    rng = np.random.default_rng(4)
    leaf = np.float32(0.05)
    k = rng.integers(-200, 200, (50_000, 3)).astype(np.float32)
    edge = (k * leaf).astype(np.float32)
    pts = np.empty((3 * edge.shape[0], 4), np.float32)
    pts[0::3, :3] = edge
    pts[1::3, :3] = np.nextafter(edge, np.float32(np.inf))
    pts[2::3, :3] = np.nextafter(edge, np.float32(-np.inf))
    pts[:, 3] = rng.uniform(-1.0, 1.0, pts.shape[0])
    _same_avg(pts, float(leaf))


def test_voxel_grid_int_min(gpu):
    """UTM-sized coordinates at a 2 mm leaf: the index leaves int range and becomes INT_MIN, as on x86."""
    pts = _cloud(100_000, 0.002, seed=5)
    pts[: 50_000, 0] += np.float32(5.0e6)
    pts[50_000:, 1] -= np.float32(5.0e6)
    st = {}
    got = P.approximate_voxel_grid(pts, 0.002, stats=st)
    assert got.tobytes() == PO.approximate_voxel_grid(pts, 0.002).tobytes()
    assert st["out_of_range_points"] == 100_000


@pytest.mark.parametrize("case", ["equal", "two_values", "signed_zeros", "n100", "n1000", "random_1e6"])
def test_equalisation(gpu, case):
    rng = np.random.default_rng(6)
    v = {
        "equal": np.full(5000, 0.3),
        "two_values": rng.choice([0.1, 0.9], 4099),
        "signed_zeros": rng.choice([0.0, -0.0, 1.0, -1.0], 3001),
        "n100": rng.normal(size=100),
        "n1000": np.round(rng.normal(size=1000), 2),
        "random_1e6": rng.normal(size=1_000_000),
    }[case].astype(np.float32)
    got = P.equalize_intensities(v)
    ref = PO.rank_equalize(v)
    assert got.tobytes() == ref.tobytes()
    assert np.array_equal(np.sort(got), np.floor(256.0 * np.arange(v.size) / v.size) / 256.0)


def test_equalisation_k128_in_the_png(gpu):
    v = np.random.default_rng(7).permutation(256).astype(np.float32)
    got = P.equalize_intensities(v)
    assert got[v == 128.0][0] == 0.5
    assert P.lidar_intensity_png(got)[v == 128.0][0] == 128


def _same_candidates(pts):
    got, uf = P.lidar_fov_candidates(pts)
    ref, ruf = PO.voxel_grid_fov(pts)
    assert uf == ruf and got.tobytes() == ref.tobytes()
    return got, uf


def test_fov_grid_random(gpu):
    rng = np.random.default_rng(8)
    pts = (S.lidar_directions("avia", 500_000, rng) * rng.uniform(0.5, 40.0, (500_000, 1))).astype(np.float32)
    got, uf = _same_candidates(pts)
    assert not uf and 0 < got.shape[0] < pts.shape[0]


def test_fov_grid_both_sides_of_the_int32_fallback(gpu):
    rng = np.random.default_rng(9)
    pts = rng.uniform(2.0, 50.0, (20_000, 3)).astype(np.float32)
    # 1289 x 1289 x 1289 voxels fit int32, 1291^3 do not (extent = (dx - 1) * 0.2 m along each axis)
    for span, want in ((1288 * 0.2, False), (1291 * 0.2, True)):
        p = pts.copy()
        p[0] = [2.0, 2.0, 2.0]
        p[1] = np.float32(2.0 + span)
        _, uf = _same_candidates(p)
        assert uf == want


def test_fov_norm_filter_edges(gpu):
    one = np.float32(1.0)
    below, above = np.nextafter(one, np.float32(0)), np.nextafter(one, np.float32(2))
    pts = np.array([[one, 0, 0], [0, below, 0], [0, 0, above], [-one, 0, 0], [0, -below, 0], [0, 0, -above], [5, 5, 5]], np.float32)
    got, _ = _same_candidates(pts)
    assert {tuple(p) for p in got.tolist()} == {(1.0, 0.0, 0.0), (0.0, 0.0, float(above)), (-1.0, 0.0, 0.0), (0.0, 0.0, -float(above)), (5.0, 5.0, 5.0)}


@pytest.mark.parametrize("m", [2, 3, 127, 128, 129, 257, 3000])
def test_min_bearing_cosine(gpu, m):
    v = np.random.default_rng(m).normal(size=(m, 3)).astype(np.float32)
    assert P.min_bearing_cosine(v) == PO.min_bearing_cosine(v)


@pytest.mark.parametrize("pattern,wide", [("frustum", False), ("sphere", True)])
def test_lidar_fov_both_sides_of_150_degrees(gpu, pattern, wide):
    rng = np.random.default_rng(10)
    pts = (S.lidar_directions(pattern, 300_000, rng) * rng.uniform(2.0, 30.0, (300_000, 1))).astype(np.float32)
    fov = P.estimate_lidar_fov(pts)
    cand, _ = PO.voxel_grid_fov(pts)
    assert fov == math.acos(PO.min_bearing_cosine(P.hull_vertices(cand)))
    assert (fov >= 150.0 * math.pi / 180.0) == wide
    model, intr, _, _ = P.virtual_lidar_camera(fov)
    if not wide:
        assert model == "plumb_bob" and intr[0] == 1024 / (2.0 * math.tan(fov / 2.0)) == intr[1]
    else:
        assert model == "equirectangular"


def test_refusals(gpu):
    pts = _cloud(1000, 0.05, seed=11)
    for col in range(4):
        bad = pts.copy()
        bad[17, col] = np.nan
        with pytest.raises(gpu.VlcalError, match="non-finite") as e:
            P.approximate_voxel_grid(bad, 0.05)
        assert e.value.code == -1
    for leaf in (0.0, -1.0, 1e-45):
        with pytest.raises(gpu.VlcalError, match="leaf size") as e:
            P.approximate_voxel_grid(pts, leaf)
        assert e.value.code == -1
    with pytest.raises(gpu.VlcalError, match="non-finite") as e:
        P.equalize_intensities(np.array([1.0, np.inf, 0.0], np.float32))
    assert e.value.code == -1
    bad = pts[:, :3].copy()
    bad[3, 2] = -np.inf
    with pytest.raises(gpu.VlcalError, match="non-finite") as e:
        P.lidar_fov_candidates(bad)
    assert e.value.code == -1
    with pytest.raises(ValueError, match="at least 4"):
        P.estimate_lidar_fov(np.zeros((10, 3), np.float32))


# ---- end to end ------------------------------------------------------------------------------------------------

INTR, DIST = "400,400,320,240", "-0.04,0.08,0.0001,-0.0003,-0.04"


def _write_map(dirpath, pattern, n):
    bag = S.make_bag("pinhole_640x480", pattern, n, config_index=9)
    rng = np.random.default_rng(12)
    cloud = np.empty((n, 4), np.float32)
    cloud[:, :3] = bag["points"][:, :3]
    cloud[:, 3] = (bag["intensities"] * 200.0 + rng.normal(0.0, 3.0, n)).astype(np.float32)  # raw, not yet equalised
    map_path = os.path.join(dirpath, "map.ply")
    vio.save_ply_binary(map_path, cloud[:, :3], cloud[:, 3])
    image_path = os.path.join(dirpath, "image.png")
    cv2.imwrite(image_path, bag["image"])
    return bag, cloud, map_path, image_path


def _run_cli(map_path, image_path, dst):
    from direct_visual_lidar_calibration_b200 import preprocess_map as cli

    return cli.main(["--map_path", map_path, "--image_path", image_path, "--dst_path", dst, "--camera_model", "plumb_bob",
                     "--camera_intrinsics", INTR, f"--camera_distortion_coeffs={DIST}"])  # '=': the value starts with '-' 


@pytest.mark.parametrize("pattern,model", [("frustum", "plumb_bob"), ("sphere", "equirectangular")])
def test_cli_matches_the_cpu_pipeline(gpu, oracle, tmp_path, capsys, pattern, model):
    bag, cloud, map_path, image_path = _write_map(str(tmp_path), pattern, 1_000_000)
    dst, ref_dst = str(tmp_path / "out"), str(tmp_path / "ref")
    assert _run_cli(map_path, image_path, dst) == 0
    out = capsys.readouterr().out
    assert "map_points=1000000 filtered=" in out and "LiDAR FoV: " in out
    ref = PO.preprocess_map_cpu(oracle, vio.load_map_cloud(map_path), image_path, ref_dst, map_path, "plumb_bob",
                                [float(v) for v in INTR.split(",")], [float(v) for v in DIST.split(",")])
    assert ref["model"] == model
    for name in ("000000.png", "000000_lidar_intensities.png"):
        a, b = cv2.imread(os.path.join(dst, name), cv2.IMREAD_UNCHANGED), cv2.imread(os.path.join(ref_dst, name), cv2.IMREAD_UNCHANGED)
        assert a.shape == b.shape and np.array_equal(a, b), name
    assert np.array_equal(vio.load_lidar_indices(os.path.join(dst, "000000_lidar_indices.png")), vio.load_lidar_indices(os.path.join(ref_dst, "000000_lidar_indices.png")))
    pa, ia = vio.load_ply(os.path.join(dst, "000000.ply"))
    pb, ib = vio.load_ply(os.path.join(ref_dst, "000000.ply"))
    assert pa.tobytes() == pb.tobytes() and ia.tobytes() == ib.tobytes()
    with open(os.path.join(dst, "calib.json")) as f, open(os.path.join(ref_dst, "calib.json")) as g:
        assert json.load(f) == json.load(g)
    idx = vio.load_lidar_indices(os.path.join(dst, "000000_lidar_indices.png"))
    assert (idx >= 0).sum() > 50_000 and idx.max() < pa.shape[0]


def _write_matches(dst, bag, n_matches=300, outlier_fraction=0.25, seed=13):
    """<bag>_matches.json from the written LiDAR index image, as synthetic.write_initial_guess_dataset makes them."""
    rng = np.random.default_rng(seed)
    index_image = vio.load_lidar_indices(os.path.join(dst, "000000_lidar_indices.png"))
    pts, _ = vio.load_ply(os.path.join(dst, "000000.ply"))
    from direct_visual_lidar_calibration_b200.camera import create_camera

    proj = create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    ys, xs = np.nonzero(index_image >= 0)
    pick = rng.permutation(xs.size)[: 4 * n_matches]
    xs, ys = xs[pick], ys[pick]
    pc = pts[index_image[ys, xs]] @ bag["T_gt"][:3, :3].T + bag["T_gt"][:3, 3]
    uv = proj.project(pc)
    ok = (pc[:, 2] > 0.1) & (uv[:, 0] >= 0) & (uv[:, 0] < bag["width"]) & (uv[:, 1] >= 0) & (uv[:, 1] < bag["height"])
    xs, ys, uv = xs[ok][:n_matches], ys[ok][:n_matches], uv[ok][:n_matches]
    n = xs.size
    n_out = int(round(outlier_fraction * n))
    uv[:n_out] = rng.uniform([0.0, 0.0], [bag["width"], bag["height"]], (n_out, 2))
    kpts1 = np.stack([xs, ys], axis=1) + rng.uniform(0.0, 0.999, (n, 2))
    with open(os.path.join(dst, "000000_matches.json"), "w") as f:
        json.dump({"kpts0": uv.reshape(-1).tolist(), "kpts1": kpts1.reshape(-1).tolist(), "matches": list(range(n)), "confidence": [1.0] * n}, f)
    return n


def _angle_deg(A, B):
    c = (np.trace(A[:3, :3].T @ B[:3, :3]) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))


def test_dataset_runs_through_initial_guess_and_calibrate(gpu, oracle, tmp_path):
    from direct_visual_lidar_calibration_b200 import calibrate as calib_cli
    from direct_visual_lidar_calibration_b200 import initial_guess_auto as guess_cli

    bag, _, map_path, image_path = _write_map(str(tmp_path), "frustum", 100_000)
    dst = str(tmp_path / "out")
    assert _run_cli(map_path, image_path, dst) == 0
    assert _write_matches(dst, bag) > 200
    assert guess_cli.main([dst]) == 0
    cfg = vio.load_calib_json(dst)
    T_gt = bag["T_gt"]
    T_auto = vio.invert_isometry(vio.tum_to_T(cfg["results"]["init_T_lidar_camera_auto"]))
    assert _angle_deg(T_auto, T_gt) < 0.5
    assert np.linalg.norm(T_auto[:3, 3] - T_gt[:3, 3]) < 0.03

    assert calib_cli.main([dst, "--registration_type", "nid_nelder_mead"]) == 0
    cfg = vio.load_calib_json(dst)
    T = vio.invert_isometry(vio.tum_to_T(cfg["results"]["T_lidar_camera"]))
    pts, inten = vio.load_ply(os.path.join(dst, "000000.ply"))
    image = cv2.imread(os.path.join(dst, "000000.png"), 0)
    ocam = oracle.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    xyzw = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1)
    ref = oracle.calibrate(ocam, [(image, xyzw, inten)], T_auto)
    assert np.abs(T - ref["T"]).max() < 1e-9
