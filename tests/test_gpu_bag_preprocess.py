"""GPU checks of `preprocess` from bags: the decode + static integration kernel byte-equal to the sequential checker
(tests/cpp/bag_oracle.c) at its edges, and the CLI end to end on ROS 1 and ROS 2 directories -- every file equal to a CPU
pipeline of the checker, the oracle's generate_lidar_image and cv2, then initial_guess_auto + calibrate on the dataset."""
import json
import math
import os

import cv2
import numpy as np
import pytest

import bag_oracle as BO
import bag_writer as BW
import preprocess_oracle as PO
from direct_visual_lidar_calibration_b200 import _lib as VL
from direct_visual_lidar_calibration_b200 import bag_io as B
from direct_visual_lidar_calibration_b200 import io as vio
from direct_visual_lidar_calibration_b200 import preprocess_bag as PB
from direct_visual_lidar_calibration_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _pack(scans):
    """scans: [(data bytes, {field: (offset, datatype)}, point_step, n)] -> (blob, [ScanDesc])"""
    parts, descs, off = [], [], 0
    for data, f, step, n in scans:
        descs.append(VL.ScanDesc(byte_offset=off, n_points=n, point_step=step, x_offset=f["x"][0], y_offset=f["y"][0], z_offset=f["z"][0],
                                 xyz_type=f["x"][1], intensity_offset=f["intensity"][0], intensity_type=f["intensity"][1]))
        parts.append(np.frombuffer(data, np.uint8))
        off += len(data)
    return (np.concatenate(parts) if parts else np.zeros(0, np.uint8)), descs


def _scan(xyz, inten, xyz_dtype="<f4", inten_dtype="<f4", offsets=None, point_step=None):
    data, fields, step = BW.cloud_bytes(np.asarray(xyz), np.asarray(inten), xyz_dtype, inten_dtype, offsets, point_step)
    return data, {name: (off, dt) for name, off, dt in fields}, step, len(xyz)


def _same(scans, res=0.002, min_distance=1.0):
    blob, descs = _pack(scans)
    st = {}
    got = PB.bag_integrate(blob, descs, res, min_distance, stats=st)
    ref, oor = BO.bag_integrate(blob, descs, res, min_distance)
    assert got.shape == ref.shape and got.tobytes() == ref.tobytes()
    assert st["out_of_range_points"] == oor
    return got


def _cloud(n, rng, span=20.0):
    xyz = rng.uniform(-span, span, (n, 3))
    return xyz, rng.uniform(0.0, 255.0, n)


def test_zero_points(gpu):
    assert _same([]).shape == (0, 4)
    rng = np.random.default_rng(1)
    assert _same([_scan(np.zeros((0, 3)), np.zeros(0)), _scan(np.zeros((0, 3)), np.zeros(0))]).shape == (0, 4)
    xyz, w = _cloud(1000, rng)
    assert _same([_scan(np.zeros((0, 3)), np.zeros(0)), _scan(xyz, w), _scan(np.zeros((0, 3)), np.zeros(0))]).shape[0] > 0


@pytest.mark.parametrize("xyz_dtype", ["<f4", "<f8"])
@pytest.mark.parametrize("inten_dtype", ["u1", "<u2", "<u4", "<f4", "<f8"])
def test_one_scan_every_datatype(gpu, xyz_dtype, inten_dtype):
    rng = np.random.default_rng(2)
    xyz, _ = _cloud(50_000, rng, span=3.0)
    top = {"u1": 255, "<u2": 65535, "<u4": 2**32 - 1}.get(inten_dtype, 1e6)
    w = rng.uniform(0, top, 50_000)
    got = _same([_scan(xyz, w, xyz_dtype, inten_dtype)], res=0.05)
    assert 0 < got.shape[0] < 50_000


def test_ten_thousand_scans_rewrite_the_same_voxels(gpu):
    rng = np.random.default_rng(3)
    base, _ = _cloud(40, rng, span=5.0)
    scans = []
    for k in range(10_000):
        xyz = base + rng.normal(0.0, 0.01, base.shape)  # the same voxels, rewritten by every scan
        scans.append(_scan(xyz, np.full(40, float(k % 251))))
    _same(scans, res=0.1)


def test_different_layouts_unaligned_offsets_and_padding(gpu):
    rng = np.random.default_rng(4)
    scans = []
    for k in range(12):
        xyz, w = _cloud(20_000, rng, span=4.0)
        xdt = "<f4" if k % 2 else "<f8"
        xs = np.dtype(xdt).itemsize
        o = 1 + k % 3 + k // 3
        offsets = {"x": o, "y": o + xs, "z": o + 2 * xs, "intensity": o + 3 * xs + k % 2}  # unaligned offsets
        step = o + 3 * xs + 9 + (k * 7) % 13  # padded point_step
        scans.append(_scan(xyz, w, xdt, ["u1", "<u2", "<u4", "<f4", "<f8"][k % 5], offsets, step))
    _same(scans, res=0.01)


def test_non_finite_and_min_distance_edges(gpu):
    rng = np.random.default_rng(5)
    xyz, w = _cloud(30_000, rng, span=3.0)
    xyz[::7, 0] = np.nan
    xyz[1::11, 1] = np.inf
    xyz[2::13, 2] = -np.inf
    one = 1.0
    d = rng.normal(size=(3000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    edge = np.concatenate([d * one, d * np.nextafter(one, 2.0), d * np.nextafter(one, 0.0)])
    for dt in ("<f8", "<f4"):
        got = _same([_scan(np.concatenate([xyz, edge]), np.concatenate([w, np.arange(edge.shape[0])]), dt)], res=0.001)
        assert np.isfinite(got).all()
    # exactly min_distance +- 1 ulp along an axis (sqrt of the square is exact there)
    ax = np.array([[1.5, 0, 0], [np.nextafter(1.5, 0), 0, 0], [np.nextafter(1.5, 2), 0, 0], [0, -1.5, 0], [0, 0, np.nextafter(-1.5, 0)]])
    got = _same([_scan(ax, np.arange(5.0), "<f8")], res=0.5, min_distance=1.5)
    # 1.5 and its upper neighbour are kept and share voxel (3, 0, 0), where the later one wins; the lower ones are dropped
    assert got[:, 3].tolist() == [2.0, 3.0]


def test_voxel_edges_and_int_min(gpu):
    rng = np.random.default_rng(6)
    res = 0.05
    k = rng.integers(-400, 400, (30_000, 3)).astype(np.float64)
    edge = k * res
    pts = np.concatenate([edge, np.nextafter(edge, np.inf), np.nextafter(edge, -np.inf)])
    pts = pts[np.linalg.norm(pts, axis=1) >= 1.0]
    _same([_scan(pts, rng.uniform(0, 1, pts.shape[0]), "<f8")], res=res)
    far = rng.uniform(-50.0, 50.0, (50_000, 3))
    far[:25_000, 0] += 5.0e6  # beyond int range at 2 mm: INT_MIN along x
    far[25_000:, 2] -= 5.0e7
    far_scan = _scan(far, rng.uniform(0, 1, 50_000), "<f8")
    _same([far_scan], res=0.002)
    assert BO.bag_integrate(*_pack([far_scan]), 0.002, 1.0)[1] == 50_000


@pytest.mark.parametrize("n", [10_000_000, 100_000_000])
def test_large(gpu, n):
    rng = np.random.default_rng(7)
    per = n // 10
    scans = []
    for _ in range(10):
        xyz = rng.uniform(-30.0, 30.0, (per, 3)).astype(np.float32)
        scans.append(_scan(xyz, rng.uniform(0, 100, per).astype(np.float32), "<f4", "<f4"))
        del xyz
    got = _same(scans, res=0.05)
    assert 0 < got.shape[0] < n


# ---- bags through the host loop --------------------------------------------------------------------------------------

def _stamp(k):
    return 100 + k // 10, (k % 10) * 100_000_000


def test_mid_bag_unconvertible_scan_stops_reading(gpu, tmp_path):
    rng = np.random.default_rng(8)
    msgs = []
    for k in range(6):
        xyz, w = _cloud(5000, rng, span=4.0)
        data, fields, step = BW.cloud_bytes(xyz, w, "<f4", "<f4")
        if k == 3:
            fields = [f for f in fields if f[0] != "y"]  # missing y: extract_raw_points returns nullptr
        msgs.append(("/points", "sensor_msgs/PointCloud2", 10**9 * (k + 1), BW.point_cloud2(*_stamp(k), fields, data, 5000, point_step=step)))
    path = str(tmp_path / "a.bag")
    BW.write_ros1(path, msgs)
    logs = []
    blob, descs, st = PB.collect_scans(B.Ros1Bag(path), "a.bag", "/points", "intensity", True, warn=logs.append)
    assert st["scans_integrated"] == 3 and any("scan 3" in m for m in logs)
    got = PB.bag_integrate(blob, descs, 0.01, 1.0)
    ref, _ = BO.bag_integrate(blob, descs, 0.01, 1.0)
    assert got.tobytes() == ref.tobytes()


# ---- end to end ------------------------------------------------------------------------------------------------------

def _write_bags(root, fmt, bag, n_bags=2, scans=10):
    """Two bags of one synthetic scene: CameraInfo, a bgr8 image and `scans` PointCloud2 scans splitting the cloud."""
    os.makedirs(root, exist_ok=True)
    cdr = fmt == "ros2"
    n = bag["points"].shape[0]
    gray = bag["image"]
    K = bag["intrinsics"]
    k9 = [K[0], 0.0, K[2], 0.0, K[1], K[3], 0.0, 0.0, 1.0]
    rng = np.random.default_rng(9)
    for b in range(n_bags):
        big = cdr and b == 1  # the second ROS 2 bag is big-endian CDR
        msgs = [("/camera/camera_info", "sensor_msgs/CameraInfo" if not cdr else "sensor_msgs/msg/CameraInfo", 10**9,
                 BW.camera_info(1, 0, bag["width"], bag["height"], "plumb_bob", bag["distortion"], k9, cdr=cdr, big=big)),
                ("/camera/image", "sensor_msgs/Image" if not cdr else "sensor_msgs/msg/Image", 10**9,
                 BW.image(1, 0, np.repeat(gray[:, :, None], 3, axis=2), "bgr8", cdr=cdr, big=big))]
        inten = (bag["intensities"] * 200.0 + rng.normal(0.0, 3.0, n)).astype(np.float32)
        for k in range(scans):
            sl = slice(k * n // scans, (k + 1) * n // scans)
            data, fields, step = BW.cloud_bytes(bag["points"][sl, :3].astype(np.float32), inten[sl], "<f4", "<f4")
            msgs.append(("/points", "sensor_msgs/PointCloud2" if not cdr else "sensor_msgs/msg/PointCloud2", 10**9 + k * 10**8,
                         BW.point_cloud2(1 + k // 10, (k % 10) * 10**8, fields, data, sl.stop - sl.start, point_step=step, cdr=cdr, big=big)))
        if cdr:
            BW.write_ros2(os.path.join(root, f"bag{b}"), msgs, n_files=2)
        else:
            BW.write_ros1(os.path.join(root, f"bag{b}.bag"), msgs, compression="bz2" if b else "none")


def _cpu_pipeline(oracle, data_path, dst):
    """The dataset from the checker, the product's host readers, scipy's hull, the oracle's renderer and cv2."""
    os.makedirs(dst, exist_ok=True)
    bags = PB.list_bags(data_path)
    clouds = []
    for path in bags:
        bag = B.open_bag(path)
        ros1 = isinstance(bag, B.Ros1Bag)
        name = os.path.basename(path)
        img = PB.first_image(bag, "/camera/image", ros1, name)
        cv2.imwrite(os.path.join(dst, name + ".png"), cv2.equalizeHist(img))
        blob, descs, _ = PB.collect_scans(bag, name, "/points", "intensity", ros1, warn=lambda m: None)
        pts, _ = BO.bag_integrate(blob, descs, 0.002, 1.0)
        inten = PO.rank_equalize(pts[:, 3])
        vio.save_ply_binary(os.path.join(dst, name + ".ply"), pts[:, :3], inten)
        clouds.append((name, pts, inten))
    cand, _ = PO.voxel_grid_fov(clouds[0][1][:, :3])
    from direct_visual_lidar_calibration_b200 import preprocess as P

    fov = math.acos(PO.min_bearing_cosine(P.hull_vertices(cand)))
    wide = not (fov < 150.0 * math.pi / 180.0)
    if wide:
        W, H, model, intr = 1920, 960, "equirectangular", [1920.0, 960.0]
    else:
        W, H = 1024, 1024
        fx = W / (2.0 * math.tan(fov / 2.0))
        model, intr = "plumb_bob", [fx, fx, W / 2.0, H / 2.0]
    R = PO.virtual_lidar_rotation(wide)
    T = np.eye(4)
    T[:3, :3] = R.T
    for i in range(3):
        T[i, 3] = -((R[0, i] * 0.0 + R[1, i] * 0.0) + R[2, i] * 0.0)
    cam = oracle.create_camera(model, intr, [])
    for name, pts, inten in clouds:
        xyzw = np.concatenate([pts[:, :3].astype(np.float64), np.ones((pts.shape[0], 1))], axis=1)
        img, idx = oracle.generate_lidar_image(cam, W, H, T, xyzw, inten)
        cv2.imwrite(os.path.join(dst, name + "_lidar_intensities.png"), np.clip(np.rint(img * 255.0), 0, 255).astype(np.uint8))
        vio.save_lidar_indices(os.path.join(dst, name + "_lidar_indices.png"), idx)
    return [c[0] for c in clouds]


@pytest.mark.parametrize("fmt", ["ros1", "ros2"])
def test_cli_matches_the_cpu_pipeline(gpu, oracle, tmp_path, capsys, fmt):
    from direct_visual_lidar_calibration_b200 import preprocess as cli

    bag = S.make_bag("pinhole_640x480", "frustum", 1_000_000, config_index=9)
    data = str(tmp_path / "bags")
    _write_bags(data, fmt, bag)
    dst, ref_dst = str(tmp_path / "out"), str(tmp_path / "ref")
    assert cli.main([data, dst, "-a"]) == 0
    names = _cpu_pipeline(oracle, data, ref_dst)
    for name in names:
        for suffix in (".png", "_lidar_intensities.png"):
            a = cv2.imread(os.path.join(dst, name + suffix), cv2.IMREAD_UNCHANGED)
            b = cv2.imread(os.path.join(ref_dst, name + suffix), cv2.IMREAD_UNCHANGED)
            assert a.shape == b.shape and np.array_equal(a, b), name + suffix
        assert np.array_equal(vio.load_lidar_indices(os.path.join(dst, name + "_lidar_indices.png")),
                              vio.load_lidar_indices(os.path.join(ref_dst, name + "_lidar_indices.png")))
        pa, ia = vio.load_ply(os.path.join(dst, name + ".ply"))
        pb, ib = vio.load_ply(os.path.join(ref_dst, name + ".ply"))
        assert pa.tobytes() == pb.tobytes() and ia.tobytes() == ib.tobytes()
        assert pa.shape[0] > 100_000
    with open(os.path.join(dst, "calib.json")) as f:
        cfg = json.load(f)
    assert cfg["meta"]["bag_names"] == names and cfg["meta"]["intensity_channel"] == "intensity"
    assert cfg["meta"]["points_topic"] == "/points" and cfg["meta"]["image_topic"] == "/camera/image"
    assert cfg["camera"]["camera_model"] == "plumb_bob"
    K = bag["intrinsics"]
    assert cfg["camera"]["intrinsics"] == [K[0], K[1], K[2], K[3]] and cfg["camera"]["distortion_coeffs"] == list(bag["distortion"])


def test_dataset_runs_through_initial_guess_and_calibrate(gpu, oracle, tmp_path):
    from direct_visual_lidar_calibration_b200 import calibrate as calib_cli
    from direct_visual_lidar_calibration_b200 import initial_guess_auto as guess_cli
    from direct_visual_lidar_calibration_b200 import preprocess as cli
    from direct_visual_lidar_calibration_b200.camera import create_camera

    bag = S.make_bag("pinhole_640x480", "frustum", 200_000, config_index=9)
    data = str(tmp_path / "bags")
    _write_bags(data, "ros1", bag, n_bags=1)
    dst = str(tmp_path / "out")
    assert cli.main([data, dst, "-a"]) == 0
    name = "bag0.bag"
    rng = np.random.default_rng(13)
    index_image = vio.load_lidar_indices(os.path.join(dst, name + "_lidar_indices.png"))
    pts, _ = vio.load_ply(os.path.join(dst, name + ".ply"))
    proj = create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    ys, xs = np.nonzero(index_image >= 0)
    pick = rng.permutation(xs.size)[:1200]
    xs, ys = xs[pick], ys[pick]
    pc = pts[index_image[ys, xs]] @ bag["T_gt"][:3, :3].T + bag["T_gt"][:3, 3]
    uv = proj.project(pc)
    ok = (pc[:, 2] > 0.1) & (uv[:, 0] >= 0) & (uv[:, 0] < bag["width"]) & (uv[:, 1] >= 0) & (uv[:, 1] < bag["height"])
    xs, ys, uv = xs[ok][:300], ys[ok][:300], uv[ok][:300]
    n = xs.size
    assert n > 200
    uv[:75] = rng.uniform([0.0, 0.0], [bag["width"], bag["height"]], (75, 2))
    kpts1 = np.stack([xs, ys], axis=1) + rng.uniform(0.0, 0.999, (n, 2))
    with open(os.path.join(dst, name + "_matches.json"), "w") as f:
        json.dump({"kpts0": uv.reshape(-1).tolist(), "kpts1": kpts1.reshape(-1).tolist(), "matches": list(range(n)), "confidence": [1.0] * n}, f)
    assert guess_cli.main([dst]) == 0
    cfg = vio.load_calib_json(dst)
    T_auto = vio.invert_isometry(vio.tum_to_T(cfg["results"]["init_T_lidar_camera_auto"]))
    T_gt = bag["T_gt"]
    c = (np.trace(T_auto[:3, :3].T @ T_gt[:3, :3]) - 1.0) / 2.0
    assert np.degrees(np.arccos(np.clip(c, -1.0, 1.0))) < 0.5
    assert calib_cli.main([dst, "--registration_type", "nid_nelder_mead"]) == 0
    cfg = vio.load_calib_json(dst)
    T = vio.invert_isometry(vio.tum_to_T(cfg["results"]["T_lidar_camera"]))
    pts, inten = vio.load_ply(os.path.join(dst, name + ".ply"))
    image = cv2.imread(os.path.join(dst, name + ".png"), 0)
    ocam = oracle.create_camera(bag["camera_model"], bag["intrinsics"], bag["distortion"])
    xyzw = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1)
    ref = oracle.calibrate(ocam, [(image, xyzw, inten)], T_auto)
    assert np.abs(T - ref["T"]).max() < 1e-9
