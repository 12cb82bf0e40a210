"""CPU checks of preprocess_map: the sequential checker (tests/cpp/preprocess_oracle.c) against plain Python restatements,
the hull, the virtual-camera rotations against the Eigen stand-in, the map loader's field rules and refusals, and the CLI's
parsing and calib.json."""
import json
import math
import os

import numpy as np
import pytest

import preprocess_oracle as PO
from direct_visual_lidar_calibration_b200 import io as vio
from direct_visual_lidar_calibration_b200 import preprocess as P
from direct_visual_lidar_calibration_b200 import preprocess_map as cli


def _f2i(f):
    return int(f) if -2147483648.0 <= f < 2147483648.0 else -(2**31)


def avg_python(points, leaf):
    """ApproximateVoxelGrid step by step: 512 slots, flush on a key change, the occupied slots flushed in slot order."""
    inv = np.float32(1.0) / np.float32(leaf)
    slots = [None] * 512  # [key, count, centroid float32 (4,)]
    out = []

    def flush(h):
        out.append(h[2] / np.float32(h[1]))

    for p in np.asarray(points, dtype=np.float32):
        key = tuple(_f2i(float(np.floor(p[k] * inv))) for k in range(3))
        slot = (key[0] * 7171 + key[1] * 3079 + key[2] * 4231) & 511
        h = slots[slot]
        if h is not None and h[1] and h[0] != key:
            flush(h)
            h = None
        if h is None or not h[1]:
            h = slots[slot] = [key, 0, np.zeros(4, np.float32)]
        h[1] += 1
        h[2] = h[2] + p
    for h in slots:
        if h is not None and h[1]:
            flush(h)
    return np.array(out, dtype=np.float32).reshape(-1, 4)


def _colliding(n, leaf=1.0):
    """Points alternating between voxels (0,0,0) and (512,0,0), which share slot 0: every point evicts the other voxel."""
    rng = np.random.default_rng(3)
    pts = rng.uniform(0.0, 0.999, (n, 4)).astype(np.float32)
    pts[1::2, 0] += np.float32(512 * leaf)
    return pts


@pytest.mark.parametrize("case", ["random", "colliding", "negative", "one_voxel", "big_coordinates"])
def test_oracle_voxel_grid_is_the_sequential_loop(case):
    rng = np.random.default_rng(hash(case) % 2**32)
    leaf = 0.05
    if case == "random":
        pts = rng.uniform(-1.0, 1.0, (3000, 4)).astype(np.float32)
    elif case == "colliding":
        pts, leaf = _colliding(2001), 1.0
    elif case == "negative":
        pts = rng.uniform(-3.0, -0.01, (2500, 4)).astype(np.float32)
    elif case == "one_voxel":
        pts = rng.uniform(0.0, 0.049, (1000, 4)).astype(np.float32)
    else:  # indices out of int range at a 2 mm leaf: INT_MIN
        pts = rng.uniform(-1.0, 1.0, (800, 4)).astype(np.float32)
        pts[:, 0] += np.float32(5.0e6)
        leaf = 0.002
    ref = avg_python(pts, leaf)
    got = PO.approximate_voxel_grid(pts, leaf)
    assert got.tobytes() == ref.tobytes()
    if case == "colliding":
        assert got.shape[0] == pts.shape[0]  # every point flushed on its own
    if case == "one_voxel":
        assert got.shape[0] == 1


def test_oracle_equalisation_is_the_stable_argsort():
    rng = np.random.default_rng(5)
    for v in [rng.normal(size=1000), np.round(rng.normal(size=777), 1), np.full(300, 0.25), np.array([0.0, -0.0, 1.0, -0.0, 0.0] * 20)]:
        v = v.astype(np.float32)
        order = np.argsort(v.astype(np.float64), kind="stable")
        ref = np.empty(v.size)
        ref[order] = np.floor(256 * np.arange(v.size, dtype=np.float64) / v.size) / 256
        assert PO.rank_equalize(v).tobytes() == ref.tobytes()


def test_hull_vertices_are_extreme_and_the_rest_inside():
    from scipy.spatial import ConvexHull

    rng = np.random.default_rng(7)
    pts = (rng.normal(size=(4000, 3)) * [5.0, 3.0, 2.0]).astype(np.float32)
    verts = P.hull_vertices(pts)
    hull = ConvexHull(pts.astype(np.float64))
    eq = hull.equations  # n . x + d <= 0 inside
    vset = {tuple(v) for v in verts.tolist()}
    tol = 1e-9 * np.abs(pts).max()
    for p in pts.astype(np.float64):
        s = eq[:, :3] @ p + eq[:, 3]
        if tuple(np.float32(p).tolist()) in vset:
            assert np.isclose(s.max(), 0.0, atol=tol)  # on the boundary
        else:
            assert s.max() <= tol
    for v in verts.astype(np.float64):  # extreme: not a convex combination of the others
        others = np.array([w for w in verts.astype(np.float64) if not np.array_equal(w, v)])
        h2 = ConvexHull(others)
        assert (h2.equations[:, :3] @ v + h2.equations[:, 3]).max() > 0.0


def test_hull_refusals():
    rng = np.random.default_rng(8)
    with pytest.raises(ValueError, match="at least 4"):
        P.hull_vertices(rng.normal(size=(3, 3)))
    flat = rng.normal(size=(500, 3))
    flat[:, 2] = 1e-5 * flat[:, 2] + 2.0
    with pytest.raises(ValueError, match="flat"):
        P.hull_vertices(flat)


def test_min_bearing_cosine_checker():
    rng = np.random.default_rng(9)
    v = rng.normal(size=(50, 3)).astype(np.float32)
    d = v.astype(np.float64) / np.linalg.norm(v.astype(np.float64), axis=1, keepdims=True)
    c = d @ d.T
    iu = np.triu_indices(50, 1)
    assert abs(PO.min_bearing_cosine(v) - c[iu].min()) < 1e-15
    assert PO.min_bearing_cosine(v[:1]) == math.pi


def test_virtual_rotations_match_the_eigen_standin():
    q, rot_q, rot_x = PO.standin_rotation_check()
    mine = P._quaternion_product(P._angle_axis_quaternion(math.pi / 2, (0.0, 1.0, 0.0)), P._angle_axis_quaternion(-math.pi / 2, (0.0, 0.0, 1.0)))
    assert [float(v).hex() for v in mine] == [float(v).hex() for v in q]
    for wide, rot in ((False, rot_q), (True, rot_x)):
        R = P.virtual_lidar_rotation(math.radians(170.0) if wide else math.radians(90.0))
        assert R.tobytes() == PO.virtual_lidar_rotation(wide).tobytes()
        assert np.abs(R - rot.T).max() < 1e-15  # columns: the images of the unit vectors
    # the pinhole camera looks along LiDAR +x with image x along -y, the equirectangular one has its y axis along -z
    Rp = P.virtual_lidar_rotation(math.radians(90.0))
    assert np.allclose(Rp, [[0, 0, 1], [-1, 0, 0], [0, -1, 0]], atol=1e-15)
    _, _, _, T = P.virtual_lidar_camera(math.radians(90.0))
    assert np.array_equal(T[:3, :3], Rp.T) and np.all(T[:3, 3] == 0.0)


def test_virtual_camera_intrinsics():
    fov = math.radians(100.0)
    model, intr, size, _ = P.virtual_lidar_camera(fov)
    assert model == "plumb_bob" and size == (1024, 1024) and intr == [1024 / (2.0 * math.tan(fov / 2.0))] * 2 + [512.0, 512.0]
    model, intr, size, _ = P.virtual_lidar_camera(150.0 * math.pi / 180.0)
    assert model == "equirectangular" and size == (1920, 960) and intr == [1920.0, 960.0]


def test_lidar_intensity_png_rounds_half_to_even():
    k = np.arange(256, dtype=np.float64) / 256.0
    png = P.lidar_intensity_png(k)
    assert png[128] == 128  # 0.5 * 255 = 127.5
    assert np.array_equal(png, np.rint(k * 255.0).astype(np.uint8))


# ---- the map loader ---------------------------------------------------------------------------------------------

def _write_pcd(path, fields, data, kind="binary"):
    """fields: [(name, TYPE, SIZE, COUNT)], data: list of per-field (N, COUNT) arrays."""
    n = data[0].shape[0]
    head = ["# .PCD v0.7", "VERSION 0.7", "FIELDS " + " ".join(f[0] for f in fields), "SIZE " + " ".join(str(f[2]) for f in fields),
            "TYPE " + " ".join(f[1] for f in fields), "COUNT " + " ".join(str(f[3]) for f in fields), f"WIDTH {n}", "HEIGHT 1",
            "VIEWPOINT 0 0 0 1 0 0 0", f"POINTS {n}", f"DATA {kind}"]
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        if kind == "ascii":
            rows = np.concatenate([d.astype(np.float64).reshape(n, -1) for d in data], axis=1)
            for r in rows:
                f.write((" ".join(repr(float(v)) for v in r) + "\n").encode())
        elif kind == "binary":
            types = {("F", 4): "<f4", ("F", 8): "<f8", ("U", 1): "u1", ("I", 4): "<i4"}
            dt = np.dtype([(fd[0] + str(i), types[(fd[1], fd[2])], (fd[3],)) for i, fd in enumerate(fields)])
            rec = np.empty(n, dt)
            for i, fd in enumerate(fields):
                rec[fd[0] + str(i)] = data[i].reshape(n, fd[3])
            f.write(rec.tobytes())


def _cloud(n=100, seed=1):
    return np.random.default_rng(seed).uniform(-5, 5, (n, 4)).astype(np.float32)


@pytest.mark.parametrize("kind", ["binary", "ascii"])
def test_load_pcd(tmp_path, kind):
    c = _cloud()
    p = str(tmp_path / "m.pcd")
    fields = [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("rgb", "U", 1, 1), ("intensity", "F", 4, 1), ("n", "F", 4, 3)]
    extra = np.zeros((c.shape[0], 3), np.float32)
    _write_pcd(p, fields, [c[:, 0:1], c[:, 1:2], c[:, 2:3], np.zeros((c.shape[0], 1), np.uint8), c[:, 3:4], extra], kind)
    assert vio.load_map_cloud(p).tobytes() == c.tobytes()


def test_load_pcd_field_rules(tmp_path):
    c = _cloud()
    msgs = []
    p = str(tmp_path / "a.pcd")
    _write_pcd(p, [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("intensity", "F", 8, 1)], [c[:, 0:1], c[:, 1:2], c[:, 2:3], c[:, 3:4].astype(np.float64)])
    got = vio.load_map_cloud(p, warn=msgs.append)
    assert np.array_equal(got[:, :3], c[:, :3]) and np.all(got[:, 3] == 0.0) and "intensity" in msgs[0]
    _write_pcd(p, [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1)], [c[:, 0:1], c[:, 1:2], c[:, 2:3]])
    msgs.clear()
    assert np.all(vio.load_map_cloud(p, warn=msgs.append)[:, 3] == 0.0) and msgs
    _write_pcd(p, [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("intensity", "F", 4, 2)], [c[:, 0:1], c[:, 1:2], c[:, 2:3], np.repeat(c[:, 3:4], 2, 1)])
    msgs.clear()
    assert np.all(vio.load_map_cloud(p, warn=msgs.append)[:, 3] == 0.0) and msgs  # count 2 does not match
    _write_pcd(p, [("x", "F", 8, 1), ("y", "F", 4, 1), ("z", "F", 4, 1)], [c[:, 0:1].astype(np.float64), c[:, 1:2], c[:, 2:3]])
    with pytest.raises(ValueError, match="field x must be float32"):
        vio.load_map_cloud(p)
    _write_pcd(p, [("y", "F", 4, 1), ("z", "F", 4, 1)], [c[:, 1:2], c[:, 2:3]])
    with pytest.raises(ValueError, match="field x"):
        vio.load_map_cloud(p)


def test_load_refusals(tmp_path):
    c = _cloud()
    p = str(tmp_path / "m.pcd")
    fields = [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("intensity", "F", 4, 1)]
    for bad in (np.nan, np.inf):
        d = c.copy()
        d[7, 1] = bad
        _write_pcd(p, fields, [d[:, k : k + 1] for k in range(4)])
        with pytest.raises(ValueError, match="non-finite"):
            vio.load_map_cloud(p)
    d = c.copy()
    d[3, 3] = np.nan
    _write_pcd(p, fields, [d[:, k : k + 1] for k in range(4)], "ascii")
    with pytest.raises(ValueError, match="non-finite"):
        vio.load_map_cloud(p)
    _write_pcd(p, fields, [c[:, k : k + 1] for k in range(4)], "binary_compressed")
    with pytest.raises(ValueError, match="binary_compressed"):
        vio.load_map_cloud(p)
    with pytest.raises(ValueError, match="unsupported map format"):
        vio.load_map_cloud(str(tmp_path / "m.obj"))


def test_load_ply(tmp_path):
    c = _cloud()
    p = str(tmp_path / "m.ply")
    vio.save_ply_binary(p, c[:, :3], c[:, 3])
    assert vio.load_map_cloud(p).tobytes() == c.tobytes()
    with open(p, "w") as f:  # ascii, double coordinates: refused
        f.write(f"ply\nformat ascii 1.0\nelement vertex {c.shape[0]}\nproperty double x\nproperty double y\nproperty double z\nend_header\n")
        for r in c:
            f.write(f"{float(r[0])!r} {float(r[1])!r} {float(r[2])!r}\n")
    with pytest.raises(ValueError, match="field x must be float32"):
        vio.load_map_cloud(p)
    with open(p, "w") as f:  # ascii floats, uchar intensity: zeros with a warning
        f.write(f"ply\nformat ascii 1.0\nelement vertex {c.shape[0]}\nproperty float x\nproperty float y\nproperty float z\nproperty uchar intensity\nend_header\n")
        for r in c:
            f.write(f"{float(r[0])!r} {float(r[1])!r} {float(r[2])!r} 7\n")
    msgs = []
    got = vio.load_map_cloud(p, warn=msgs.append)
    assert np.array_equal(got[:, :3], c[:, :3]) and np.all(got[:, 3] == 0) and msgs


# ---- the CLI ----------------------------------------------------------------------------------------------------

def test_cli_missing_flags_print_the_usage(capsys):
    assert cli.main(["--map_path", "m.pcd"]) == 0
    assert "usage: preprocess_map" in capsys.readouterr().out


def test_cli_flags_keep_the_reference_names_and_defaults():
    a = cli.build_parser().parse_args(["--map_path", "m", "--image_path", "i", "--dst_path", "d", "--camera_model", "plumb_bob",
                                       "--camera_intrinsics", "1,2,3,4", "--camera_distortion_coeffs", "0,0,0,0,0"])
    assert a.voxel_resolution == 0.002 and a.min_distance is None and a.device == -1
    assert P.parse_values("810.5,810.25,320,240", "camera_intrinsics") == [810.5, 810.25, 320.0, 240.0]
    with pytest.raises(ValueError, match="camera_distortion_coeffs"):
        P.parse_values("0,,0", "camera_distortion_coeffs")


def test_cli_bad_values_fail_cleanly(tmp_path, capsys):
    rc = cli.main(["--map_path", "m.pcd", "--image_path", str(tmp_path / "none.png"), "--dst_path", str(tmp_path / "d"), "--camera_model", "plumb_bob",
                   "--camera_intrinsics", "1,2,x", "--camera_distortion_coeffs", "0", "--min_distance", "2.0"])
    cap = capsys.readouterr()
    assert rc == 1 and "camera_intrinsics" in cap.err and "--min_distance has no effect" in cap.out


def test_calib_json_content():
    cfg = P.calib_config("/maps/a.pcd", "plumb_bob", [1.0, 2.0, 3.0, 4.0], [0.1, 0.0, 0.0, 0.0, 0.0])
    text = json.dumps(cfg, indent=2, sort_keys=True)
    assert json.loads(text) == {
        "camera": {"camera_model": "plumb_bob", "distortion_coeffs": [0.1, 0.0, 0.0, 0.0, 0.0], "intrinsics": [1.0, 2.0, 3.0, 4.0]},
        "meta": {"bag_names": ["000000"], "camera_info_topic": "N/A", "data_path": "/maps/a.pcd", "image_topic": "N/A", "intensity_channel": "N/A", "points_topic": "N/A"},
    }
    assert text.index('"camera"') < text.index('"meta"') and text.index('"camera_info_topic"') < text.index('"data_path"')
