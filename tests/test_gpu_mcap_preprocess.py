"""`preprocess` on compressed bags, end to end on the GPU: the same seeded scans, image and camera info written as a
sqlite3 bag (the path tests/test_gpu_bag_preprocess.py checks against the CPU pipeline), as rosbag2 MCAP with
uncompressed, zstd, lz4 and mixed chunks over two files, as sqlite3 with per-message zstd, and as a ROS 1 bag with lz4
chunks next to the same bag uncompressed.  Every dataset must be byte-identical to that of its reference form: every
PNG, every PLY and calib.json.  The committed zstd MCAP bag (tests/golden/mcap_bag) runs through preprocess and
initial_guess_search, so that path is covered where libzstd is absent."""
import os
import shutil

import numpy as np
import pytest

import bag_writer as BW
import codec_data as CD
import mcap_writer as MW
from direct_visual_lidar_calibration_b200 import preprocess as cli
from direct_visual_lidar_calibration_b200 import synthetic as S

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
needs_libs = pytest.mark.skipif(not (CD.have_zstd() and CD.have_lz4()), reason="libzstd / liblz4 not available to write the bags")


def _messages(cdr, scans=12):
    bag = S.make_bag("pinhole_640x480", "frustum", 300_000, config_index=9)
    K = bag["intrinsics"]
    k9 = [K[0], 0.0, K[2], 0.0, K[1], K[3], 0.0, 0.0, 1.0]
    typ = (lambda t: "sensor_msgs/msg/" + t) if cdr else (lambda t: "sensor_msgs/" + t)
    msgs = [("/camera/camera_info", typ("CameraInfo"), 10**9, BW.camera_info(1, 0, bag["width"], bag["height"], "plumb_bob", bag["distortion"], k9, cdr=cdr)),
            ("/camera/image", typ("Image"), 10**9, BW.image(1, 0, np.repeat(bag["image"][:, :, None], 3, axis=2), "bgr8", cdr=cdr))]
    rng = np.random.default_rng(31)
    n = bag["points"].shape[0]
    inten = (bag["intensities"] * 200.0 + rng.normal(0.0, 3.0, n)).astype(np.float32)
    for k in range(scans):
        sl = slice(k * n // scans, (k + 1) * n // scans)
        data, fields, step = BW.cloud_bytes(bag["points"][sl, :3].astype(np.float32), inten[sl], "<f4", "<f4")
        msgs.append(("/points", typ("PointCloud2"), 10**9 + k * 10**8,
                     BW.point_cloud2(1 + k // 10, (k % 10) * 10**8, fields, data, sl.stop - sl.start, point_step=step, cdr=cdr)))
    return msgs


def _dataset(root, write=None, name="bag0"):
    """preprocess on root (after emptying it and writing root/name with `write`); calib.json records root, so every form
    of a comparison is written to the same root in turn"""
    if write is not None:
        shutil.rmtree(root, ignore_errors=True)
        os.makedirs(root)
        write(os.path.join(root, name))
    dst = root + "_out"
    shutil.rmtree(dst, ignore_errors=True)
    assert cli.main([root, dst, "-a"]) == 0
    files = sorted(os.listdir(dst))
    assert "calib.json" in files and any(f.endswith(".ply") for f in files) and any(f.endswith("_lidar_indices.png") for f in files)
    out = {}
    for fn in files:
        with open(os.path.join(dst, fn), "rb") as f:
            out[fn] = f.read()
    return out


@needs_libs
def test_ros2_forms_give_the_sqlite3_dataset(gpu, tmp_path):
    msgs = _messages(cdr=True)
    forms = {
        "sqlite3": lambda d: BW.write_ros2(d, msgs, n_files=2),
        "mcap_none": lambda d: MW.write_ros2_mcap(d, msgs, n_files=2, compressions=("",), per_chunk=3),
        "mcap_zstd": lambda d: MW.write_ros2_mcap(d, msgs, n_files=2, compressions=("zstd",), per_chunk=3),
        "mcap_lz4": lambda d: MW.write_ros2_mcap(d, msgs, n_files=2, compressions=("lz4",), per_chunk=3),
        "mcap_mixed": lambda d: MW.write_ros2_mcap(d, msgs, n_files=2, compressions=("zstd", "", "lz4"), per_chunk=2, unchunked={1, 6}),
        "sqlite3_message_zstd": lambda d: MW.write_ros2_message_zstd(d, msgs, n_files=2),
    }
    sets = {name: _dataset(str(tmp_path / "bags"), write) for name, write in forms.items()}
    ref = sets.pop("sqlite3")
    for name, got in sets.items():
        assert sorted(got) == sorted(ref), name
        for fn in ref:
            assert got[fn] == ref[fn], (name, fn)


@needs_libs
@pytest.mark.parametrize("independent", [False, True])
def test_ros1_lz4_gives_the_uncompressed_dataset(gpu, tmp_path, independent):
    msgs = _messages(cdr=False)
    root = str(tmp_path / "bags")
    ref = _dataset(root, lambda p: BW.write_ros1(p, msgs), "bag0.bag")
    got = _dataset(root, lambda p: MW.write_ros1_lz4(p, msgs, independent=independent, block_checksum=True, content_checksum=True), "bag0.bag")
    assert sorted(got) == sorted(ref)
    for fn in ref:
        assert got[fn] == ref[fn], fn


def test_committed_mcap_bag_through_preprocess_and_initial_guess_search(gpu, tmp_path):
    from direct_visual_lidar_calibration_b200 import bag_io as B
    from direct_visual_lidar_calibration_b200 import initial_guess_search as igs

    root = str(tmp_path / "bags")
    shutil.copytree(os.path.join(GOLDEN, "mcap_bag"), os.path.join(root, "mcap_bag"))
    bag = B.Ros2Bag(os.path.join(root, "mcap_bag"))
    assert bag.storage == "mcap" and ("/points", "sensor_msgs/msg/PointCloud2") in bag.topics_and_types()
    with open(bag.files[0], "rb") as f:
        assert b"zstd" in f.read()
    ds = _dataset(root)
    assert len(ds["mcap_bag.ply"]) > 50_000
    assert igs.main([root + "_out", "--rot_step_deg", "6", "--keep", "16"]) == 0
    assert os.path.exists(os.path.join(root + "_out", "initial_guess_search.json"))
