"""Host checks of `preprocess` from bags (no GPU): the ROS 1 / ROS 2 readers against bags written from the format specs
(tests/bag_writer.py), the message decoders, every refusal, topic / channel / camera selection, the TimeKeeper
restatement and the checker's field extraction."""
import numpy as np
import pytest

import bag_oracle as BO
import bag_writer as BW
from direct_visual_lidar_calibration_b200 import _lib as VL
from direct_visual_lidar_calibration_b200 import bag_io as B
from direct_visual_lidar_calibration_b200 import preprocess as cli
from direct_visual_lidar_calibration_b200 import preprocess_bag as PB


def _cloud_msg(k, n=4, cdr=False, big=False, xyz_dtype="<f4", inten_dtype="<f4", **kw):
    xyz = np.arange(3 * n, dtype=np.float64).reshape(n, 3) + k
    data, fields, step = BW.cloud_bytes(xyz, np.full(n, float(k)), xyz_dtype, inten_dtype)
    return BW.point_cloud2(k, 500, fields, data, n, point_step=step, cdr=cdr, big=big, **kw)


def _interleaved(cdr):
    t = "sensor_msgs/msg/" if cdr else "sensor_msgs/"
    msgs = []
    # receive times out of file order, with ties between topics and within a topic
    for k, ns in enumerate([5, 3, 3, 9, 1, 3, 7, 7]):
        msgs.append(("/points", t + "PointCloud2", ns, _cloud_msg(k, cdr=cdr)))
        msgs.append(("/image", t + "Image", ns, BW.image(k, 0, np.full((2, 3), k, np.uint8), "mono8", cdr=cdr)))
    return msgs


@pytest.mark.parametrize("compression", ["none", "bz2"])
def test_ros1_order_and_values(tmp_path, compression):
    path = str(tmp_path / "a.bag")
    BW.write_ros1(path, _interleaved(False), compression=compression, per_chunk=3)
    bag = B.Ros1Bag(path)
    assert bag.topics_and_types() == [("/points", "sensor_msgs/PointCloud2"), ("/image", "sensor_msgs/Image")]
    got = [B.decode_point_cloud2(raw, cdr=False)["stamp"] for _, raw in bag.messages("/points")]
    order = sorted(range(8), key=lambda k: ([5, 3, 3, 9, 1, 3, 7, 7][k], k))  # time, then file position
    assert got == [float(k) + 1e-9 * 500.0 for k in order]
    imgs = [B.image_to_mono8(B.decode_image(raw, cdr=False)) for _, raw in bag.messages("/image")]
    assert [int(i[0, 0]) for i in imgs] == order


@pytest.mark.parametrize("big", [False, True])
def test_ros2_order_values_and_files(tmp_path, big):
    msgs = [(t, typ, ns, _cloud_msg(k, cdr=True, big=big) if "Point" in typ else BW.image(k, 0, np.full((2, 3), k, np.uint8), "mono8", cdr=True, big=big))
            for k, (t, typ, ns, _) in enumerate(_interleaved(True))]
    path = str(tmp_path / "b2")
    BW.write_ros2(path, msgs, n_files=3)
    bag = B.Ros2Bag(path)
    assert len(bag.files) == 3
    got = [B.decode_point_cloud2(raw, cdr=True) for _, raw in bag.messages("/points")]
    per = -(-len(msgs) // 3)
    want = []
    for f in range(3):  # file by file, then timestamp, then id
        part = [(ns, i, m) for i, m in enumerate(msgs[f * per:(f + 1) * per]) for ns in [m[2]] if m[0] == "/points"]
        want += [B.decode_point_cloud2(m[3], cdr=True)["stamp"] for ns, i, m in sorted(part, key=lambda e: (e[0], e[1]))]
    assert [g["stamp"] for g in got] == want
    g = got[0]
    assert g["width"] == 4 and g["point_step"] == 16 and [f[0] for f in g["fields"]] == ["x", "y", "z", "intensity"]


def test_decoders_both_serialisations():
    for cdr, big in ((False, False), (True, False), (True, True)):
        ci = B.decode_camera_info(BW.camera_info(3, 7, 640, 480, "plumb_bob", [0.1, -0.2, 0.0, 0.001, 0.05], [400.0, 0, 320.0, 0, 410.0, 240.0, 0, 0, 1.0],
                                                 cdr=cdr, big=big), cdr=cdr)
        assert ci["distortion_model"] == "plumb_bob" and ci["d"] == [0.1, -0.2, 0.0, 0.001, 0.05]
        assert (ci["k"][0], ci["k"][4], ci["k"][2], ci["k"][5]) == (400.0, 410.0, 320.0, 240.0) and (ci["width"], ci["height"]) == (640, 480)
        rgb = np.random.default_rng(1).integers(0, 255, (5, 7, 3)).astype(np.uint8)
        for enc in ("bgr8", "rgb8"):
            m = B.decode_image(BW.image(1, 2, rgb, enc, cdr=cdr, big=big, pad=3), cdr=cdr)
            import cv2

            want = cv2.cvtColor(rgb, cv2.COLOR_BGR2GRAY if enc == "bgr8" else cv2.COLOR_RGB2GRAY)
            assert np.array_equal(B.image_to_mono8(m), want)
        import cv2

        ok, png = cv2.imencode(".png", rgb)
        m = B.decode_compressed_image(BW.compressed_image(1, 2, "bgr8; png compressed", png.tobytes(), cdr=cdr, big=big), cdr=cdr)
        assert np.array_equal(B.compressed_to_mono8(m), cv2.cvtColor(rgb, cv2.COLOR_BGR2GRAY))
    ros2 = B.decode_point_cloud2(_cloud_msg(0, cdr=True), cdr=True)["stamp"]
    assert ros2 == 0 + 500 / 1e9


def test_refusals(tmp_path, capsys):
    BW.write_ros1(str(tmp_path / "l.bag"), [("/p", "sensor_msgs/PointCloud2", 1, _cloud_msg(0))], compression="lz4")
    with pytest.raises(B.BagError, match=r"l\.bag.*lz4.*rosbag decompress"):
        B.Ros1Bag(str(tmp_path / "l.bag"))
    BW.write_ros2(str(tmp_path / "m"), [("/p", "sensor_msgs/msg/PointCloud2", 1, _cloud_msg(0, cdr=True))], storage="mcap")
    with pytest.raises(B.BagError, match="zstd.*ros2 bag convert"):
        B.Ros2Bag(str(tmp_path / "m"))
    with pytest.raises(B.BagError, match="encoding 'yuv422'"):
        B.image_to_mono8({"encoding": "yuv422", "height": 1, "width": 1, "step": 2, "data": b"\0\0"})
    # big-endian cloud, a points topic without the intensity channel
    for kw, match in (({"is_bigendian": True}, "big-endian"), ({}, "no 'reflectivity' field")):
        path = str(tmp_path / "e.bag")
        BW.write_ros1(path, [("/p", "sensor_msgs/PointCloud2", 1, _cloud_msg(0, **kw))])
        with pytest.raises(B.BagError, match=r"e\.bag: scan 0.*" + match):
            PB.collect_scans(B.Ros1Bag(path), "e.bag", "/p", "reflectivity" if not kw else "intensity", True, warn=lambda m: None)
    # no image
    d = tmp_path / "noimg"
    d.mkdir()
    BW.write_ros1(str(d / "x.bag"), [("/p", "sensor_msgs/PointCloud2", 1, _cloud_msg(0))])
    assert cli.main([str(d), str(tmp_path / "o"), "--points_topic", "/p", "--image_topic", "/img"]) == 1
    assert "x.bag: no image message on topic '/img'" in capsys.readouterr().err
    assert cli.main([str(d), str(tmp_path / "o"), "-d"]) == 1
    assert "error: x.bag: dynamic LiDAR integration (-d" in capsys.readouterr().err
    assert cli.main([str(d), str(tmp_path / "o"), "-v", "--points_topic", "/p", "--image_topic", "/img"]) == 1
    assert "note: there is no viewer (-v)" in capsys.readouterr().out
    assert cli.main([]) == 0
    # 16-bit compressed images are refused (cv_bridge would go through mono16)
    import cv2

    ok, png16 = cv2.imencode(".png", np.full((4, 5), 40000, np.uint16))
    with pytest.raises(B.BagError, match="only 8-bit compressed"):
        B.compressed_to_mono8(B.decode_compressed_image(BW.compressed_image(1, 2, "mono16; png compressed", png16.tobytes()), cdr=False))


def _layout(fields, width=1, height=1, channel="intensity"):
    return PB.scan_layout({"fields": [(n, o, t, 1) for n, o, t in fields], "width": width, "height": height}, channel)


def test_scan_layout_quirks():
    fields = [("x", 0, 7), ("y", 4, 7), ("z", 8, 8), ("intensity", 16, 2)]
    n, offs, xt, tf, inten = _layout(fields, 3, 2)
    assert n == 6 and offs == (0, 4, 8) and xt == 7 and inten == (16, 2) and tf == (-1, 0)  # z read as float32, x's type
    for bad in ([("x", 0, 7), ("y", 4, 8), ("z", 8, 7)], [("x", 0, 7), ("z", 8, 7)], [("x", 0, 2), ("y", 1, 2), ("z", 2, 2)]):
        with pytest.raises(PB.Unconvertible):
            _layout(bad)
    with pytest.raises(PB.Unconvertible, match="intensity"):
        _layout(fields[:3] + [("intensity", 16, 5)])
    _layout(fields[:3] + [("intensity", 16, 5)], 0)  # 0 points: never read
    with pytest.raises(PB.Unconvertible, match="missing"):  # -i x: the "x" field fills the intensity, x stays unset
        _layout(fields, channel="x")
    _, _, _, tf, _ = _layout(fields + [("t", 20, 6), ("timestamp", 24, 8)])
    assert tf == (24, 8)  # the last time field in the message wins


def test_checker_extraction_every_datatype():
    rng = np.random.default_rng(2)
    for xdt in ("<f4", "<f8"):
        for idt in ("u1", "<u2", "<u4", "<f4", "<f8"):
            xyz = rng.normal(size=(100, 3)) * 10
            w = rng.uniform(0, 200, 100)
            xs = np.dtype(xdt).itemsize
            offsets = {"x": 3, "y": 3 + xs, "z": 3 + 2 * xs, "intensity": 3 + 3 * xs}  # unaligned
            data, fields, step = BW.cloud_bytes(xyz, w, xdt, idt, offsets, point_step=41)
            f = {n: (o, t) for n, o, t in fields}
            d = VL.ScanDesc(byte_offset=0, n_points=100, point_step=step, x_offset=f["x"][0], y_offset=f["y"][0], z_offset=f["z"][0], xyz_type=f["x"][1],
                            intensity_offset=f["intensity"][0], intensity_type=f["intensity"][1])
            got = BO.extract_scan(np.frombuffer(data, np.uint8), d)
            assert np.array_equal(got[:, :3], xyz.astype(xdt).astype(np.float64))
            assert np.array_equal(got[:, 3], w.astype(idt).astype(np.float64))


def test_topic_channel_and_camera_selection():
    tt = [("/a/info", "sensor_msgs/CameraInfo"), ("/a/img", "sensor_msgs/CompressedImage"), ("/lidar", "sensor_msgs/PointCloud2"),
          ("/b/img", "sensor_msgs/Image")]
    logs = []
    assert PB.get_topics(tt, True, warn=logs.append) == ("/a/info", "/b/img", "/lidar") and len(logs) == 1
    assert PB.get_topics(tt, False, "/c", "/i", "/p") == ("/c", "/i", "/p")
    assert PB.get_topics(tt[:1], True, "/c", "/i", "/p") == ("/a/info", "/i", "/p")
    assert PB.get_intensity_channel(["x", "y", "z", "intensity", "reflectivity"]) == "reflectivity"
    assert PB.get_intensity_channel(["x", "reflectivity", "intensity"]) == "reflectivity"
    assert PB.get_intensity_channel(["x", "intensity"]) == "intensity"
    assert PB.get_intensity_channel(["x", "y"]) == "auto"
    assert PB.get_intensity_channel(["x", "y"], "ambient") == "ambient"
    assert PB.camera_params(None, True, "b", "", (640, 480), "equirectangular") == ("equirectangular", [640.0, 480.0], [])
    assert PB.camera_params(None, True, "b", "", (640, 480), "fisheye", "1,2,3,4", "0.1,0.2") == ("fisheye", [1.0, 2.0, 3.0, 4.0], [0.1, 0.2])
    for bad in ("atan", "rational_polynomial"):
        with pytest.raises(ValueError, match="invalid camera model"):
            PB.camera_params(None, True, "b", "", (640, 480), bad, "1,2,3,4", "0")


def test_time_keeper():
    tk = PB.TimeKeeper()
    # no per-point times: the frame stamp decides, a rewind is skipped
    assert [tk.process(s) for s in (10.0, 10.1, 10.05, 10.2, 10.2)] == [True, True, False, True, True]
    # relative times (< 1): the stamp is kept
    tk = PB.TimeKeeper()
    assert [tk.process(s, (0.0, 0.09, 0.0)) for s in (5.0, 4.0, 6.0)] == [True, False, True]
    # absolute times close to the stamp: the first point time replaces it
    tk = PB.TimeKeeper()
    assert tk.process(100.0, (100.5, 100.6, 100.5)) and tk.last_points_stamp == 100.5
    assert not tk.process(100.9, (100.4, 100.5, 100.4))
    # far from the stamp: the first frame's offset is kept for all later frames
    tk = PB.TimeKeeper()
    assert tk.process(1000.0, (10.0, 10.1, 10.0)) and tk.point_time_offset == 990.0 and tk.last_points_stamp == 1000.0
    assert tk.process(5.0, (10.2, 10.3, 10.2)) and tk.last_points_stamp == 10.2 + 990.0
    # nanoseconds above 1e16 become seconds
    tk = PB.TimeKeeper()
    assert tk.process(2.0e7, (2.0e16, 2.0e16, 2.0e16)) and tk.last_points_stamp == 2.0e16 * 1e-9
    # negative times are shifted by the minimum, frame stamp with them
    tk = PB.TimeKeeper()
    assert tk.process(50.0, (-0.05, 0.02, -0.1)) and tk.last_points_stamp == 50.0 - (-0.1)
    # 1000 frames without times fix the scan duration estimate
    tk = PB.TimeKeeper()
    for k in range(1001):
        tk.process(0.1 * k)
    assert tk.estimated_scan_duration == (0.1 * 999 - 0.0) / 999
