"""`preprocess` from bags: a calibration dataset from a directory of ROS 1 / ROS 2 bags with static point integration
(src/vlcal/preprocess/preprocess.cpp, src/preprocess_ros1.cpp, src/preprocess_ros2.cpp).

    per bag: first image --mono8, equalizeHist--> <bag>.png
             PointCloud2 scans --host: layout, TimeKeeper--> accepted scans --GPU: decode + static integration-->
             rank equalisation (GPU) --> <bag>.ply
    first bag's points --estimate_lidar_fov--> virtual LiDAR camera --K5--> <bag>_lidar_intensities.png, _lidar_indices.png
    calib.json (meta + camera)

Deviation (DESIGN §4c): the integrated points come out in first-write order, where the reference gives its hash table's
iteration order.  Input on which the reference is undefined is refused (a points topic without the intensity channel,
big-endian clouds, a bag without an image)."""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import numpy as np

from . import _lib
from . import bag_io as B

VALID_CAMERA_MODELS = ("plumb_bob", "fisheye", "equidistant", "omnidir", "equirectangular")  # preprocess.cpp:362, no atan
TIME_FIELDS = ("t", "time", "time_stamp", "timestamp")


class TimeKeeper:
    """vlcal::TimeKeeper::process (time_keeper.cpp:44-180) with the default AbsPointTimeParams (replace_frame_timestamp and
    wrt_first_frame_timestamp true).  The decision needs the frame stamp and, when the scan has per-point times, the
    first, last and minimum point time; the per-point arithmetic on the first time is restated literally."""

    def __init__(self):
        self.first_warning = True
        self.last_points_stamp = -1.0
        self.num_scans = 0
        self.first_points_stamp = 0.0
        self.estimated_scan_duration = -1.0
        self.point_time_offset = 0.0

    def _estimate_scan_duration(self, stamp):
        if self.estimated_scan_duration > 0.0:
            return self.estimated_scan_duration
        n = self.num_scans
        self.num_scans += 1
        if n == 0:
            self.first_points_stamp = stamp
            return -1.0
        d = (stamp - self.first_points_stamp) / (self.num_scans - 1)
        if self.num_scans == 1000:
            self.estimated_scan_duration = d
        return d

    def _replace_points_stamp(self, stamp, times):
        if times is None:  # no per-point times (or no points)
            self.first_warning = False
            self._estimate_scan_duration(stamp)
            return stamp
        front, back, tmin = times
        if front < 0.0 or back < 0.0:
            front = front - tmin
            stamp = stamp - tmin
        if front < 1.0:
            return stamp
        if front > 1e16:
            front = front * 1e-9
        if not (abs(stamp - front) < 1.0):  # wrt_first_frame_timestamp
            if self.first_warning:
                self.point_time_offset = stamp - front
            stamp = front + self.point_time_offset
        else:
            self.point_time_offset = 0.0
            stamp = front
        self.first_warning = False
        return stamp

    def process(self, stamp: float, times=None) -> bool:
        """times: None, or (first, last, min) of the scan's per-point times -> False when the frame is skipped."""
        stamp = self._replace_points_stamp(stamp, times)
        if self.last_points_stamp < 0.0:
            pass
        elif stamp - self.last_points_stamp < 0.0:
            return False
        self.last_points_stamp = stamp
        return True


class Unconvertible(Exception):
    """extract_raw_points returns nullptr for this scan: the reference stops reading the bag there."""


def scan_layout(msg: dict, intensity_channel: str):
    """extract_raw_points' field lookup (ros_cloud_converter.hpp:63-105, 121-170) -> (n_points, (x, y, z offsets),
    x_type, (time offset, time type), (intensity offset, intensity type)); raises Unconvertible where the reference
    returns nullptr."""
    xs, ys, zs = [0, -1], [0, -1], [0, -1]
    slots = {"x": xs, "y": ys, "z": zs}
    time_slot, inten_slot = [0, -1], [0, -1]
    for name in TIME_FIELDS:
        slots[name] = time_slot
    # fields[intensity_channel] replaces the entry of that name: with -i x, the "x" field fills the intensity and x's
    # offset stays -1
    slots[intensity_channel] = inten_slot
    for name, offset, datatype, _ in msg["fields"]:
        if name in slots:
            slots[name][0], slots[name][1] = datatype, offset
    n = (msg["width"] * msg["height"]) & 0xFFFFFFFF
    n = n - (1 << 32) if n >= 1 << 31 else n  # int num_points = width * height
    if xs[1] < 0 or ys[1] < 0 or zs[1] < 0:
        raise Unconvertible("missing point coordinate fields")
    if xs[0] not in (B.FLOAT32, B.FLOAT64) or xs[0] != ys[0]:
        raise Unconvertible("unsupported points type")
    if n > 0 and time_slot[1] >= 0 and time_slot[0] not in (B.UINT32, B.FLOAT32, B.FLOAT64):
        raise Unconvertible(f"unsupported time type {time_slot[0]}")
    if n > 0 and inten_slot[1] >= 0 and inten_slot[0] not in (B.UINT8, B.UINT16, B.UINT32, B.FLOAT32, B.FLOAT64):
        raise Unconvertible("unsupported intensity type")
    return max(n, 0), (xs[1], ys[1], zs[1]), xs[0], (time_slot[1], time_slot[0]), (inten_slot[1], inten_slot[0])


def _field_view(data, n, step, offset, dtype):
    return np.ndarray((n,), dtype=np.dtype(dtype).newbyteorder("<"), buffer=data, offset=offset, strides=(step,))


def point_times(msg: dict, n: int, time_field):
    """(first, last, min) of the per-point times as extract_raw_points converts them, or None without times."""
    off, typ = time_field
    if off < 0 or n == 0:
        return None
    v = _field_view(msg["data"], n, msg["point_step"], off, {B.UINT32: np.uint32, B.FLOAT32: np.float32, B.FLOAT64: np.float64}[typ])
    t = v.astype(np.float64) / 1e9 if typ == B.UINT32 else v.astype(np.float64)
    return float(t[0]), float(t[-1]), float(t.min())


def collect_scans(bag, bag_name: str, points_topic: str, intensity_channel: str, ros1: bool, warn=print):
    """The reader loop of get_image_and_points (preprocess.cpp:442-460) up to the integrator -> (data blob (uint8),
    list of ScanDesc, stats).  Scans skipped by the TimeKeeper are left out; an unconvertible scan ends the bag."""
    keeper = TimeKeeper()
    parts, descs = [], []
    offset, skipped, read = 0, 0, 0
    for k, (typ, raw) in enumerate(bag.messages(points_topic)):
        if ros1 and typ != "sensor_msgs/PointCloud2":  # instantiate<PointCloud2>() gives nullptr: read_next ends the bag
            warn(f"warning: {bag_name}: scan {k} on {points_topic} is a {typ}, not a sensor_msgs/PointCloud2; reading stops there")
            break
        msg = B.decode_point_cloud2(raw, cdr=not ros1)
        try:
            n, (xo, yo, zo), xt, tf, (io, it) = scan_layout(msg, intensity_channel)
        except Unconvertible as e:
            warn(f"warning: {bag_name}: scan {k} cannot be converted ({e}); like the reference, reading the bag stops there")
            break
        read += 1
        if n > 0:
            if msg["is_bigendian"]:
                raise B.BagError(f"{bag_name}: scan {k} is big-endian (is_bigendian = true), which is not supported")
            if io < 0:
                raise B.BagError(f"{bag_name}: scan {k} has no '{intensity_channel}' field; the reference would read an empty intensity vector")
            need = msg["point_step"] * (n - 1) + max(xo + B.FIELD_SIZE[xt], yo + B.FIELD_SIZE[xt], zo + B.FIELD_SIZE[xt], io + B.FIELD_SIZE[it],
                                                     tf[0] + B.FIELD_SIZE[tf[1]] if tf[0] >= 0 else 0)
            if len(msg["data"]) < need:
                raise B.BagError(f"{bag_name}: scan {k}: {len(msg['data'])} data bytes do not hold {n} points of {msg['point_step']} bytes")
        if not keeper.process(msg["stamp"], point_times(msg, n, tf)):
            warn(f"warning: {bag_name}: skip frame {k} with an invalid timestamp")
            skipped += 1
            continue
        if n == 0:
            continue
        d = _lib.ScanDesc(byte_offset=offset, n_points=n, point_step=msg["point_step"], x_offset=xo, y_offset=yo, z_offset=zo, xyz_type=xt,
                          intensity_offset=io, intensity_type=it)
        size = len(msg["data"])
        parts.append(np.frombuffer(msg["data"], dtype=np.uint8))
        descs.append(d)
        offset += size
    blob = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    return blob, descs, {"scans_read": read, "scans_skipped": skipped, "scans_integrated": len(descs)}


def bag_integrate(blob, descs, voxel_resolution=0.002, min_distance=1.0, device: int = -1, stats: dict | None = None) -> np.ndarray:
    """vlcal_bag_integrate: decode + static integration on the GPU -> float32 (M, 4) x, y, z, intensity in first-write
    order."""
    L = _lib.load_library()
    blob = np.ascontiguousarray(blob, dtype=np.uint8)
    arr = (_lib.ScanDesc * max(len(descs), 1))(*descs)
    total = sum(d.n_points for d in descs)
    out = np.empty((max(total, 1), 4), np.float32)
    n_out, oor = C.c_int64(), C.c_int64()
    ms = (C.c_double * 3)()
    _lib.check(L.vlcal_bag_integrate(device, blob.ctypes.data, blob.size, arr, len(descs), float(voxel_resolution), float(min_distance), out.ctypes.data,
                                     C.byref(n_out), C.byref(oor), ms))
    if stats is not None:
        stats["out_of_range_points"] = int(oor.value)
        stats["stage_ms"] = list(ms)
    return out[: n_out.value].copy()


# ---- topic, channel and camera selection (preprocess.cpp:266-404) ------------------------------------------------------

def get_topics(topics_and_types, auto_topic: bool, camera_info_topic=None, image_topic=None, points_topic=None, warn=print):
    ci, im, pt = "", "", ""
    if auto_topic:
        for topic, typ in topics_and_types:
            if "CameraInfo" in typ:
                if ci:
                    warn("warning: bag constains multiple camera_info topics!!")
                ci = topic
            elif "Image" in typ:
                if im:
                    warn("warning: bag constains multiple image topics!!")
                im = topic
            elif "PointCloud2" in typ:
                if pt:
                    warn("warning: bag constains multiple points topics!!")
                pt = topic
    ci = ci or (camera_info_topic or "")
    im = im or (image_topic or "")
    pt = pt or (points_topic or "")
    return ci, im, pt


def get_intensity_channel(field_names, intensity_channel: str = "auto") -> str:
    if intensity_channel != "auto":
        return intensity_channel
    prio = {"auto": -1, "intensity": 1, "reflectivity": 2}
    for f in field_names:
        if f in prio and prio[intensity_channel] < prio[f]:
            intensity_channel = f
    return intensity_channel


def _first(bag, topic):
    for typ, raw in bag.messages(topic):
        return typ, raw
    return None


def first_image(bag, image_topic: str, ros1: bool, bag_name: str) -> np.ndarray:
    """get_image: the first message as mono8.  ROS 1 tries Image, then CompressedImage; ROS 2 picks by whether the topic's
    name contains "compressed"."""
    if ros1:
        for want, dec, conv in (("sensor_msgs/Image", B.decode_image, B.image_to_mono8), ("sensor_msgs/CompressedImage", B.decode_compressed_image, B.compressed_to_mono8)):
            for typ, raw in bag.messages(image_topic):
                if typ == want:
                    return conv(dec(raw, cdr=False))
    else:
        m = _first(bag, image_topic)
        if m is not None:
            if "compressed" in image_topic:
                return B.compressed_to_mono8(B.decode_compressed_image(m[1], cdr=True))
            return B.image_to_mono8(B.decode_image(m[1], cdr=True))
    raise B.BagError(f"{bag_name}: no image message on topic '{image_topic}'")


def camera_params(bag, ros1: bool, bag_name: str, camera_info_topic: str, image_size, camera_model="auto", intrinsics=None, distortion=None):
    """get_camera_params -> (camera_model, intrinsics, distortion_coeffs)."""
    if camera_model != "auto":
        if camera_model not in VALID_CAMERA_MODELS:
            raise ValueError(f"invalid camera model {camera_model}; supported camera models are {' '.join(VALID_CAMERA_MODELS)}")
        if camera_model == "equirectangular":
            return camera_model, [float(image_size[0]), float(image_size[1])], []
        if intrinsics is None or distortion is None:
            raise ValueError("camera_intrinsics and camera_distortion_coeffs must be set when camera_model is not auto")
        from .preprocess import parse_values

        return camera_model, parse_values(intrinsics, "camera_intrinsics"), parse_values(distortion, "camera_distortion_coeffs")
    m = _first(bag, camera_info_topic)
    if m is None:
        raise B.BagError(f"{bag_name}: no CameraInfo message on topic '{camera_info_topic}'")
    ci = B.decode_camera_info(m[1], cdr=not ros1)
    k = ci["k"]
    return ci["distortion_model"], [k[0], k[4], k[2], k[5]], list(ci["d"])


def list_bags(data_path: str):
    return sorted(os.path.join(data_path, e) for e in os.listdir(data_path) if B.is_ros1_bag(os.path.join(data_path, e)) or B.is_ros2_bag(os.path.join(data_path, e)))


def preprocess_bags(data_path: str, dst_path: str, auto_topic=False, camera_info_topic=None, image_topic=None, points_topic=None,
                    intensity_channel="auto", camera_model="auto", camera_intrinsics=None, camera_distortion_coeffs=None, voxel_resolution=0.002,
                    min_distance=1.0, bag_id=None, first_n_bags=None, device: int = -1, stats: dict | None = None, log=print) -> dict:
    """Preprocess::run with the static integrator (preprocess.cpp:37-264): writes <bag>.png, <bag>.ply,
    <bag>_lidar_intensities.png, <bag>_lidar_indices.png per bag and calib.json into dst_path.  Returns calib.json."""
    import time

    import cv2

    from . import io as vio
    from . import preprocess as P
    from .camera import create_camera
    from .culling import generate_lidar_image

    stats = {} if stats is None else stats
    os.makedirs(dst_path, exist_ok=True)
    bags = list_bags(data_path)
    if not bags:
        raise B.BagError(f"no input bags in {data_path}")
    if bag_id is not None:
        bags = [bags[bag_id]]
    if first_n_bags is not None:
        bags = bags[:first_n_bags]
    first = B.open_bag(bags[0])
    ros1 = isinstance(first, B.Ros1Bag)
    ci_topic, im_topic, pt_topic = get_topics(first.topics_and_types(), auto_topic, camera_info_topic, image_topic, points_topic, warn=log)
    log(f"selected topics:\n- camera_info: {ci_topic}\n- image      : {im_topic}\n- points     : {pt_topic}")
    m = _first(first, pt_topic)
    if m is None:
        raise B.BagError(f"{os.path.basename(bags[0])}: no message on the points topic '{pt_topic}'")
    fields = [f[0] for f in B.decode_point_cloud2(m[1], cdr=not ros1)["fields"]]
    channel = get_intensity_channel(fields, intensity_channel)
    if channel == "auto":
        raise B.BagError(f"{os.path.basename(bags[0])}: failed to determine the point intensity channel automatically (fields: {', '.join(fields)}); "
                         "set --intensity_channel")
    if channel not in fields:
        raise B.BagError(f"{os.path.basename(bags[0])}: the points topic '{pt_topic}' has no intensity channel '{channel}'")
    log(f"intensity_channel: {channel}")
    image0 = first_image(first, im_topic, ros1, os.path.basename(bags[0]))
    model, intrinsics, distortion = camera_params(first, ros1, os.path.basename(bags[0]), ci_topic, (image0.shape[1], image0.shape[0]), camera_model,
                                                  camera_intrinsics, camera_distortion_coeffs)
    log(f"camera_model: {model}")

    clouds, per_bag = [], []
    t_io = t_gpu = 0.0
    for k, path in enumerate(bags):
        name = os.path.basename(path.rstrip("/"))
        t0 = time.perf_counter()
        bag = first if k == 0 else B.open_bag(path)
        is1 = isinstance(bag, B.Ros1Bag)
        image = image0 if k == 0 else first_image(bag, im_topic, is1, name)
        blob, descs, st = collect_scans(bag, name, pt_topic, channel, is1, warn=log)
        t1 = time.perf_counter()
        integ = {}
        pts = bag_integrate(blob, descs, voxel_resolution, min_distance, device=device, stats=integ)
        if integ["out_of_range_points"]:
            log(f"warning: {name}: {integ['out_of_range_points']} points have a voxel index outside int range; like the reference, "
                "their index becomes INT_MIN, which merges voxels along that axis")
        eq = {}
        inten = P.equalize_intensities(pts[:, 3], device=device, stats=eq)
        t2 = time.perf_counter()
        cv2.imwrite(os.path.join(dst_path, name + ".png"), cv2.equalizeHist(image))
        vio.save_ply_binary(os.path.join(dst_path, name + ".ply"), pts[:, :3], inten)
        t3 = time.perf_counter()
        t_io += (t1 - t0) + (t3 - t2)
        t_gpu += t2 - t1
        clouds.append((name, pts, inten))
        per_bag.append(dict(st, name=name, points_in=int(sum(d.n_points for d in descs)), points_out=int(pts.shape[0]), integrate=integ, equalize=eq))
        log(f"processed {name}: {st['scans_integrated']} scans, {pts.shape[0]} points")

    lidar_fov = P.estimate_lidar_fov(clouds[0][1][:, :3], device=device)
    log(f"LiDAR FoV: {lidar_fov * 180.0 / math.pi}[deg]")
    vmodel, vintr, size, T_camera_lidar = P.virtual_lidar_camera(lidar_fov)
    proj = create_camera(vmodel, vintr, [])
    for name, pts, inten in clouds:
        xyzw = np.concatenate([pts[:, :3].astype(np.float64), np.ones((pts.shape[0], 1))], axis=1)
        img, idx = generate_lidar_image(proj, size, T_camera_lidar, xyzw, inten, device=device)
        cv2.imwrite(os.path.join(dst_path, name + "_lidar_intensities.png"), P.lidar_intensity_png(img))
        vio.save_lidar_indices(os.path.join(dst_path, name + "_lidar_indices.png"), idx)

    config = {
        "camera": {"camera_model": model, "distortion_coeffs": list(distortion), "intrinsics": list(intrinsics)},
        "meta": {"bag_names": [c[0] for c in clouds], "camera_info_topic": ci_topic, "data_path": data_path, "image_topic": im_topic,
                 "intensity_channel": channel, "points_topic": pt_topic},
    }
    with open(os.path.join(dst_path, "calib.json"), "w") as f:
        f.write(json.dumps(config, indent=2, sort_keys=True) + "\n")  # nlohmann's std::map keeps keys sorted
    stats.update(bags=per_bag, lidar_fov=lidar_fov, virtual_camera=vmodel, io_s=t_io, gpu_s=t_gpu)
    return config
