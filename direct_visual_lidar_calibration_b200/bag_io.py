"""Bag readers and message decoders for `preprocess`, standard library only (plus numpy / cv2 for the image).

    ROS 1 (bag format 2.0, chunks `none` or `bz2`)   Ros1Bag
    ROS 2 (a directory of metadata.yaml + *.db3)   Ros2Bag
    sensor_msgs PointCloud2, Image, CompressedImage, CameraInfo in ROS 1 serialisation and in CDR (both endiannesses)

A bag's messages on a topic come back in the order the reference reads them: ROS 1 in rosbag::View order (receive time,
then file position), ROS 2 file by file as metadata.yaml lists them, each file's messages by timestamp, then id.  lz4
chunks and MCAP storage are refused with a message that says how to convert the bag."""
from __future__ import annotations

import bz2
import mmap
import os
import re
import sqlite3
import struct

import numpy as np

ROS1_VERSION = b"#ROSBAG V2.0\n"

# sensor_msgs/PointField datatypes
INT8, UINT8, INT16, UINT16, INT32, UINT32, FLOAT32, FLOAT64 = range(1, 9)
FIELD_SIZE = {INT8: 1, UINT8: 1, INT16: 2, UINT16: 2, INT32: 4, UINT32: 4, FLOAT32: 4, FLOAT64: 8}


class BagError(ValueError):
    """A bag this project cannot read, with the reason and the fix where there is one."""


# ---- ROS 1 -------------------------------------------------------------------------------------------------------------

def _ros1_header(buf, pos, end):
    fields = {}
    while pos < end:
        (n,) = struct.unpack_from("<I", buf, pos)
        pos += 4
        raw = bytes(buf[pos:pos + n])
        pos += n
        k, _, v = raw.partition(b"=")
        fields[k.decode()] = v
    return fields


def _ros1_records(buf, pos, end):
    """(header fields, data start, data end, record start) of each record in buf[pos:end]."""
    while pos + 4 <= end:
        start = pos
        (hl,) = struct.unpack_from("<I", buf, pos)
        h = _ros1_header(buf, pos + 4, pos + 4 + hl)
        pos += 4 + hl
        (dl,) = struct.unpack_from("<I", buf, pos)
        pos += 4
        yield h, pos, pos + dl, start
        pos += dl


class Ros1Bag:
    """A ROS 1 bag (format 2.0) read whole: its connections and an index of its messages."""

    def __init__(self, path: str):
        self.path = path
        with open(path, "rb") as f:
            # mapped, not read: uncompressed chunks are sliced from the page cache (bz2 chunks are held decompressed)
            self._buf = memoryview(mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)) if os.fstat(f.fileno()).st_size else memoryview(b"")
        if bytes(self._buf[: len(ROS1_VERSION)]) != ROS1_VERSION:
            raise BagError(f"{path}: not a ROS 1 bag of format 2.0 (the first line is not '#ROSBAG V2.0')")
        self.connections = {}  # conn id -> (topic, datatype)
        self._index = []  # (time_ns, chunk position, offset, conn, data memoryview)
        buf = self._buf
        for h, ds, de, rs in _ros1_records(buf, len(ROS1_VERSION), len(buf)):
            op = h.get("op", b"\0")[0]
            if op == 0x05:  # chunk
                comp = h["compression"].decode()
                if comp == "none":
                    chunk = buf[ds:de]
                elif comp == "bz2":
                    chunk = memoryview(bz2.decompress(buf[ds:de]))
                else:
                    raise BagError(f"{path}: a chunk is compressed with '{comp}', which this reader does not support "
                                   f"(only 'none' and 'bz2'); run `rosbag decompress {os.path.basename(path)}` first")
                for ih, ids, ide, irs in _ros1_records(chunk, 0, len(chunk)):
                    self._record(ih, chunk, ids, ide, rs, irs)
            else:
                self._record(h, buf, ds, de, rs, 0)
        self._index.sort(key=lambda e: (e[0], e[1], e[2]))

    def _record(self, h, buf, ds, de, chunk_pos, offset):
        op = h.get("op", b"\0")[0]
        if op == 0x07:
            conn = struct.unpack("<I", h["conn"])[0]
            ch = _ros1_header(buf, ds, de)
            self.connections.setdefault(conn, (h["topic"].decode(), ch["type"].decode()))
        elif op == 0x02:
            conn = struct.unpack("<I", h["conn"])[0]
            sec, nsec = struct.unpack("<II", h["time"])
            self._index.append((sec * 1_000_000_000 + nsec, chunk_pos, offset, conn, buf[ds:de]))

    def topics_and_types(self):
        return [self.connections[c] for c in sorted(self.connections)]

    def messages(self, topic: str):
        """(datatype, raw message) of every message on `topic`, in rosbag::View order."""
        for _, _, _, conn, data in self._index:
            t, typ = self.connections[conn]
            if t == topic:
                yield typ, data


# ---- ROS 2 (sqlite3) ----------------------------------------------------------------------------------------------------

def _metadata(path: str):
    with open(os.path.join(path, "metadata.yaml")) as f:
        text = f.read()
    m = re.search(r"storage_identifier:\s*['\"]?([\w-]+)", text)
    storage = m.group(1) if m else ""
    files = []
    m = re.search(r"relative_file_paths:\s*\n((?:\s+-\s*.*\n?)+)", text)
    if m:
        files = [ln.split("-", 1)[1].strip().strip("'\"") for ln in m.group(1).splitlines() if ln.strip().startswith("-")]
    else:
        m = re.search(r"relative_file_paths:\s*\[(.*?)\]", text)
        if m:
            files = [s.strip().strip("'\"") for s in m.group(1).split(",") if s.strip()]
    return storage, files


class Ros2Bag:
    """A ROS 2 bag with sqlite3 storage: a directory holding metadata.yaml and the *.db3 files it lists."""

    def __init__(self, path: str):
        self.path = path
        if not os.path.isfile(os.path.join(path, "metadata.yaml")):
            raise BagError(f"{path}: not a ROS 2 bag (no metadata.yaml)")
        storage, files = _metadata(path)
        if storage != "sqlite3":
            raise BagError(f"{path}: storage '{storage}' is not supported, only sqlite3 (rosbag2's MCAP writer compresses with zstd "
                           "by default, and zstd is not in Python's standard library); convert the bag with `ros2 bag convert` to "
                           "storage_id sqlite3")
        if not files:
            files = sorted(f for f in os.listdir(path) if f.endswith(".db3"))
        self.files = [os.path.join(path, f) for f in files]
        self._topics = []  # (name, type) over all files, first appearance
        for fn in self.files:
            with sqlite3.connect(f"file:{fn}?mode=ro", uri=True) as db:
                for name, typ in db.execute("SELECT name, type FROM topics ORDER BY id"):
                    if (name, typ) not in self._topics:
                        self._topics.append((name, typ))

    def topics_and_types(self):
        return list(self._topics)

    def messages(self, topic: str):
        for fn in self.files:
            db = sqlite3.connect(f"file:{fn}?mode=ro", uri=True)
            try:
                q = ("SELECT t.type, m.data FROM messages m JOIN topics t ON m.topic_id = t.id WHERE t.name = ? "
                     "ORDER BY m.timestamp, m.id")
                for typ, data in db.execute(q, (topic,)):
                    yield typ, memoryview(data)
            finally:
                db.close()


def is_ros1_bag(path: str) -> bool:
    """valid_bag of preprocess_ros1.cpp: rosbag::Bag opens it (a file whose version line is #ROSBAG V2.0)."""
    try:
        with open(path, "rb") as f:
            return f.read(len(ROS1_VERSION)) == ROS1_VERSION
    except OSError:
        return False


def is_ros2_bag(path: str) -> bool:
    return os.path.isdir(path) and os.path.isfile(os.path.join(path, "metadata.yaml"))


def open_bag(path: str):
    return Ros1Bag(path) if is_ros1_bag(path) else Ros2Bag(path)


# ---- message decoding ---------------------------------------------------------------------------------------------------

class _Reader:
    """ROS 1 serialisation (little-endian, packed, uint32-prefixed strings without NUL) or CDR (the encapsulation header
    picks the endianness; every primitive aligned to its size, measured from the end of that header)."""

    def __init__(self, data, cdr: bool):
        self.b = data
        self.cdr = cdr
        if cdr:
            if len(data) < 4 or data[0] != 0 or data[1] not in (0, 1):
                raise BagError("not a CDR message (unknown encapsulation header)")
            self.e = "<" if data[1] == 1 else ">"
            self.base, self.p = 4, 4
        else:
            self.e, self.base, self.p = "<", 0, 0

    def _align(self, n):
        if self.cdr:
            r = (self.p - self.base) % n
            if r:
                self.p += n - r

    def prim(self, fmt):
        n = struct.calcsize(fmt)
        self._align(n)
        (v,) = struct.unpack_from(self.e + fmt, self.b, self.p)
        self.p += n
        return v

    def array(self, fmt, count):
        n = struct.calcsize(fmt)
        if count:
            self._align(n)
        v = struct.unpack_from(f"{self.e}{count}{fmt}", self.b, self.p)
        self.p += n * count
        return list(v)

    def string(self):
        n = self.prim("I")
        s = bytes(self.b[self.p:self.p + n])
        self.p += n
        return (s[:-1] if self.cdr and s.endswith(b"\0") else s).decode(errors="replace")

    def blob(self):
        n = self.prim("I")
        v = self.b[self.p:self.p + n]
        self.p += n
        return v

    def stamp(self):
        """the header stamp in seconds as the reference's to_sec gives it"""
        if self.cdr:
            sec, nsec = self.prim("i"), self.prim("I")
            return sec + nsec / 1e9  # stamp.sec + stamp.nanosec / 1e9
        sec, nsec = self.prim("I"), self.prim("I")
        return float(sec) + 1e-9 * float(nsec)  # ros::Time::toSec

    def header(self):
        if not self.cdr:
            self.prim("I")  # seq
        stamp = self.stamp()
        self.string()  # frame_id
        return stamp


def decode_point_cloud2(data, cdr: bool) -> dict:
    r = _Reader(data, cdr)
    stamp = r.header()
    height, width = r.prim("I"), r.prim("I")
    fields = []
    for _ in range(r.prim("I")):
        name = r.string()
        offset = r.prim("I")
        datatype = r.prim("B")
        count = r.prim("I")
        fields.append((name, offset, datatype, count))
    is_bigendian = bool(r.prim("B"))
    point_step, row_step = r.prim("I"), r.prim("I")
    blob = r.blob()
    return {"stamp": stamp, "height": height, "width": width, "fields": fields, "is_bigendian": is_bigendian, "point_step": point_step,
            "row_step": row_step, "data": blob}


def decode_image(data, cdr: bool) -> dict:
    r = _Reader(data, cdr)
    r.header()
    height, width = r.prim("I"), r.prim("I")
    encoding = r.string()
    is_bigendian = r.prim("B")
    step = r.prim("I")
    return {"height": height, "width": width, "encoding": encoding, "is_bigendian": is_bigendian, "step": step, "data": r.blob()}


def decode_compressed_image(data, cdr: bool) -> dict:
    r = _Reader(data, cdr)
    r.header()
    fmt = r.string()
    return {"format": fmt, "data": r.blob()}


def decode_camera_info(data, cdr: bool) -> dict:
    """ROS 1 names these D K R P, ROS 2 d k r p; the same layout."""
    r = _Reader(data, cdr)
    r.header()
    height, width = r.prim("I"), r.prim("I")
    model = r.string()
    d = r.array("d", r.prim("I"))
    k = r.array("d", 9)
    rr = r.array("d", 9)
    p = r.array("d", 12)
    return {"height": height, "width": width, "distortion_model": model, "d": d, "k": k, "r": rr, "p": p}


_TO_GRAY = {"bgr8": ("COLOR_BGR2GRAY", 3), "rgb8": ("COLOR_RGB2GRAY", 3), "bgra8": ("COLOR_BGRA2GRAY", 4), "rgba8": ("COLOR_RGBA2GRAY", 4)}


def image_to_mono8(msg: dict) -> np.ndarray:
    """cv_bridge::toCvCopy(msg, "mono8") for mono8, bgr8, rgb8, bgra8 and rgba8 Images; other encodings are refused."""
    import cv2

    enc = msg["encoding"]
    if enc != "mono8" and enc not in _TO_GRAY:
        raise BagError(f"image encoding '{enc}' is not supported (mono8, bgr8, rgb8, bgra8 and rgba8 are)")
    ch = 1 if enc == "mono8" else _TO_GRAY[enc][1]
    h, w, step = msg["height"], msg["width"], msg["step"]
    raw = np.frombuffer(msg["data"], dtype=np.uint8)
    if step < w * ch or raw.size < step * h:
        raise BagError(f"image of {w}x{h} {enc}: step {step} and {raw.size} data bytes do not hold it")
    img = raw[: step * h].reshape(h, step)[:, : w * ch].reshape(h, w, ch) if h else np.zeros((0, w, ch), np.uint8)
    if ch == 1:
        return np.ascontiguousarray(img[:, :, 0])
    return cv2.cvtColor(np.ascontiguousarray(img), getattr(cv2, _TO_GRAY[enc][0]))


def compressed_to_mono8(msg: dict) -> np.ndarray:
    """cv_bridge::toCvCopy(compressed, "mono8") for 8-bit images: imdecode(IMREAD_UNCHANGED), then colour to gray.
    Images of another depth (16-bit PNG) are refused: cv_bridge would convert them through mono16."""
    import cv2

    img = cv2.imdecode(np.frombuffer(msg["data"], dtype=np.uint8), cv2.IMREAD_UNCHANGED)
    if img is None:
        raise BagError(f"compressed image ({msg['format']}) could not be decoded")
    if img.dtype != np.uint8:
        raise BagError(f"compressed image ({msg['format']}) has {img.dtype} pixels; only 8-bit compressed images are supported")
    if img.ndim == 2:
        return img
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY if img.shape[2] == 3 else cv2.COLOR_BGRA2GRAY)
