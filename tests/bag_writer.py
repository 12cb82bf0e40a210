"""A bag writer for the tests, written from the format specifications: ROS 1 bag format 2.0 (chunks `none`, `bz2` or a
named compression), ROS 2 sqlite3 bags (metadata.yaml + *.db3), and the four sensor_msgs messages in ROS 1
serialisation and in CDR of either endianness."""
import bz2
import os
import sqlite3
import struct

import numpy as np

# ---- message serialisation --------------------------------------------------------------------------------------------


class _W:
    def __init__(self, cdr, big=False):
        self.cdr, self.e = cdr, (">" if big else "<")
        self.b = bytearray(b"\x00\x00\x00\x00" if not big else b"\x00\x00\x00\x00") if cdr else bytearray()
        if cdr:
            self.b[1] = 0 if big else 1
        self.base = 4 if cdr else 0

    def _align(self, n):
        if self.cdr:
            while (len(self.b) - self.base) % n:
                self.b.append(0)

    def prim(self, fmt, v):
        self._align(struct.calcsize(fmt))
        self.b += struct.pack(self.e + fmt, v)

    def array(self, fmt, vals):
        if len(vals):
            self._align(struct.calcsize(fmt))
        self.b += struct.pack(f"{self.e}{len(vals)}{fmt}", *vals)

    def string(self, s):
        raw = s.encode() + (b"\0" if self.cdr else b"")
        self.prim("I", len(raw))
        self.b += raw

    def blob(self, data):
        self.prim("I", len(data))
        self.b += bytes(data)

    def header(self, sec, nsec, frame="frame"):
        if not self.cdr:
            self.prim("I", 0)
            self.prim("I", sec)
        else:
            self.prim("i", sec)
        self.prim("I", nsec)
        self.string(frame)


def point_cloud2(sec, nsec, fields, data, width, height=1, point_step=None, is_bigendian=False, cdr=False, big=False):
    """fields: [(name, offset, datatype)]"""
    w = _W(cdr, big)
    w.header(sec, nsec)
    w.prim("I", height)
    w.prim("I", width)
    w.prim("I", len(fields))
    for name, off, dt in fields:
        w.string(name)
        w.prim("I", off)
        w.prim("B", dt)
        w.prim("I", 1)
    w.prim("B", 1 if is_bigendian else 0)
    w.prim("I", point_step)
    w.prim("I", point_step * width)
    w.blob(data)
    w.prim("B", 1)
    return bytes(w.b)


def image(sec, nsec, pixels, encoding, cdr=False, big=False, pad=0):
    h, wd = pixels.shape[:2]
    ch = 1 if pixels.ndim == 2 else pixels.shape[2]
    step = wd * ch + pad
    rows = np.zeros((h, step), np.uint8)
    rows[:, : wd * ch] = pixels.reshape(h, wd * ch)
    w = _W(cdr, big)
    w.header(sec, nsec)
    w.prim("I", h)
    w.prim("I", wd)
    w.string(encoding)
    w.prim("B", 0)
    w.prim("I", step)
    w.blob(rows.tobytes())
    return bytes(w.b)


def compressed_image(sec, nsec, fmt, data, cdr=False, big=False):
    w = _W(cdr, big)
    w.header(sec, nsec)
    w.string(fmt)
    w.blob(data)
    return bytes(w.b)


def camera_info(sec, nsec, width, height, model, d, k, cdr=False, big=False):
    w = _W(cdr, big)
    w.header(sec, nsec)
    w.prim("I", height)
    w.prim("I", width)
    w.string(model)
    w.prim("I", len(d))
    w.array("d", list(d))
    w.array("d", list(k))
    w.array("d", [1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0])
    w.array("d", [k[0], 0, k[2], 0, 0, k[4], k[5], 0, 0, 0, 1.0, 0])
    w.prim("I", 0)
    w.prim("I", 0)
    for _ in range(4):
        w.prim("I", 0)
    w.prim("B", 0)
    return bytes(w.b)


def cloud_bytes(xyz, intensity, xyz_dtype="<f4", inten_dtype="<f4", offsets=None, point_step=None, times=None, time_dtype="<f8"):
    """Packs points into a PointCloud2 data blob -> (data, fields, point_step).  offsets: dict name -> byte offset."""
    n = xyz.shape[0]
    xs, isz = np.dtype(xyz_dtype).itemsize, np.dtype(inten_dtype).itemsize
    if offsets is None:
        offsets = {"x": 0, "y": xs, "z": 2 * xs, "intensity": 3 * xs}
        if times is not None:
            offsets["time"] = 3 * xs + isz
    end = max(offsets[k] + (xs if k in "xyz" else isz if k == "intensity" else np.dtype(time_dtype).itemsize) for k in offsets)
    step = point_step or end
    buf = np.zeros((n, step), np.uint8)
    cols = {"x": (xyz[:, 0], xyz_dtype), "y": (xyz[:, 1], xyz_dtype), "z": (xyz[:, 2], xyz_dtype), "intensity": (intensity, inten_dtype)}
    if times is not None:
        cols["time"] = (times, time_dtype)
    dt_code = {"<f4": 7, "<f8": 8, "u1": 2, "<u2": 4, "<u4": 6, "|u1": 2}
    fields = []
    for name, off in offsets.items():
        v, dt = cols[name]
        a = np.asarray(v).astype(dt)
        buf[:, off:off + a.dtype.itemsize] = a.view(np.uint8).reshape(n, a.dtype.itemsize)
        fields.append((name, off, dt_code[np.dtype(dt).str]))
    return buf.tobytes(), fields, step


# ---- ROS 1 ---------------------------------------------------------------------------------------------------------------

def _hdr(fields):
    out = bytearray()
    for k, v in fields.items():
        f = k.encode() + b"=" + v
        out += struct.pack("<I", len(f)) + f
    return bytes(out)


def _record(fields, data):
    h = _hdr(fields)
    return struct.pack("<I", len(h)) + h + struct.pack("<I", len(data)) + data


def _t(ns):
    return struct.pack("<II", ns // 1_000_000_000, ns % 1_000_000_000)


def write_ros1(path, messages, compression="none", per_chunk=3):
    """messages: [(topic, type, time_ns, raw)] in file order; chunks of `per_chunk` messages."""
    conns, conn_recs = {}, {}
    for topic, typ, _, _ in messages:
        if topic not in conns:
            cid = len(conns)
            conns[topic] = cid
            conn_recs[cid] = _record({"op": b"\x07", "topic": topic.encode(), "conn": struct.pack("<I", cid)},
                                     _hdr({"topic": topic.encode(), "type": typ.encode(), "md5sum": b"0" * 32, "message_definition": b""}))
    body = bytearray()
    chunk_infos = []
    base = len(b"#ROSBAG V2.0\n") + 4096 + 8 + 4096  # (approximate header position; positions only need to be increasing)
    seen = set()
    for c0 in range(0, len(messages), per_chunk):
        inner = bytearray()
        for topic, typ, t, raw in messages[c0:c0 + per_chunk]:
            cid = conns[topic]
            if cid not in seen:
                inner += conn_recs[cid]
                seen.add(cid)
            inner += _record({"op": b"\x02", "conn": struct.pack("<I", cid), "time": _t(t)}, raw)
        data = bytes(inner) if compression == "none" else bz2.compress(bytes(inner)) if compression == "bz2" else bytes(inner)
        pos = base + len(body)
        body += _record({"op": b"\x05", "compression": compression.encode(), "size": struct.pack("<I", len(inner))}, data)
        chunk_infos.append(pos)
    index_tail = b"".join(conn_recs[c] for c in sorted(conn_recs))
    for pos in chunk_infos:
        index_tail += _record({"op": b"\x06", "ver": struct.pack("<I", 1), "chunk_pos": struct.pack("<Q", pos), "start_time": _t(0), "end_time": _t(0),
                               "count": struct.pack("<I", 0)}, b"")
    header_fields = {"op": b"\x03", "index_pos": struct.pack("<Q", 0), "conn_count": struct.pack("<I", len(conns)), "chunk_count": struct.pack("<I", len(chunk_infos))}
    h = _hdr(header_fields)
    pad = 4096 - (4 + len(h) + 4)
    header = struct.pack("<I", len(h)) + h + struct.pack("<I", pad) + b" " * pad
    version = b"#ROSBAG V2.0\n"
    index_pos = len(version) + len(header) + len(body)
    header_fields["index_pos"] = struct.pack("<Q", index_pos)
    h = _hdr(header_fields)
    header = struct.pack("<I", len(h)) + h + struct.pack("<I", pad) + b" " * pad
    with open(path, "wb") as f:
        f.write(version + header + bytes(body) + index_tail)


# ---- ROS 2 ---------------------------------------------------------------------------------------------------------------

def write_ros2(path, messages, n_files=1, storage="sqlite3"):
    """messages: [(topic, type, time_ns, raw)]; spread over n_files .db3 files in order (file k holds a contiguous part)."""
    os.makedirs(path, exist_ok=True)
    name = os.path.basename(path.rstrip("/"))
    files = [f"{name}_{k}.db3" for k in range(n_files)]
    topics = []
    for topic, typ, _, _ in messages:
        if (topic, typ) not in topics:
            topics.append((topic, typ))
    per = -(-len(messages) // n_files) if messages else 0
    for k, fn in enumerate(files):
        db = sqlite3.connect(os.path.join(path, fn))
        db.execute("CREATE TABLE topics(id INTEGER PRIMARY KEY, name TEXT NOT NULL, type TEXT NOT NULL, serialization_format TEXT NOT NULL, "
                   "offered_qos_profiles TEXT NOT NULL)")
        db.execute("CREATE TABLE messages(id INTEGER PRIMARY KEY, topic_id INTEGER NOT NULL, timestamp INTEGER NOT NULL, data BLOB NOT NULL)")
        for i, (topic, typ) in enumerate(topics):
            db.execute("INSERT INTO topics VALUES (?, ?, ?, 'cdr', '')", (i + 1, topic, typ))
        for topic, typ, t, raw in messages[k * per:(k + 1) * per]:
            db.execute("INSERT INTO messages(topic_id, timestamp, data) VALUES (?, ?, ?)", (topics.index((topic, typ)) + 1, t, raw))
        db.commit()
        db.close()
    with open(os.path.join(path, "metadata.yaml"), "w") as f:
        f.write("rosbag2_bagfile_information:\n  version: 5\n  storage_identifier: " + storage + "\n  relative_file_paths:\n")
        for fn in files:
            f.write(f"    - {fn}\n")
        f.write(f"  message_count: {len(messages)}\n")
