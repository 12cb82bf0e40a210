"""Bag readers and message decoders for `preprocess` (standard library, numpy / cv2 for the image, and the GPU frame
decoder of frame_decode.py for compressed chunks).

    ROS 1 (bag format 2.0, chunks `none`, `bz2` or `lz4`)                    Ros1Bag
    ROS 2 (a directory of metadata.yaml + *.db3 or *.mcap files)            Ros2Bag, McapBag for each MCAP file
    rosbag2 per-message zstd compression (compression_mode: message)        Ros2Bag
    sensor_msgs PointCloud2, Image, CompressedImage, CameraInfo in ROS 1 serialisation and in CDR (both endiannesses)

A bag's messages on a topic come back in the order the reference reads them: ROS 1 in rosbag::View order (receive time,
then file position), ROS 2 file by file as metadata.yaml lists them, each sqlite3 file's messages by timestamp, then id,
each MCAP file's as McapBag documents.  lz4 chunks of ROS 1 bags, zstd / lz4 chunks of MCAP files and zstd-compressed
rosbag2 messages are decoded on the GPU, all those of one file in one call, when the file is opened (ROS 1, MCAP) or
when a topic is read (rosbag2 messages).  rosbag2's file-mode compression (one zstd frame per storage file) and bare
.mcap files outside a bag directory are refused with a message that says how to convert the bag."""
from __future__ import annotations

import bz2
import mmap
import os
import re
import sqlite3
import struct

import numpy as np

from . import _lib
from . import frame_decode as FD

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
        lz4 = []  # (record start, data start, data end, uncompressed size): decoded together after the scan
        for h, ds, de, rs in _ros1_records(buf, len(ROS1_VERSION), len(buf)):
            op = h.get("op", b"\0")[0]
            if op == 0x05:  # chunk
                comp = h["compression"].decode()
                if comp == "none":
                    chunk = buf[ds:de]
                elif comp == "bz2":
                    chunk = memoryview(bz2.decompress(buf[ds:de]))
                elif comp == "lz4":
                    problem = FD.lz4_header_problem(buf[ds:de])
                    if problem:
                        raise BagError(f"{path}: the lz4 chunk at byte {rs} cannot be read: {problem}; "
                                       f"run `rosbag decompress {os.path.basename(path)}` first")
                    lz4.append((rs, ds, de, struct.unpack("<I", h["size"])[0]))
                    continue
                else:
                    raise BagError(f"{path}: a chunk is compressed with '{comp}', which this reader does not support "
                                   f"(only 'none', 'bz2' and 'lz4'); run `rosbag decompress {os.path.basename(path)}` first")
                for ih, ids, ide, irs in _ros1_records(chunk, 0, len(chunk)):
                    self._record(ih, chunk, ids, ide, rs, irs)
            else:
                self._record(h, buf, ds, de, rs, 0)
        if lz4:
            out, offs = _decode(path, buf, [(ds, de - ds, size, FD.CODEC_LZ4_FRAME, None) for _, ds, de, size in lz4],
                                [f"the lz4 chunk at byte {rs}" for rs, *_ in lz4], f"; run `rosbag decompress {os.path.basename(path)}` first")
            self._decoded = out  # the messages below are views into it
            for (rs, _, _, size), o in zip(lz4, offs):
                chunk = memoryview(out)[o:o + size]
                for ih, ids, ide, irs in _ros1_records(chunk, 0, len(chunk)):
                    self._record(ih, chunk, ids, ide, rs, irs)
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


def _decode(path, src, frames, names, hint=""):
    """FD.decode_frames of one file's frames -> (output, offsets); a BagError naming the file and the frame (names[i])
    for a declared size its compressed bytes cannot hold (checked before anything is allocated), a frame that fails,
    or a batch that cannot be allocated"""
    for (_, n, size, codec, _), name in zip(frames, names):
        if size > FD.max_decoded_size(codec, n):
            raise BagError(f"{path}: {name} cannot be read: it declares {size} decompressed bytes, more than its {n} compressed "
                           f"bytes can hold{hint}")
    try:
        out, offs, status = FD.decode_frames(src, frames)
    except (MemoryError, _lib.VlcalError) as e:
        raise BagError(f"{path}: decoding its {len(frames)} compressed frames ({sum(f[2] for f in frames)} bytes) failed: {e}") from e
    for name, st in zip(names, status):
        if st != FD.OK:
            raise BagError(f"{path}: {name} cannot be read: {FD.STATUS_REASONS[int(st)]}{hint}")
    return out, offs


# ---- MCAP -------------------------------------------------------------------------------------------------------------

MCAP_MAGIC = b"\x89MCAP0\r\n"
_MCAP_HEADER, _MCAP_FOOTER, _MCAP_SCHEMA, _MCAP_CHANNEL, _MCAP_MESSAGE, _MCAP_CHUNK, _MCAP_DATA_END = 0x01, 0x02, 0x03, 0x04, 0x05, 0x06, 0x0F


class _Cursor:
    """Little-endian fields of one MCAP record; running past its end is a truncated record."""

    def __init__(self, buf, pos, end, where):
        self.b, self.p, self.end, self.where = buf, pos, end, where

    def take(self, n):
        if self.p + n > self.end:
            raise BagError(f"{self.where()}: a record ends inside one of its fields")
        v = self.b[self.p:self.p + n]
        self.p += n
        return v

    def u(self, fmt):
        return struct.unpack(fmt, self.take(struct.calcsize(fmt)))[0]

    def string(self):
        return bytes(self.take(self.u("<I"))).decode(errors="replace")


class McapBag:
    """One MCAP file of a rosbag2 bag, read whole.

    The layout is written from memory of the MCAP specification and has not been checked against a file written by the
    mcap library; check it against a real rosbag2 MCAP recording when one is at hand.  Magic `89 4D 43 41 50 30 0D 0A`
    at both ends; records `opcode u8, length u64, content`, strings `u32 length + bytes`.  Read: Schema 0x03 (id u16,
    name, encoding, data), Channel 0x04 (id u16, schema_id u16, topic, message_encoding, metadata), Message 0x05
    (channel_id u16, sequence u32, log_time u64, publish_time u64, data), Chunk 0x06 (message_start_time u64,
    message_end_time u64, uncompressed_size u64, uncompressed_crc u32, compression, records u64 + bytes); DataEnd 0x0F
    (or a Footer 0x02) ends the data section.  Every other opcode is skipped by its length.  The data section is scanned
    linearly; the summary section is not read.

    Chunks compressed with zstd or lz4 (the LZ4 frame format) are decoded on the GPU, all those of the file in one
    call, when the file is opened; the CRC-32 of their content is checked when uncompressed_crc is not 0.  A message's
    type is its channel's schema name; a topic whose message_encoding is not `cdr` is refused when it is read.

    Order: messages come in log_time order; ties go by position -- first the file offset of the chunk that holds the
    message (of the message record itself outside chunks), then the message's offset inside the decompressed chunk.
    This is meant to mirror the mcap library's log-time read order, which rosbag2 uses; that has not been checked
    against rosbag2."""

    def __init__(self, path: str):
        self.path = path
        with open(path, "rb") as f:
            size = os.fstat(f.fileno()).st_size
            buf = memoryview(mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)) if size else memoryview(b"")
        if bytes(buf[:8]) != MCAP_MAGIC:
            raise BagError(f"{path}: not an MCAP file (no magic); MCAP with uncompressed, zstd or lz4 chunks and sqlite3 are read; "
                           "convert other bags with `ros2 bag convert`")
        self._buf = buf
        self.schemas = {}   # id -> name
        self.channels = {}  # id -> (topic, schema id, message_encoding)
        self._index = []    # (log_time, position, inner offset, channel id, data)
        chunks = []         # (record offset, compression, uncompressed size, crc, compressed offset, compressed size)
        pos = 8
        while True:
            if pos + 9 > len(buf):
                raise BagError(f"{path}: truncated at byte {pos}: the data section ends without a DataEnd record")
            op, length = struct.unpack_from("<BQ", buf, pos)
            end = pos + 9 + length
            if end > len(buf):
                raise BagError(f"{path}: truncated inside the record at byte {pos} (opcode 0x{op:02x}, {length} bytes)")
            if op in (_MCAP_DATA_END, _MCAP_FOOTER):
                break
            if op == _MCAP_CHUNK:
                c = _Cursor(buf, pos + 9, end, lambda p=pos: f"{path}: the chunk at byte {p}")
                c.u("<Q"), c.u("<Q")
                usize, crc, comp = c.u("<Q"), c.u("<I"), c.string()
                data = c.take(c.u("<Q"))
                if comp == "":
                    self._records(data, pos)
                elif comp in ("zstd", "lz4"):
                    problem = (FD.zstd_header_problem if comp == "zstd" else FD.lz4_header_problem)(data)
                    if problem:
                        raise BagError(f"{path}: the {comp} chunk at byte {pos} cannot be read: {problem}")
                    chunks.append((pos, comp, usize, crc, c.p - len(data), len(data)))
                else:
                    raise BagError(f"{path}: the chunk at byte {pos} is compressed with '{comp}', which is not supported "
                                   "(only uncompressed, zstd and lz4 chunks are read); convert the bag with `ros2 bag convert`")
            else:
                self._record(op, buf, pos + 9, end, pos, 0)
            pos = end
        if chunks:
            frames = [(start, n, usize, FD.CODEC_ZSTD if comp == "zstd" else FD.CODEC_LZ4_FRAME, crc or None) for _, comp, usize, crc, start, n in chunks]
            out, offs = _decode(path, buf, frames, [f"the {comp} chunk at byte {pos}" for pos, comp, *_ in chunks])
            self._decoded = out  # messages of compressed chunks are views into it
            for (pos, _, usize, *_), o in zip(chunks, offs):
                self._records(memoryview(out)[o:o + usize], pos)
        self._index.sort(key=lambda e: (e[0], e[1], e[2]))

    def _records(self, data, chunk_pos):
        """the records of one chunk's content"""
        p = 0
        while p < len(data):
            if p + 9 > len(data):
                raise BagError(f"{self.path}: the chunk at byte {chunk_pos} ends inside a record header (offset {p} of its content)")
            op, length = struct.unpack_from("<BQ", data, p)
            if p + 9 + length > len(data):
                raise BagError(f"{self.path}: the chunk at byte {chunk_pos} is truncated inside the record at offset {p} of its content")
            self._record(op, data, p + 9, p + 9 + length, chunk_pos, p)
            p += 9 + length

    def _record(self, op, buf, start, end, pos, inner):
        where = lambda: f"{self.path}: byte {pos}" + (f", offset {inner} in its chunk" if inner else "")  # noqa: E731
        if op == _MCAP_SCHEMA:
            c = _Cursor(buf, start, end, where)
            sid, name = c.u("<H"), c.string()
            self.schemas.setdefault(sid, name)
        elif op == _MCAP_CHANNEL:
            c = _Cursor(buf, start, end, where)
            cid, sid, topic, enc = c.u("<H"), c.u("<H"), c.string(), c.string()
            self.channels.setdefault(cid, (topic, sid, enc))
        elif op == _MCAP_MESSAGE:
            c = _Cursor(buf, start, end, where)
            cid, _, log_time, _ = c.u("<H"), c.u("<I"), c.u("<Q"), c.u("<Q")
            self._index.append((log_time, pos, inner, cid, buf[c.p:end]))

    def _type(self, cid):
        return self.schemas.get(self.channels[cid][1], "")

    def topics_and_types(self):
        return [(self.channels[c][0], self._type(c)) for c in sorted(self.channels)]

    def messages(self, topic: str):
        """(datatype, raw message) of every message on `topic`, in log-time order (see the class docstring)."""
        for c, (t, _, enc) in self.channels.items():
            if t == topic and enc != "cdr":
                raise BagError(f"{self.path}: topic '{topic}' has message encoding '{enc}'; only cdr is read")
        for _, _, _, cid, data in self._index:
            ch = self.channels.get(cid)
            if ch is not None and ch[0] == topic:
                yield self._type(cid), data


# ---- ROS 2 ----------------------------------------------------------------------------------------------------------------

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
    # rosbag2 writes the mode in capitals (MESSAGE, FILE); neither value is read case-sensitively
    mode = re.search(r"compression_mode:\s*['\"]?(\w*)", text)
    fmt = re.search(r"compression_format:\s*['\"]?(\w*)", text)
    compression = ((mode.group(1) if mode else "").lower(), (fmt.group(1) if fmt else "").lower())
    return storage, files, compression


class Ros2Bag:
    """A ROS 2 bag: a directory holding metadata.yaml and the sqlite3 (*.db3) or MCAP (*.mcap) files it lists, read file
    by file.  With compression_mode `message` and compression_format `zstd` every message blob is one zstd frame; a
    topic's blobs of a file are decoded on the GPU in one call when the topic is read."""

    def __init__(self, path: str):
        self.path = path
        if not os.path.isfile(os.path.join(path, "metadata.yaml")):
            raise BagError(f"{path}: not a ROS 2 bag (no metadata.yaml)")
        storage, files, (mode, fmt) = _metadata(path)
        if storage not in ("sqlite3", "mcap"):
            raise BagError(f"{path}: storage '{storage}' is not supported, only sqlite3 and mcap (with uncompressed, zstd or lz4 "
                           "chunks); convert the bag with `ros2 bag convert` to storage_id sqlite3")
        if mode == "file":
            raise BagError(f"{path}: file-mode compression ({fmt}) is not supported; convert the bag with `ros2 bag convert` "
                           "to an uncompressed or message-compressed bag")
        if mode == "message" and fmt != "zstd":
            raise BagError(f"{path}: message compression '{fmt}' is not supported, only zstd; convert the bag with `ros2 bag convert`")
        self.storage = storage
        self.message_zstd = mode == "message"
        if not files:
            ext = ".db3" if storage == "sqlite3" else ".mcap"
            files = sorted(f for f in os.listdir(path) if f.endswith(ext))
        self.files = [os.path.join(path, f) for f in files]
        self._topics = []  # (name, type) over all files, first appearance
        self._mcap = (None, None)  # (path, McapBag): one MCAP file's decoded chunks are held at a time
        for fn in self.files:
            if storage == "mcap":
                pairs = self._mcap_file(fn).topics_and_types()
            else:
                with sqlite3.connect(f"file:{fn}?mode=ro", uri=True) as db:
                    pairs = list(db.execute("SELECT name, type FROM topics ORDER BY id"))
            for pair in pairs:
                if pair not in self._topics:
                    self._topics.append(pair)

    def topics_and_types(self):
        return list(self._topics)

    def _mcap_file(self, fn):
        """the McapBag of fn; opening another file releases the previous one (messages already handed out keep their
        own file's buffer alive)"""
        if self._mcap[0] != fn:
            self._mcap = (None, None)
            self._mcap = (fn, McapBag(fn))
        return self._mcap[1]

    def _file_messages(self, fn, topic):
        if self.storage == "mcap":
            yield from self._mcap_file(fn).messages(topic)
            return
        db = sqlite3.connect(f"file:{fn}?mode=ro", uri=True)
        try:
            q = ("SELECT t.type, m.data FROM messages m JOIN topics t ON m.topic_id = t.id WHERE t.name = ? "
                 "ORDER BY m.timestamp, m.id")
            for typ, data in db.execute(q, (topic,)):
                yield typ, memoryview(data)
        finally:
            db.close()

    def messages(self, topic: str):
        for fn in self.files:
            if not self.message_zstd:
                yield from self._file_messages(fn, topic)
                continue
            msgs = list(self._file_messages(fn, topic))
            yield from zip((t for t, _ in msgs), _decode_messages(fn, topic, [d for _, d in msgs]))


def _decode_messages(fn, topic, blobs):
    """the zstd-compressed message blobs of one topic of one file, decoded on the GPU in one call"""
    if not blobs:
        return []
    src = b"".join(bytes(b) for b in blobs)
    frames, off = [], 0
    for k, b in enumerate(blobs):
        problem = FD.zstd_header_problem(b)
        size = FD.zstd_content_size(b)
        if problem is None and size is None:
            problem = "its zstd frame does not declare its decompressed size"
        if problem:
            raise BagError(f"{fn}: message {k} on topic '{topic}' cannot be read: {problem}")
        frames.append((off, len(b), size, FD.CODEC_ZSTD, None))
        off += len(b)
    out, offs = _decode(fn, src, frames, [f"message {k} on topic '{topic}'" for k in range(len(frames))])
    view = memoryview(out)
    return [view[o:o + f[2]] for o, f in zip(offs, frames)]


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
