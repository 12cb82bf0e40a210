"""An MCAP writer for the tests, and the compressed variants of the other bag forms: rosbag2 MCAP directories with
uncompressed, zstd or lz4 chunks, rosbag2 sqlite3 bags with per-message zstd, and ROS 1 bags with lz4 chunks.

It is written from the same memory of the MCAP specification as the reader (direct_visual_lidar_calibration_b200/
bag_io.py McapBag): a mistake shared by both would pass these tests.  Messages are (topic, type, time_ns, raw) as in
bag_writer; the CDR payloads come from bag_writer's helpers."""
import os
import struct
import zlib

import bag_writer as BW
import codec_data as CD

MAGIC = b"\x89MCAP0\r\n"


def _str(s):
    b = s.encode()
    return struct.pack("<I", len(b)) + b


def record(op, body):
    return struct.pack("<BQ", op, len(body)) + body


def header():
    return record(0x01, _str("ros2") + _str("vlcal tests"))


def schema(sid, name):
    return record(0x03, struct.pack("<H", sid) + _str(name) + _str("ros2msg") + struct.pack("<I", 0))


def channel(cid, sid, topic, encoding="cdr"):
    return record(0x04, struct.pack("<HH", cid, sid) + _str(topic) + _str(encoding) + struct.pack("<I", 0))


def message(cid, seq, t, data):
    return record(0x05, struct.pack("<HIQQ", cid, seq, t, t) + data)


def compress(data, compression, level=3):
    if compression == "":
        return data
    if compression == "zstd":
        return CD.zstd_compress(data, level)
    if compression == "lz4":
        return CD.lz4_compress(data, content_checksum=True)
    raise ValueError(compression)


def chunk(records, compression="", crc=True, payload=None):
    """A Chunk record of `records`; payload replaces the compressed bytes (for refusal tests)."""
    data = compress(records, compression) if payload is None else payload
    body = struct.pack("<QQQI", 0, 0, len(records), zlib.crc32(records) if crc else 0) + _str(compression) + struct.pack("<Q", len(data)) + data
    return record(0x06, body)


def data_end():
    return record(0x0F, struct.pack("<I", 0))


def footer():
    return record(0x02, struct.pack("<QQI", 0, 0, 0))


def file_bytes(body):
    return MAGIC + header() + body + data_end() + footer() + MAGIC


class _Ids:
    """schema and channel ids of the topics, and their records the first time a topic is used"""

    def __init__(self, encoding="cdr"):
        self.ids, self.encoding = {}, encoding

    def records(self, topic, typ):
        if (topic, typ) in self.ids:
            return b""
        k = len(self.ids) + 1
        self.ids[(topic, typ)] = k
        return schema(k, typ) + channel(k, k, topic, self.encoding)


def write_mcap(path, messages, compressions=("",), per_chunk=3, unchunked=(), encoding="cdr", extra=b""):
    """messages in chunks of `per_chunk`, the chunks' compressions cycling through `compressions`; the messages whose
    index is in `unchunked` are written as bare records ahead of the chunk they would have joined.  `extra` (records)
    goes right after the header."""
    ids = _Ids(encoding)
    body = bytearray(extra)
    seq = 0
    groups = [messages[i:i + per_chunk] for i in range(0, len(messages), per_chunk)]
    for g, group in enumerate(groups):
        inner = bytearray()
        for k, (topic, typ, t, raw) in enumerate(group):
            body += ids.records(topic, typ)
            rec = message(ids.ids[(topic, typ)], seq, t, raw)
            seq += 1
            if g * per_chunk + k in unchunked:
                body += rec
            else:
                inner += rec
        if inner:
            body += chunk(bytes(inner), compressions[g % len(compressions)])
    with open(path, "wb") as f:
        f.write(file_bytes(bytes(body)))


def _metadata(path, storage, files, n, compression=None):
    with open(os.path.join(path, "metadata.yaml"), "w") as f:
        f.write("rosbag2_bagfile_information:\n  version: 5\n  storage_identifier: " + storage + "\n  relative_file_paths:\n")
        for fn in files:
            f.write(f"    - {fn}\n")
        f.write(f"  message_count: {n}\n")
        if compression:
            f.write(f"  compression_format: {compression[1]}\n  compression_mode: {compression[0]}\n")


def write_ros2_mcap(path, messages, n_files=2, compressions=("",), per_chunk=3, unchunked=()):
    """A rosbag2 MCAP directory: the messages spread over n_files files in order."""
    os.makedirs(path, exist_ok=True)
    name = os.path.basename(path.rstrip("/"))
    files = [f"{name}_{k}.mcap" for k in range(n_files)]
    per = -(-len(messages) // n_files) if messages else 0
    for k, fn in enumerate(files):
        write_mcap(os.path.join(path, fn), messages[k * per:(k + 1) * per], compressions, per_chunk, unchunked)
    _metadata(path, "mcap", files, len(messages))


def write_ros2_message_zstd(path, messages, n_files=1, level=3, mode="MESSAGE"):
    """A rosbag2 sqlite3 bag whose message blobs are zstd frames (compression_mode: message)."""
    BW.write_ros2(path, [(t, ty, ts, CD.zstd_compress(raw, level)) for t, ty, ts, raw in messages], n_files=n_files)
    name = os.path.basename(path.rstrip("/"))
    _metadata(path, "sqlite3", [f"{name}_{k}.db3" for k in range(n_files)], len(messages), (mode, "zstd"))


def write_ros1_lz4(path, messages, per_chunk=3, **lz4_options):
    """bag_writer's ROS 1 bag with every chunk's records compressed into an LZ4 frame (compression=lz4)."""
    BW.write_ros1(path, messages, per_chunk=per_chunk)
    with open(path, "rb") as f:
        buf = f.read()
    out = bytearray(buf[:len(BW_VERSION)])
    pos = len(BW_VERSION)
    while pos < len(buf):
        (hl,) = struct.unpack_from("<I", buf, pos)
        h = buf[pos + 4:pos + 4 + hl]
        (dl,) = struct.unpack_from("<I", buf, pos + 4 + hl)
        data = buf[pos + 8 + hl:pos + 8 + hl + dl]
        fields = _fields(h)
        if fields.get("op") == b"\x05":
            fields["compression"] = b"lz4"
            data = CD.lz4_compress(data, **lz4_options)
            h = BW._hdr(fields)
        out += struct.pack("<I", len(h)) + h + struct.pack("<I", len(data)) + data
        pos += 8 + hl + dl
    with open(path, "wb") as f:
        f.write(bytes(out))


BW_VERSION = b"#ROSBAG V2.0\n"


def _fields(h):
    fields, p = {}, 0
    while p < len(h):
        (n,) = struct.unpack_from("<I", h, p)
        k, _, v = h[p + 4:p + 4 + n].partition(b"=")
        fields[k.decode()] = v
        p += 4 + n
    return fields
