"""MCAP reading on the CPU (uncompressed chunks; nothing here needs a GPU): topics and types, the log-time order with its
ties across chunks and bare message records, bag directories of several files, unknown opcodes, and the refusals that
happen before any frame reaches the GPU decoder."""
import os
import struct

import pytest

import bag_writer as BW
import mcap_writer as MW
from direct_visual_lidar_calibration_b200 import bag_io as B


def _msgs(times, topics=("/a", "/b")):
    return [(topics[k % len(topics)], f"pkg/msg/T{k % len(topics)}", t, b"\x00\x01\x00\x00" + struct.pack("<I", k)) for k, t in enumerate(times)]


def _ids(seq):
    return [struct.unpack("<I", bytes(d[4:8]))[0] for _, d in seq]


def _expected(msgs, topic, per_chunk, unchunked):
    """file order (a group's bare records ahead of its chunk), then a stable sort by log time"""
    order = []
    for g in range(0, len(msgs), per_chunk):
        idx = range(g, min(g + per_chunk, len(msgs)))
        order += [i for i in idx if i in unchunked] + [i for i in idx if i not in unchunked]
    order.sort(key=lambda i: msgs[i][2])
    return [i for i in order if msgs[i][0] == topic]


def test_topics_types_and_order(tmp_path):
    times = [5, 1, 5, 3, 1, 5, 2, 5, 1, 5, 5, 0]
    msgs = _msgs(times)
    unchunked = {2, 7, 9}
    path = str(tmp_path / "a.mcap")
    MW.write_mcap(path, msgs, per_chunk=4, unchunked=unchunked)
    bag = B.McapBag(path)
    assert bag.topics_and_types() == [("/a", "pkg/msg/T0"), ("/b", "pkg/msg/T1")]
    for topic in ("/a", "/b"):
        got = list(bag.messages(topic))
        assert all(typ == ("pkg/msg/T0" if topic == "/a" else "pkg/msg/T1") for typ, _ in got)
        assert _ids(got) == _expected(msgs, topic, 4, unchunked)
    assert list(bag.messages("/none")) == []


def test_several_files_are_read_in_metadata_order(tmp_path):
    times = [10, 9, 8, 7, 6, 5, 4, 3]  # later files hold earlier times: files are not merged
    msgs = _msgs(times, topics=("/a",))
    d = str(tmp_path / "bag")
    MW.write_ros2_mcap(d, msgs, n_files=2, per_chunk=2, unchunked={1})
    bag = B.Ros2Bag(d)
    assert bag.topics_and_types() == [("/a", "pkg/msg/T0")]
    assert _ids(bag.messages("/a")) == [3, 2, 1, 0, 7, 6, 5, 4]
    assert B.is_ros2_bag(d) and isinstance(B.open_bag(d), B.Ros2Bag)


def test_unknown_and_skipped_opcodes(tmp_path):
    msgs = _msgs([1, 2, 3])
    extra = (MW.record(0x7E, b"\xff" * 17) + MW.record(0x09, b"\x00" * 40) + MW.record(0x0C, b"") + MW.record(0x0B, b"\x01" * 8)
             + MW.record(0x07, b"\x02" * 12) + MW.record(0x08, b"\x03" * 30))
    path = str(tmp_path / "x.mcap")
    MW.write_mcap(path, msgs, extra=extra)
    assert _ids(B.McapBag(path).messages("/a")) == [0, 2]


def test_refusals(tmp_path):
    msgs = _msgs([1, 2, 3, 4])
    path = str(tmp_path / "t.mcap")
    MW.write_mcap(path, msgs, per_chunk=2)
    with open(path, "rb") as f:
        full = f.read()
    # truncated inside a record: the file and the record's byte offset are named
    data_end = len(full) - len(MW.MAGIC) - len(MW.footer())  # the end of the DataEnd record
    for cut in list(range(9, data_end, 7)) + [data_end - 1]:
        with open(path, "wb") as f:
            f.write(full[:cut])
        with pytest.raises(B.BagError, match=r"t\.mcap: truncated.* at byte \d+"):
            B.McapBag(path)
    # not cdr
    MW.write_mcap(path, msgs, encoding="json")
    bag = B.McapBag(path)
    with pytest.raises(B.BagError, match=r"t\.mcap: topic '/a' has message encoding 'json'; only cdr"):
        list(bag.messages("/a"))
    # unknown compression, a zstd frame that needs a dictionary, an lz4 chunk without an LZ4 frame: before any GPU work
    records = MW.message(1, 0, 1, b"\x00\x01\x00\x00")
    head = MW.schema(1, "pkg/msg/T0") + MW.channel(1, 1, "/a")
    dict_frame = struct.pack("<I", 0xFD2FB528) + bytes([0x21, 0x07]) + b"\x00" * 8  # single segment, 1-byte dictionary id 7
    for comp, payload, match in (("bz2", b"BZh9", r"compressed with 'bz2'.*ros2 bag convert"),
                                 ("zstd", dict_frame, r"zstd chunk at byte \d+ cannot be read: it needs a zstd dictionary"),
                                 ("lz4", b"not an lz4 frame", r"lz4 chunk at byte \d+ cannot be read: it does not hold an LZ4 frame")):
        with open(path, "wb") as f:
            f.write(MW.file_bytes(head + MW.chunk(records, comp, payload=payload)))
        with pytest.raises(B.BagError, match=r"t\.mcap: .*" + match):
            B.McapBag(path)
    with open(path, "wb") as f:
        f.write(b"\x89MCAP0\r\n" + b"\x01")
    with pytest.raises(B.BagError, match=r"truncated at byte 8"):
        B.McapBag(path)


def test_rosbag2_compression_modes_refused_on_the_host(tmp_path):
    msgs = [("/p", "sensor_msgs/msg/PointCloud2", 1, b"\x00\x01\x00\x00")]
    d = str(tmp_path / "f")
    BW.write_ros2(d, msgs)
    with open(os.path.join(d, "metadata.yaml"), "a") as f:
        f.write("  compression_format: zstd\n  compression_mode: FILE\n")
    with pytest.raises(B.BagError, match=r"file-mode compression .*ros2 bag convert"):
        B.Ros2Bag(d)
    # message mode: a zstd frame without Frame_Content_Size is refused when the topic is read
    import codec_data as CD

    if not CD.have_zstd():
        pytest.skip("libzstd is not available to write the frames")
    d = str(tmp_path / "m")
    BW.write_ros2(d, [("/p", "sensor_msgs/msg/PointCloud2", 1, CD.zstd_compress(b"\x00\x01\x00\x00" * 50, content_size=False))])
    with open(os.path.join(d, "metadata.yaml"), "a") as f:
        f.write("  compression_format: zstd\n  compression_mode: message\n")
    with pytest.raises(B.BagError, match=r"message 0 on topic '/p' cannot be read: its zstd frame does not declare its decompressed size"):
        list(B.Ros2Bag(d).messages("/p"))


def test_declared_sizes_a_frame_cannot_hold_are_refused_before_decoding(tmp_path):
    """a chunk's uncompressed_size (or a message frame's content size) above what its compressed bytes can decode to is
    a BagError naming the file and the chunk, before anything is allocated"""
    head = MW.schema(1, "pkg/msg/T0") + MW.channel(1, 1, "/a")
    frame = struct.pack("<I", 0xFD2FB528) + bytes([0x20, 0x00]) + b"\x01\x00\x00"  # a 1-byte content size, an empty raw block
    body = struct.pack("<QQQI", 0, 0, 1 << 50, 0) + MW._str("zstd") + struct.pack("<Q", len(frame)) + frame
    path = str(tmp_path / "big.mcap")
    with open(path, "wb") as f:
        f.write(MW.file_bytes(head + MW.record(0x06, body)))
    with pytest.raises(B.BagError, match=r"big\.mcap: the zstd chunk at byte \d+ cannot be read: it declares 1125899906842624 decompressed bytes, "
                                         r"more than its 9 compressed bytes can hold"):
        B.McapBag(path)
    d = str(tmp_path / "m")
    big = struct.pack("<I", 0xFD2FB528) + bytes([0xE0]) + struct.pack("<Q", 1 << 40) + b"\x01\x00\x00"  # an 8-byte content size
    BW.write_ros2(d, [("/p", "sensor_msgs/msg/PointCloud2", 1, big)])
    with open(os.path.join(d, "metadata.yaml"), "a") as f:
        f.write("  compression_format: zstd\n  compression_mode: message\n")
    with pytest.raises(B.BagError, match=r"message 0 on topic '/p' cannot be read: it declares 1099511627776 decompressed bytes"):
        list(B.Ros2Bag(d).messages("/p"))
