"""Seeded plaintexts and the libzstd / liblz4 encoders (through ctypes) of the frame decoder's tests, its fixture script
and tools/decode_probe.py.  The product never loads either library; here they only write frames to decode."""
from __future__ import annotations

import ctypes as C
import ctypes.util
import struct

import numpy as np

KINDS = ("zeros", "random", "text", "cloud")

_WORDS = (b"lidar camera point cloud intensity edge voxel frame chunk topic stamp header sensor_msgs PointCloud2 ring time "
          b"reflectivity calibration the of and to in is").split()


def plaintext(kind: str, size: int, seed: int) -> bytes:
    """`size` bytes of the content kind: zeros, random bytes, repetitive text, PointCloud2-like float records."""
    rng = np.random.default_rng(seed)
    if kind == "zeros":
        return bytes(size)
    if kind == "random":
        return rng.integers(0, 256, size, dtype=np.uint8).tobytes()
    if kind == "text":  # a passage of ~2 KB repeated, one word in fifty replaced at random
        words = rng.integers(0, len(_WORDS), 300)
        out = bytearray()
        while len(out) < size:
            swap = rng.random(len(words)) < 0.02
            for w, s, r in zip(words, swap, rng.integers(0, len(_WORDS), len(words))):
                out += _WORDS[r if s else w] + b" "
        return bytes(out[:size])
    if kind == "cloud":  # x y z intensity (f4), ring (u2), pad (u2), time (f4): a slowly turning scan, quantized to mm
        n = size // 20 + 1
        a = np.cumsum(rng.normal(0.002, 0.0005, n)).astype(np.float64)
        r = 5.0 + np.round(rng.normal(0.0, 0.3, n), 3)
        rec = np.zeros(n, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("i", "<f4"), ("ring", "<u2"), ("pad", "<u2"), ("t", "<f4")])
        rec["x"], rec["y"] = np.round(r * np.cos(a), 3), np.round(r * np.sin(a), 3)
        rec["z"] = np.round(rng.normal(0.0, 0.5, n), 2)
        rec["i"] = rng.integers(0, 64, n)
        rec["ring"] = np.arange(n) % 32
        rec["t"] = np.arange(n, dtype=np.float32) * 1e-5
        return rec.tobytes()[:size]
    raise ValueError(kind)


def _load(name):
    path = ctypes.util.find_library(name)
    for cand in ([path] if path else []) + [f"lib{name}.so.1", f"lib{name}.so"]:
        try:
            return C.CDLL(cand)
        except OSError:
            continue
    return None


_zstd = _load("zstd")
_lz4 = _load("lz4")
if _zstd is not None:
    _zstd.ZSTD_compressBound.restype = C.c_size_t
    _zstd.ZSTD_compressBound.argtypes = [C.c_size_t]
    _zstd.ZSTD_isError.argtypes = [C.c_size_t]
    _zstd.ZSTD_createCCtx.restype = C.c_void_p
    _zstd.ZSTD_freeCCtx.argtypes = [C.c_void_p]
    _zstd.ZSTD_CCtx_setParameter.argtypes = [C.c_void_p, C.c_int, C.c_int]
    _zstd.ZSTD_CCtx_setParameter.restype = C.c_size_t
    _zstd.ZSTD_compress2.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    _zstd.ZSTD_compress2.restype = C.c_size_t
    _zstd.ZSTD_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    _zstd.ZSTD_decompress.restype = C.c_size_t
if _lz4 is not None:
    _lz4.LZ4F_compressFrameBound.restype = C.c_size_t
    _lz4.LZ4F_compressFrameBound.argtypes = [C.c_size_t, C.c_void_p]
    _lz4.LZ4F_compressFrame.restype = C.c_size_t
    _lz4.LZ4F_compressFrame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    _lz4.LZ4F_isError.argtypes = [C.c_size_t]


def have_zstd() -> bool:
    return _zstd is not None


def have_lz4() -> bool:
    return _lz4 is not None


_ZSTD_C_LEVEL, _ZSTD_C_CHECKSUM, _ZSTD_C_CONTENT_SIZE = 100, 201, 200


def zstd_compress(data: bytes, level: int = 3, checksum: bool = True, content_size: bool = True) -> bytes:
    cctx = _zstd.ZSTD_createCCtx()
    try:
        for p, v in ((_ZSTD_C_LEVEL, level), (_ZSTD_C_CHECKSUM, int(checksum)), (_ZSTD_C_CONTENT_SIZE, int(content_size))):
            if _zstd.ZSTD_isError(_zstd.ZSTD_CCtx_setParameter(cctx, p, v)):
                raise RuntimeError("ZSTD_CCtx_setParameter failed")
        cap = _zstd.ZSTD_compressBound(len(data))
        out = C.create_string_buffer(cap)
        n = _zstd.ZSTD_compress2(cctx, out, cap, data, len(data))
        if _zstd.ZSTD_isError(n):
            raise RuntimeError("ZSTD_compress2 failed")
        return out.raw[:n]
    finally:
        _zstd.ZSTD_freeCCtx(cctx)


def zstd_decompress(frame: bytes, size: int) -> bytes:
    out = C.create_string_buffer(max(size, 1))
    n = _zstd.ZSTD_decompress(out, size, frame, len(frame))
    if _zstd.ZSTD_isError(n):
        raise RuntimeError("ZSTD_decompress failed")
    return out.raw[:n]


class _LZ4FrameInfo(C.Structure):
    _fields_ = [("blockSizeID", C.c_int), ("blockMode", C.c_int), ("contentChecksumFlag", C.c_int), ("frameType", C.c_int),
                ("contentSize", C.c_ulonglong), ("dictID", C.c_uint), ("blockChecksumFlag", C.c_int)]


class _LZ4Prefs(C.Structure):
    _fields_ = [("frameInfo", _LZ4FrameInfo), ("compressionLevel", C.c_int), ("autoFlush", C.c_uint), ("favorDecSpeed", C.c_uint),
                ("reserved", C.c_uint * 3)]


def lz4_compress(data: bytes, independent: bool = False, content_checksum: bool = False, block_checksum: bool = False, content_size: bool = False,
                 block_size_id: int = 4, level: int = 0) -> bytes:
    """An LZ4 frame; block_size_id 4..7: 64 KiB, 256 KiB, 1 MiB, 4 MiB blocks."""
    prefs = _LZ4Prefs()
    prefs.frameInfo.blockSizeID = block_size_id
    prefs.frameInfo.blockMode = int(independent)
    prefs.frameInfo.contentChecksumFlag = int(content_checksum)
    prefs.frameInfo.blockChecksumFlag = int(block_checksum)
    prefs.frameInfo.contentSize = len(data) if content_size else 0
    prefs.compressionLevel = level
    cap = _lz4.LZ4F_compressFrameBound(len(data), C.byref(prefs))
    out = C.create_string_buffer(cap)
    n = _lz4.LZ4F_compressFrame(out, cap, data, len(data), C.byref(prefs))
    if _lz4.LZ4F_isError(n):
        raise RuntimeError("LZ4F_compressFrame failed")
    return out.raw[:n]


def skippable(payload: bytes, nibble: int = 0) -> bytes:
    return struct.pack("<II", 0x184D2A50 | nibble, len(payload)) + payload


# ---- the committed fixtures and their corrupted variants ------------------------------------------------------------

def load_fixtures(golden_dir):
    """[(name, codec id (1 zstd, 2 lz4), frame bytes, plaintext, has a checksum over the content)] of codec_fixtures.*;
    plaintexts come from codec_data.plaintext (seeded) or, for the hand-built frames, from codec_data.hand_built"""
    import json
    import os

    with open(os.path.join(golden_dir, "codec_fixtures.json")) as f:
        manifest = json.load(f)
    with open(os.path.join(golden_dir, "codec_fixtures.bin"), "rb") as f:
        blob = f.read()
    out = []
    hand = {name: plain for name, _, plain in hand_built()}
    for e in manifest:
        if e["generator"] == "codec_data.hand_built":
            plain = hand[e["name"]]
        else:
            plain = b"".join(plaintext(p["kind"], p["size"], p["seed"]) for p in e["parts"])
        o = e["options"]
        checked = o.get("checksum", False) if e["codec"] == "zstd" else o.get("content_checksum", False)
        out.append((e["name"], 1 if e["codec"] == "zstd" else 2, blob[e["offset"]:e["offset"] + e["size"]], plain, checked))
    return out


def corruptions(fixtures, cuts=9, flips=12, seed=5):
    """[(fixture index, codec, damaged frame, what)]: each fixture truncated at `cuts` points (the first and last byte
    among them) and with `flips` single-bit flips, all seeded"""
    rng = np.random.default_rng(seed)
    out = []
    for i, (_, codec, frame, _, _) in enumerate(fixtures):
        n = len(frame)
        for cut in sorted({0, 1, n - 1, *rng.integers(0, max(n, 1), cuts - 3).tolist()}):
            if 0 <= cut < n:
                out.append((i, codec, frame[:cut], f"cut {cut}"))
        for bit in rng.integers(0, 8 * n, flips).tolist():
            b = bytearray(frame)
            b[bit // 8] ^= 1 << (bit % 8)
            out.append((i, codec, bytes(b), f"flip {bit}"))
    return out


def lz4_decompress(frame: bytes, size: int) -> bytes:
    """one LZ4 frame through liblz4's frame decoder (for host timings)"""
    ctx = C.c_void_p()
    if _lz4.LZ4F_isError(_lz4.LZ4F_createDecompressionContext(C.byref(ctx), 100)):
        raise RuntimeError("LZ4F_createDecompressionContext failed")
    try:
        out = C.create_string_buffer(max(size, 1))
        dst_n, src_n = C.c_size_t(size), C.c_size_t(len(frame))
        r = _lz4.LZ4F_decompress(ctx, out, C.byref(dst_n), frame, C.byref(src_n), None)
        if _lz4.LZ4F_isError(r) or dst_n.value != size:
            raise RuntimeError("LZ4F_decompress failed")
        return out.raw[:size]
    finally:
        _lz4.LZ4F_freeDecompressionContext(ctx)


if _lz4 is not None:
    _lz4.LZ4F_createDecompressionContext.argtypes = [C.POINTER(C.c_void_p), C.c_uint]
    _lz4.LZ4F_createDecompressionContext.restype = C.c_size_t
    _lz4.LZ4F_freeDecompressionContext.argtypes = [C.c_void_p]
    _lz4.LZ4F_decompress.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p]
    _lz4.LZ4F_decompress.restype = C.c_size_t


# ---- hand-built zstd frames: paths the encoder at any level rarely takes -------------------------------------------

def _zstd_frame(blocks, content_size):
    """a single-segment zstd frame with a 4-byte content size; blocks: [(type, content bytes, decompressed size for RLE)]"""
    out = bytearray(struct.pack("<IB", 0xFD2FB528, 0xA0) + struct.pack("<I", content_size))
    for k, (typ, content, rle_size) in enumerate(blocks):
        size = rle_size if typ == 1 else len(content)
        out += (((size << 3) | (typ << 1) | (k == len(blocks) - 1))).to_bytes(3, "little") + content
    return bytes(out)


def _rle_literals(regen, byte):
    """a compressed block of RLE literals and no sequences, with the 1-, 2- or 3-byte literals header regen needs"""
    if regen < 32:
        head = bytes([1 | (regen << 3)])
    elif regen < 4096:
        head = bytes([1 | (1 << 2) | ((regen & 15) << 4), regen >> 4])
    else:
        head = bytes([1 | (3 << 2) | ((regen & 15) << 4), (regen >> 4) & 0xFF, regen >> 12])
    return head + bytes([byte, 0])


def hand_built():
    """[(name, frame, plaintext)]: RLE literals with every header size; RLE mode for all three sequence tables with a
    3-byte Number_of_Sequences and the repeat-offset shift of literal length 0; Huffman weights given directly"""
    out = []
    sizes = (20, 1000, 100000)
    plain = b"".join(bytes([0x78 + k]) * n for k, n in enumerate(sizes))
    out.append(("zstd_hand_rle_literals", _zstd_frame([(2, _rle_literals(n, 0x78 + k), 0) for k, n in enumerate(sizes)], len(plain)), plain))

    nseq = 32600  # >= 0x7F00: the 3-byte form; every sequence is LL code 0, OF code 0, ML code 0 from RLE tables
    block = bytes([0x00, 0xFF]) + struct.pack("<H", nseq - 0x7F00) + bytes([0x54, 0, 0, 0, 0x01])
    buf, rep = bytearray(b"abcdefgh"), [1, 4, 8]
    for _ in range(nseq):  # offset value 1 with literal length 0 is repeat offset 2, swapped to the front
        off = rep[1]
        rep[0], rep[1] = rep[1], rep[0]
        for _ in range(3):
            buf.append(buf[-off])
    out.append(("zstd_hand_rle_tables_3byte_nseq", _zstd_frame([(0, b"abcdefgh", 0), (2, block, 0)], len(buf)), bytes(buf)))

    # four symbols, weights 2, 1, 1 given directly (the last, 3, implied): codes 01, 000, 001, 1
    rng = np.random.default_rng(77)
    lits = rng.choice(4, 300, p=[0.25, 0.125, 0.125, 0.5]).astype(np.uint8).tobytes()
    codes = {0: (0b01, 2), 1: (0b000, 3), 2: (0b001, 3), 3: (0b1, 1)}
    acc, nbits = 0, 0
    for s in reversed(lits):  # the decoder reads the stream from its end: the first literal is written last
        v, n = codes[s]
        acc |= v << nbits
        nbits += n
    acc |= 1 << nbits
    stream = acc.to_bytes(nbits // 8 + 1, "little")
    tree = bytes([127 + 3, (2 << 4) | 1, 1 << 4])
    csize = len(tree) + len(stream)
    head = (2 | (len(lits) << 4) | (csize << 14)).to_bytes(3, "little")
    out.append(("zstd_hand_direct_huffman_weights", _zstd_frame([(2, head + tree + stream + b"\x00", 0)], len(lits)), lits))
    return out
