"""vlcal_decode_frames: a batch of zstd / LZ4-frame compressed frames decoded on the GPU (DESIGN §4f), and the header
checks the bag readers make on the host before they hand frames to it."""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np

from . import _lib

CODEC_ZSTD = 1
CODEC_LZ4_FRAME = 2

OK, CORRUPT, CHECKSUM, SIZE, UNSUPPORTED = range(5)
STATUS_REASONS = {
    CORRUPT: "the compressed data is corrupt",
    CHECKSUM: "a checksum does not match",
    SIZE: "it does not decode to the size the container declares",
    UNSUPPORTED: "it uses a dictionary, the legacy LZ4 format or a window above 2 GiB, which are not supported",
}

ZSTD_MAGIC = 0xFD2FB528
LZ4_MAGIC = 0x184D2204
LZ4_LEGACY_MAGIC = 0x184C2102


def _skippable(magic: int) -> bool:
    return magic & 0xFFFFFFF0 == 0x184D2A50


def _first_frame(buf) -> tuple[int, int]:
    """(magic, offset) of the first frame that is not a skippable frame; (-1, -1) when there is none."""
    p = 0
    while p + 4 <= len(buf):
        (magic,) = struct.unpack_from("<I", buf, p)
        if not _skippable(magic):
            return magic, p
        if p + 8 > len(buf):
            break
        p += 8 + struct.unpack_from("<I", buf, p + 4)[0]
    return -1, -1


def zstd_header_problem(buf) -> str | None:
    """Why the first zstd frame of buf cannot be decoded here, judged from its header alone; None when it can be tried."""
    magic, p = _first_frame(buf)
    if magic != ZSTD_MAGIC or p + 5 > len(buf):
        return "it does not start with a zstd frame"
    fhd = buf[p + 4]
    q = p + 5 + (0 if fhd & 0x20 else 1)
    n = (0, 1, 2, 4)[fhd & 3]
    if q + n > len(buf):
        return "its zstd frame header is truncated"
    if n and int.from_bytes(bytes(buf[q:q + n]), "little"):
        return "it needs a zstd dictionary, which is not supported"
    return None


def zstd_content_size(buf) -> int | None:
    """Frame_Content_Size of the first zstd frame of buf, None when the header does not carry it."""
    magic, p = _first_frame(buf)
    if magic != ZSTD_MAGIC or p + 5 > len(buf):
        return None
    fhd = buf[p + 4]
    fcs_flag, single = fhd >> 6, (fhd >> 5) & 1
    q = p + 5 + (0 if single else 1) + (0, 1, 2, 4)[fhd & 3]
    n = (single, 2, 4, 8)[fcs_flag]
    if n == 0 or q + n > len(buf):
        return None
    v = int.from_bytes(bytes(buf[q:q + n]), "little")
    return v + 256 if n == 2 else v


def lz4_header_problem(buf) -> str | None:
    """Why the first LZ4 frame of buf cannot be decoded here, judged from its header alone; None when it can be tried."""
    magic, p = _first_frame(buf)
    if magic == LZ4_LEGACY_MAGIC:
        return "it is in the legacy LZ4 format, which is not supported"
    if magic != LZ4_MAGIC or p + 6 > len(buf) or buf[p + 4] >> 6 != 1:
        return "it does not hold an LZ4 frame"
    if buf[p + 4] & 1:
        return "it needs an LZ4 dictionary, which is not supported"
    return None


def max_decoded_size(codec: int, src_size: int) -> int:
    """The most bytes src_size compressed bytes can decode to: a zstd block takes at least 4 bytes (a 3-byte header
    and an RLE byte) and writes at most 128 KiB; an LZ4 sequence writes at most 255 bytes more per byte it takes."""
    return (src_size // 4 + 1) * 131072 if codec == CODEC_ZSTD else 256 * src_size + 65536


def decode_frames(src, frames, device: int = -1, stats: dict | None = None):
    """Decodes frames = [(src_offset, src_size, dst_size, codec, crc32 or None)] of the bytes-like src on the GPU, in
    one call.  -> (dst, offsets, status): the outputs laid end to end in a uint8 array, frame i's at
    dst[offsets[i]:offsets[i] + dst_size], and its status (OK, CORRUPT, CHECKSUM, SIZE, UNSUPPORTED).  stats, when
    given, receives the copy-in, kernel and copy-out times in ms."""
    L = _lib.load_library()
    s = np.frombuffer(src, dtype=np.uint8) if len(src) else np.zeros(1, np.uint8)
    n = len(frames)
    arr = (_lib.Frame * max(n, 1))()
    offsets = np.zeros(n, np.int64)
    total = 0
    for i, (so, ss, ds, codec, crc) in enumerate(frames):
        arr[i] = _lib.Frame(so, ss, total, ds, codec, 0 if crc is None else 1, 0 if crc is None else crc, 0)
        offsets[i] = total
        total += ds
    dst = np.empty(max(total, 1), np.uint8)
    status = np.zeros(max(n, 1), np.int32)
    ms = (C.c_double * 3)()
    _lib.check(L.vlcal_decode_frames(device, s.ctypes.data, len(src), arr, n, dst.ctypes.data, total, status.ctypes.data_as(C.POINTER(C.c_int32)), ms))
    if stats is not None:
        stats.update(h2d_ms=ms[0], kernel_ms=ms[1], d2h_ms=ms[2])
    return dst[:total], offsets, status[:n]
