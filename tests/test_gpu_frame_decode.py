"""GPU checks of vlcal_decode_frames (csrc/frame_decode.cu): the committed fixtures and a seeded batch of thousands of
mixed frames decode to their plaintext byte for byte; the corrupted fixtures get the statuses the host build of the same
core gives (tests/test_codec_host.py runs that set under the sanitizers); the warp's CRC-32 accepts the right value and
rejects a wrong one; invalid arguments are refused on the host before any GPU work."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

import codec_data as CD
from direct_visual_lidar_calibration_b200 import _lib as VL
from direct_visual_lidar_calibration_b200 import frame_decode as FD

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def fixtures():
    return CD.load_fixtures(GOLDEN)


def _batch(items, crcs=None):
    """items: [(codec, frame, dst_size)] -> (outputs, status) from one vlcal_decode_frames call"""
    src = b"".join(f for _, f, _ in items)
    frames, off = [], 0
    for k, (codec, f, size) in enumerate(items):
        frames.append((off, len(f), size, codec, None if crcs is None else crcs[k]))
        off += len(f)
    st = {}
    dst, offs, status = FD.decode_frames(src, frames, stats=st)
    assert st["kernel_ms"] > 0.0
    return [dst[o:o + s].tobytes() for o, (_, _, s) in zip(offs, items)], status


def test_fixtures(gpu, fixtures):
    outs, status = _batch([(codec, frame, len(plain)) for _, codec, frame, plain, _ in fixtures])
    for (name, _, _, plain, _), out, st in zip(fixtures, outs, status):
        assert st == 0 and out == plain, name


@pytest.mark.skipif(not (CD.have_zstd() and CD.have_lz4()), reason="libzstd / liblz4 not available to write frames")
def test_seeded_mixed_batch(gpu):
    rng = np.random.default_rng(21)
    items, plains = [], []
    for k in range(3000):
        kind = CD.KINDS[k % 4]
        size = int(rng.choice([0, 1, 65536, 131073, 786432]) if rng.random() < 0.1 else rng.integers(0, 60000))
        plain = CD.plaintext(kind, size, 5000 + k)
        if rng.random() < 0.6:
            items.append((1, CD.zstd_compress(plain, int(rng.choice([-5, 1, 3, 9, 19])), checksum=bool(rng.random() < 0.5)), len(plain)))
        else:
            items.append((2, CD.lz4_compress(plain, independent=bool(rng.random() < 0.5), content_checksum=bool(rng.random() < 0.5),
                                             block_checksum=bool(rng.random() < 0.5)), len(plain)))
        plains.append(plain)
    crcs = [zlib.crc32(p) if k % 3 == 0 else None for k, p in enumerate(plains)]
    outs, status = _batch(items, crcs)
    assert np.all(status == 0)
    for k, (out, plain) in enumerate(zip(outs, plains)):
        assert out == plain, k


@pytest.fixture(scope="module")
def host_checker(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path_factory.mktemp("codec") / "frame_decode_check")
    subprocess.run([nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", f"-I{os.path.join(ROOT, 'direct_visual_lidar_calibration_b200', 'csrc')}", "-o", exe,
                    os.path.join(ROOT, "tests", "cpp", "frame_decode_check.cu")], check=True)
    return exe


def test_corrupted_statuses_equal_the_host_build(gpu, fixtures, host_checker, tmp_path):
    cases = CD.corruptions(fixtures)
    items = [(codec, frame, len(fixtures[i][3])) for i, codec, frame, _ in cases]
    path = str(tmp_path / "cases.bin")
    with open(path, "wb") as f:
        for codec, frame, size in items:
            f.write(struct.pack("<IQQ", codec, len(frame), size) + frame)
    r = subprocess.run([host_checker, "decode", path], capture_output=True, text=True, check=True)
    host = [int(ln.split()[0]) for ln in r.stdout.splitlines()]
    _, status = _batch(items)
    assert len(host) == len(items) and status.tolist() == host
    assert sum(s != 0 for s in host) > 0.8 * len(items)


def test_crc32(gpu, fixtures):
    picks = [f for f in fixtures if len(f[3]) in (0, 1, 20000, 131071, 4 << 20)][:24]
    assert any(len(p[3]) == 4 << 20 for p in picks)
    items = [(codec, frame, len(plain)) for _, codec, frame, plain, _ in picks]
    good = [zlib.crc32(p[3]) for p in picks]
    _, status = _batch(items, good)
    assert np.all(status == 0)
    _, status = _batch(items, [c ^ (1 << (k % 32)) for k, c in enumerate(good)])
    assert np.all(status == 2)


def test_argument_refusals(gpu):
    L = VL.load_library()
    src = np.zeros(64, np.uint8)
    dst = np.zeros(64, np.uint8)
    status = np.zeros(4, np.int32)

    def call(frames, src_bytes=64, dst_bytes=64):
        arr = (VL.Frame * len(frames))(*[VL.Frame(*f) for f in frames])
        return L.vlcal_decode_frames(0, src.ctypes.data, src_bytes, arr, len(frames), dst.ctypes.data, dst_bytes, status.ctypes.data_as(C.POINTER(C.c_int32)), None)

    ok = (0, 8, 0, 8, 1, 0, 0, 0)
    for bad in [(0, 8, 0, 8, 3, 0, 0, 0), (0, 8, 0, 8, 1, 2, 0, 0), (60, 8, 0, 8, 1, 0, 0, 0), (-1, 8, 0, 8, 1, 0, 0, 0), (0, 8, 60, 8, 2, 0, 0, 0),
                (0, 8, 0, -1, 1, 0, 0, 0), (0, 8, 4, 8, 1, 0, 0, 0)]:
        assert call([ok, bad]) == VL.ERR_INVALID_ARGUMENT, bad
        assert "decode_frames" in L.vlcal_nid_last_error().decode()
    assert call([ok, (8, 8, 8, 8, 2, 0, 0, 0), (16, 0, 3, 0, 1, 0, 0, 0)]) == VL.OK  # adjacent and empty ranges are fine
    assert list(status[:3]) == [1, 1, 1]  # zero bytes are not a frame
    assert call([ok], src_bytes=-1) == VL.ERR_INVALID_ARGUMENT
    assert L.vlcal_decode_frames(0, None, 0, None, 0, None, 0, None, None) == VL.OK
