"""CPU checks of the zstd / LZ4-frame decoder core (csrc/frame_decode.cuh): tests/cpp/frame_decode_check.cu is the same
source the GPU kernel runs, built host-only under AddressSanitizer and UndefinedBehaviorSanitizer.  Every committed
fixture decodes to its regenerated plaintext; a seeded fuzz over levels, content kinds and sizes where libzstd / liblz4
load; every fixture truncated and bit-flipped ends in a non-ok status (or, where the damage is harmless or nothing
checks the content, in any output) without a sanitizer report; XXH32, XXH64 and CRC-32 against known values, the
libraries' own checksums and zlib.  tests/test_gpu_frame_decode.py repeats the decoding and the statuses on the GPU."""
import os
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

import codec_data as CD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "direct_visual_lidar_calibration_b200", "csrc")
GOLDEN = os.path.join(ROOT, "tests", "golden")
SAN_ENV = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("codec") / "frame_decode_check")
    san = ["-Xcompiler", "-fsanitize=address", "-Xcompiler", "-fsanitize=undefined", "-Xcompiler", "-fno-sanitize-recover=all", "-Xcompiler", "-fno-omit-frame-pointer"]
    subprocess.run([nvcc, "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", *san, f"-I{CSRC}", "-o", exe,
                    os.path.join(ROOT, "tests", "cpp", "frame_decode_check.cu")], check=True)
    return exe


@pytest.fixture(scope="module")
def fixtures():
    return CD.load_fixtures(GOLDEN)


def decode(checker, tmp_path, cases):
    """cases: [(codec, frame, dst_size)] -> [(status, produced, crc32 of the dst_size output bytes)]; fails on any
    sanitizer report"""
    path = str(tmp_path / "cases.bin")
    with open(path, "wb") as f:
        for codec, frame, size in cases:
            f.write(struct.pack("<IQQ", codec, len(frame), size) + frame)
    r = subprocess.run([checker, "decode", path], capture_output=True, text=True, env=SAN_ENV)
    assert r.returncode == 0 and "ERROR" not in r.stderr and "runtime error" not in r.stderr, r.stderr[-4000:]
    out = [tuple(int(v) for v in ln.split()) for ln in r.stdout.splitlines()]
    assert len(out) == len(cases)
    return out


def test_fixtures_decode_to_their_plaintext(checker, fixtures, tmp_path):
    assert len(fixtures) > 150
    assert sum(len(f[2]) for f in fixtures) < 1 << 20
    res = decode(checker, tmp_path, [(codec, frame, len(plain)) for _, codec, frame, plain, _ in fixtures])
    for (name, _, _, plain, _), (st, produced, crc) in zip(fixtures, res):
        assert (st, produced, crc) == (0, len(plain), zlib.crc32(plain)), name
    # the fixture set reaches what it is meant to: both codecs, multi-block and empty outputs, every zstd level
    names = [f[0] for f in fixtures]
    assert any(n.startswith("zstd_l19_zeros_4194304") for n in names) and any(n.startswith("lz4_ind_c1b1_zeros_4194304") for n in names)
    assert {f"zstd_l{lv}_" for lv in (-5, 1, 3, 9, 19)} <= {n[: n.index("_", 5) + 1] for n in names if n.startswith("zstd_l")}
    # hand-built: RLE literals (1-, 2- and 3-byte headers), RLE mode for LL / OF / ML with a 3-byte sequence count,
    # Huffman weights given directly -- paths libzstd's levels do not reach in the seeded fixtures
    assert {"zstd_hand_rle_literals", "zstd_hand_rle_tables_3byte_nseq", "zstd_hand_direct_huffman_weights"} <= set(names)


def test_decode_frames_argument_refusals_without_a_gpu():
    """vlcal_decode_frames checks its ranges on the host before it looks for a device: overlapping dst ranges are refused
    even with an empty range sorted between them or with equal offsets"""
    import ctypes as C

    from direct_visual_lidar_calibration_b200 import _lib as VL

    L = VL.load_library()
    src, dst, status = np.zeros(256, np.uint8), np.zeros(256, np.uint8), np.zeros(8, np.int32)

    def call(dst_ranges):
        arr = (VL.Frame * len(dst_ranges))(*[VL.Frame(0, 8, o, n, 1, 0, 0, 0) for o, n in dst_ranges])
        return L.vlcal_decode_frames(0, src.ctypes.data, 256, arr, len(dst_ranges), dst.ctypes.data, 256, status.ctypes.data_as(C.POINTER(C.c_int32)), None)

    for ranges in ([(0, 100), (10, 0), (20, 10)], [(0, 100), (50, 0), (60, 0), (99, 1)], [(0, 10), (0, 10)], [(5, 10), (0, 0), (5, 1)],
                   [(0, 200), (100, 10), (150, 10)], [(40, 10), (0, 100)]):
        assert call(ranges) == VL.ERR_INVALID_ARGUMENT, ranges
        assert "overlap" in L.vlcal_nid_last_error().decode()


def test_size_mismatch_and_unsupported(checker, fixtures, tmp_path):
    name, codec, frame, plain, _ = next(f for f in fixtures if f[0] == "zstd_l3_text_131073")
    res = decode(checker, tmp_path, [(codec, frame, len(plain) - 1), (codec, frame, len(plain) + 1), (codec, b"", 0), (2, frame, len(plain)),
                                     (1, struct.pack("<I", 0x184C2102) + b"\0" * 8, 0), (2, struct.pack("<I", 0x184C2102) + b"\0" * 8, 0)])
    assert [r[0] for r in res] == [3, 3, 1, 1, 1, 4]
    # a zstd dictionary id, an LZ4 DictID: unsupported
    zd = struct.pack("<I", 0xFD2FB528) + bytes([0x21, 0x07, 0x05]) + b"\x01\x00\x00"
    fl = bytearray(next(f for f in fixtures if f[0].startswith("lz4_linked_c0b0_text_1"))[2])
    fl[4] |= 1  # DictID flag; the header checksum is rewritten so that the dictionary is what stops it
    fl = bytes(fl[:6]) + b"\x01\x00\x00\x00" + bytes([(_xxh32(checker, tmp_path, bytes(fl[4:6]) + b"\x01\x00\x00\x00") >> 8) & 0xFF]) + bytes(fl[7:])
    assert [r[0] for r in decode(checker, tmp_path, [(1, zd, 5), (2, fl, 1)])] == [4, 4]


def _hashes(checker, tmp_path, blobs):
    path = str(tmp_path / "hash.bin")
    with open(path, "wb") as f:
        for b in blobs:
            f.write(struct.pack("<Q", len(b)) + b)
    r = subprocess.run([checker, "hash", path], capture_output=True, text=True, env=SAN_ENV, check=True)
    return [tuple(int(v) for v in ln.split()) for ln in r.stdout.splitlines()]


def _xxh32(checker, tmp_path, b):
    return _hashes(checker, tmp_path, [b])[0][0]


def test_checksums(checker, fixtures, tmp_path):
    rng = np.random.default_rng(3)
    blobs = [b"", b"a", b"abc"] + [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in (3, 15, 16, 17, 31, 32, 33, 63, 1000, 70001)]
    res = _hashes(checker, tmp_path, blobs)
    for b, (x32, x64, crc, joined) in zip(blobs, res):
        assert crc == joined == zlib.crc32(b)
    # published XXH32 / XXH64 values of the empty input and of "abc" (seed 0)
    assert (res[0][0], res[0][1]) == (0x02CC5D05, 0xEF46DB3751D8E999)
    assert (res[2][0], res[2][1]) == (0x32D153FF, 0x44BC2CF5AD770999)
    # checksums the libraries wrote verify (zstd: XXH64 content checksum; LZ4: XXH32 header, block and content checksums) ...
    checked = [f for f in fixtures if f[4] or "b1_" in f[0]]
    assert len(checked) > 40
    assert all(r[0] == 0 for r in decode(checker, tmp_path, [(c, fr, len(p)) for _, c, fr, p, _ in checked]))
    # ... and a changed content checksum, or LZ4 header checksum, is a checksum mismatch (status 2)
    cases = []
    for _, codec, frame, plain, has in fixtures:
        if has and len(plain) > 0 and "concatenated" not in _:
            b = bytearray(frame)
            b[-1] ^= 0x40
            cases.append((codec, bytes(b), len(plain)))
        if codec == 2:
            b = bytearray(frame)
            hc = 6 + (8 if b[4] & 8 else 0)
            b[hc] ^= 0x01
            cases.append((codec, bytes(b), len(plain)))
    assert len(cases) > 60
    assert all(r[0] == 2 for r in decode(checker, tmp_path, cases))


def test_corruption_sweep(checker, fixtures, tmp_path):
    cases = CD.corruptions(fixtures)
    res = decode(checker, tmp_path, [(codec, frame, len(fixtures[i][3])) for i, codec, frame, _ in cases])
    bad = 0
    for (i, _, frame, what), (st, _, crc) in zip(cases, res):
        name, _, _, plain, checked = fixtures[i]
        if what.startswith("cut"):
            assert st != 0, (name, what)  # a truncated frame never decodes to the full size
        elif st == 0 and checked:
            assert crc == zlib.crc32(plain), (name, what)  # a checked frame decodes to its plaintext or fails
        bad += st != 0
    assert bad > 0.8 * len(cases)


@pytest.mark.skipif(not (CD.have_zstd() and CD.have_lz4()), reason="libzstd / liblz4 not available to write frames")
def test_seeded_fuzz(checker, tmp_path):
    rng = np.random.default_rng(11)
    cases, plains = [], []
    for k in range(2500):
        kind = CD.KINDS[k % 4]
        size = int(rng.choice([0, 1, 2, 3, 7, 64, 1000, 4095, 65536, 65537, 131071, 131072, 131073, 200000, 300001]) if rng.random() < 0.4
                   else rng.integers(0, 40000))
        plain = CD.plaintext(kind, size, 1000 + k)
        if k % 2 == 0:
            frame = CD.zstd_compress(plain, int(rng.choice([-7, -5, -1, 1, 2, 3, 5, 7, 9, 12, 15, 19])), checksum=bool(rng.random() < 0.5),
                                     content_size=bool(rng.random() < 0.8))
            codec = 1
        else:
            frame = CD.lz4_compress(plain, independent=bool(rng.random() < 0.5), content_checksum=bool(rng.random() < 0.5),
                                    block_checksum=bool(rng.random() < 0.5), content_size=bool(rng.random() < 0.5),
                                    block_size_id=int(rng.integers(4, 8)), level=int(rng.choice([0, 3, 9, 12])))
            codec = 2
        cases.append((codec, frame, len(plain)))
        plains.append(plain)
    res = decode(checker, tmp_path, cases)
    for k, ((st, produced, crc), plain) in enumerate(zip(res, plains)):
        assert (st, produced, crc) == (0, len(plain), zlib.crc32(plain)), k
