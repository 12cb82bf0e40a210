"""GPU probe of the frame decoder (csrc/frame_decode.cu, DESIGN §4f): a seeded PointCloud2-like workload of about 2 GiB
cut into 768 KiB chunks (MCAP's default chunk size), compressed with zstd level 1, zstd level 3 and lz4 (the LZ4 frame
format) through libzstd / liblz4.  Reports per codec: the kernel time between CUDA events (median of repeated calls after
a warm-up) with the output GB/s, the whole vlcal_decode_frames call with its copies, and one host core of libzstd /
liblz4 on the same frames; then `preprocess` wall time on a seeded sqlite3 bag and on the same bag as MCAP with zstd
chunks; and the card's name and power limit, read in the same run.  Prints JSON lines; --out also writes them to a file.

    python tools/decode_probe.py [--gib 2.0] [--repeats 5] [--out result.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import codec_data as CD  # noqa: E402
from direct_visual_lidar_calibration_b200 import frame_decode as FD  # noqa: E402

CHUNK = 768 * 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi failed)"


def workload(gib):
    n = max(1, int(gib * (1 << 30)) // CHUNK)
    return [CD.plaintext("cloud", CHUNK, 70_000 + k) for k in range(n)]


def measure(name, plains, frames, codec, repeats):
    src = b"".join(frames)
    desc, off = [], 0
    for f, p in zip(frames, plains):
        desc.append((off, len(f), len(p), codec, zlib.crc32(p) if codec == FD.CODEC_ZSTD else None))
        off += len(f)
    total = sum(len(p) for p in plains)
    FD.decode_frames(src, desc)  # warm-up
    kernel, call = [], []
    for _ in range(repeats):
        st = {}
        t0 = time.perf_counter()
        dst, offs, status = FD.decode_frames(src, desc, stats=st)
        call.append((time.perf_counter() - t0) * 1e3)
        kernel.append(st["kernel_ms"])
        assert np.all(status == 0)
    assert all(dst[o:o + CHUNK].tobytes() == p for o, p in zip(offs[:: max(1, len(plains) // 16)], plains[:: max(1, len(plains) // 16)]))
    t0 = time.perf_counter()
    for f, p in zip(frames, plains):
        (CD.zstd_decompress if codec == FD.CODEC_ZSTD else CD.lz4_decompress)(f, len(p))
    host_ms = (time.perf_counter() - t0) * 1e3
    k, c = float(np.median(kernel)), float(np.median(call))
    return {"codec": name, "frames": len(frames), "uncompressed_bytes": total, "compressed_bytes": len(src), "ratio": total / len(src),
            "kernel_ms": k, "kernel_gbps": total / k / 1e6, "call_ms": c, "call_gbps": total / c / 1e6, "host_1core_ms": host_ms,
            "host_1core_gbps": total / host_ms / 1e6, "kernel_ms_all": kernel}


def preprocess_times():
    import bag_writer as BW
    import mcap_writer as MW
    from direct_visual_lidar_calibration_b200 import preprocess as cli
    from direct_visual_lidar_calibration_b200 import synthetic as S

    bag = S.make_bag("pinhole_640x480", "frustum", 2_000_000, config_index=9)
    K = bag["intrinsics"]
    k9 = [K[0], 0.0, K[2], 0.0, K[1], K[3], 0.0, 0.0, 1.0]
    msgs = [("/camera/camera_info", "sensor_msgs/msg/CameraInfo", 10**9, BW.camera_info(1, 0, bag["width"], bag["height"], "plumb_bob", bag["distortion"], k9, cdr=True)),
            ("/camera/image", "sensor_msgs/msg/Image", 10**9, BW.image(1, 0, np.repeat(bag["image"][:, :, None], 3, axis=2), "bgr8", cdr=True))]
    n = bag["points"].shape[0]
    for k in range(40):
        sl = slice(k * n // 40, (k + 1) * n // 40)
        data, fields, step = BW.cloud_bytes(bag["points"][sl, :3].astype(np.float32), (bag["intensities"][sl] * 200).astype(np.float32), "<f4", "<f4")
        msgs.append(("/points", "sensor_msgs/msg/PointCloud2", 10**9 + k * 10**7, BW.point_cloud2(1, k * 10**7, fields, data, sl.stop - sl.start, point_step=step, cdr=True)))
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for form in ("sqlite3", "mcap_zstd"):
            root = os.path.join(tmp, form)
            os.makedirs(root)
            if form == "sqlite3":
                BW.write_ros2(os.path.join(root, "bag0"), msgs)
            else:
                MW.write_ros2_mcap(os.path.join(root, "bag0"), msgs, n_files=1, compressions=("zstd",), per_chunk=1)
            times = []
            for r in range(3):
                dst = os.path.join(tmp, f"{form}_out{r}")
                t0 = time.perf_counter()
                assert cli.main([root, dst, "-a"]) == 0
                times.append(time.perf_counter() - t0)
            out[form] = {"wall_s_median_of_3": float(np.median(times)), "wall_s": times}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not (CD.have_zstd() and CD.have_lz4()):
        sys.exit("decode_probe: libzstd and liblz4 are needed to write the workload and time the host decoders; neither may be missing")
    info = {"card": card()}
    plains = workload(args.gib)
    results = []
    for name, codec, enc in (("zstd-1", FD.CODEC_ZSTD, lambda p: CD.zstd_compress(p, 1, checksum=False)),
                             ("zstd-3", FD.CODEC_ZSTD, lambda p: CD.zstd_compress(p, 3, checksum=False)),
                             ("lz4", FD.CODEC_LZ4_FRAME, lambda p: CD.lz4_compress(p, content_checksum=False))):
        frames = [enc(p) for p in plains]
        results.append(measure(name, plains, frames, codec, args.repeats))
        print(json.dumps({k: v for k, v in results[-1].items() if k != "kernel_ms_all"}), flush=True)
    del plains
    info.update(decode=results, preprocess=preprocess_times(), card_after=card())
    print(json.dumps(info["preprocess"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)
    print(json.dumps({"card": info["card"]}))


if __name__ == "__main__":
    main()
