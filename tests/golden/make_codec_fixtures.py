"""Writes the frame decoder's committed fixtures with libzstd / liblz4 (through ctypes; tests/codec_data.py):

    codec_fixtures.bin   the compressed frames end to end
    codec_fixtures.json  per frame: codec, byte range, and the generator, kind, size and seed of its plaintext
                         (codec_data.plaintext), which the tests regenerate instead of storing it
    mcap_bag/            a small rosbag2 MCAP bag with zstd chunks: camera info, a mono8 image and PointCloud2 scans of a
                         synthetic scene, so the end-to-end test runs where libzstd is absent

zstd frames at levels -5, 1, 3, 9 and 19, LZ4 frames with and without each checksum in linked and independent mode, over
zeros, random bytes, repetitive text and PointCloud2-like records of 0, 1, 128 KiB +- 1 and 4 MiB (multi-block) bytes,
plus concatenated and skippable frames, and the hand-built zstd frames of codec_data.hand_built (RLE literals, RLE
sequence tables with a 3-byte sequence count, Huffman weights given directly), each checked against libzstd.  Run from the repository root: python tests/golden/make_codec_fixtures.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import codec_data as CD  # noqa: E402

K128 = 128 * 1024


def cases():
    """(name, codec, [(kind, size, seed)] of the concatenated plaintext parts, encoder options)"""
    out = []
    seed = 100
    for level in (-5, 1, 3, 9, 19):
        for kind in CD.KINDS:
            sizes = [0, 1, K128 - 1, K128, K128 + 1]
            if kind == "zeros":
                sizes.append(4 << 20)
            if kind == "random":
                sizes = [0, 1, 4000]
            if kind == "cloud":  # float records barely compress: small ones keep the fixtures small
                sizes = [1, 20000]
            for size in sizes:
                seed += 1
                out.append((f"zstd_l{level}_{kind}_{size}", "zstd", [(kind, size, seed)], {"level": level, "checksum": (seed % 2) == 0}))
    for independent in (False, True):
        for csum in (False, True):
            for bsum in (False, True):
                for kind in ("zeros", "text", "cloud", "random"):
                    same = csum == bsum  # both checksums or neither: the larger sizes only there
                    sizes = {"random": [1, 4000], "cloud": [1, 20000] if same else [1], "text": [0, 1, K128 + 1] if same and csum == independent else [0, 1, 5000]}.get(
                        kind, [0, 1, K128 - 1, K128 + 1])
                    if kind == "random" and independent and csum and bsum:
                        sizes.append(20000)
                    if kind == "zeros" and same and csum == independent:
                        sizes.append(4 << 20)
                    for size in sizes:
                        seed += 1
                        opts = {"independent": independent, "content_checksum": csum, "block_checksum": bsum, "content_size": (seed % 3) == 0}
                        out.append((f"lz4_{'ind' if independent else 'linked'}_c{int(csum)}b{int(bsum)}_{kind}_{size}", "lz4", [(kind, size, seed)], opts))
    out.append(("zstd_concatenated_with_skippable", "zstd", [("text", 5000, 900), ("cloud", 7000, 901), ("zeros", 300, 902)], {"level": 3, "checksum": True}))
    out.append(("lz4_concatenated_with_skippable", "lz4", [("text", 5000, 903), ("cloud", 20000, 904)], {"content_checksum": True}))
    out.append(("lz4_256k_blocks", "lz4", [("text", 300000, 905)], {"block_size_id": 5, "block_checksum": True}))
    return out


def encode(codec, parts, opts):
    blobs = []
    for k, (kind, size, seed) in enumerate(parts):
        plain = CD.plaintext(kind, size, seed)
        frame = CD.zstd_compress(plain, **opts) if codec == "zstd" else CD.lz4_compress(plain, **opts)
        if len(parts) > 1:  # a skippable frame ahead of every part but the first, and one at the end
            blobs.append(CD.skippable(b"skip" * k, nibble=k) if k else b"")
        blobs.append(frame)
    if len(parts) > 1:
        blobs.append(CD.skippable(b"", nibble=15))
    return b"".join(blobs)


def write_mcap_bag(path):
    import numpy as np

    import bag_writer as BW
    import mcap_writer as MW
    from direct_visual_lidar_calibration_b200 import synthetic as S

    bag = S.make_bag("pinhole_640x480", "frustum", 10_000, config_index=9)
    K = np.asarray(bag["intrinsics"]) / 2.0  # the image at half size keeps the bag small
    k9 = [K[0], 0.0, K[2], 0.0, K[1], K[3], 0.0, 0.0, 1.0]
    img = bag["image"].reshape(bag["height"] // 2, 2, bag["width"] // 2, 2).mean(axis=(1, 3)).round().astype(np.uint8)
    msgs = [("/camera/camera_info", "sensor_msgs/msg/CameraInfo", 10**9,
             BW.camera_info(1, 0, bag["width"] // 2, bag["height"] // 2, "plumb_bob", bag["distortion"], k9, cdr=True)),
            ("/camera/image", "sensor_msgs/msg/Image", 10**9, BW.image(1, 0, img, "mono8", cdr=True))]
    n = bag["points"].shape[0]
    inten = np.round(bag["intensities"] * 200.0).astype(np.float32)
    for k in range(6):
        sl = slice(k * n // 6, (k + 1) * n // 6)
        pts = np.round(bag["points"][sl, :3], 3).astype(np.float32)  # mm: the scans compress
        data, fields, step = BW.cloud_bytes(pts, inten[sl], "<f4", "<f4")
        msgs.append(("/points", "sensor_msgs/msg/PointCloud2", 10**9 + k * 10**8,
                     BW.point_cloud2(1, k * 10**8, fields, data, sl.stop - sl.start, point_step=step, cdr=True)))
    MW.write_ros2_mcap(path, msgs, n_files=1, compressions=("zstd",), per_chunk=2)


def main():
    manifest, blob = [], bytearray()
    for name, codec, parts, opts in cases():
        frame = encode(codec, parts, opts)
        manifest.append({"name": name, "codec": codec, "offset": len(blob), "size": len(frame), "generator": "codec_data.plaintext",
                         "parts": [{"kind": k, "size": s, "seed": sd} for k, s, sd in parts], "options": opts})
        blob += frame
    for name, frame, plain in CD.hand_built():
        assert CD.zstd_decompress(frame, len(plain)) == plain, name  # libzstd agrees with the hand-built frame
        manifest.append({"name": name, "codec": "zstd", "offset": len(blob), "size": len(frame), "generator": "codec_data.hand_built",
                         "parts": [], "options": {}})
        blob += frame
    with open(os.path.join(HERE, "codec_fixtures.bin"), "wb") as f:
        f.write(bytes(blob))
    with open(os.path.join(HERE, "codec_fixtures.json"), "w") as f:
        json.dump(manifest, f, separators=(",", ":"))
    write_mcap_bag(os.path.join(HERE, "mcap_bag"))
    print(f"{len(manifest)} frames, {len(blob)} bytes")


if __name__ == "__main__":
    main()
