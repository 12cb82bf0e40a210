"""Measures `preprocess` from bags: the decode + static integration kernels at 10^7 and 10^8 points (CUDA events), the
single-thread sequential checker at 10^7 points, and the whole pipeline's wall time on a ROS 1 bag directory with the
share spent reading bags and writing files.  Prints one JSON line; `--out FILE` also writes it there.

    python tools/bag_preprocess_probe.py [--out results.json]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bag_oracle as BO  # noqa: E402
import bag_writer as BW  # noqa: E402
from direct_visual_lidar_calibration_b200 import _lib as VL  # noqa: E402
from direct_visual_lidar_calibration_b200 import preprocess_bag as PB  # noqa: E402
from direct_visual_lidar_calibration_b200 import synthetic as S  # noqa: E402


def _scans(n, n_scans, rng):
    per = n // n_scans
    parts, descs, off = [], [], 0
    for _ in range(n_scans):
        xyz = rng.uniform(-30.0, 30.0, (per, 3)).astype(np.float32)
        data, fields, step = BW.cloud_bytes(xyz, rng.uniform(0, 100, per).astype(np.float32), "<f4", "<f4")
        f = {nm: (o, t) for nm, o, t in fields}
        descs.append(VL.ScanDesc(byte_offset=off, n_points=per, point_step=step, x_offset=f["x"][0], y_offset=f["y"][0], z_offset=f["z"][0],
                                 xyz_type=f["x"][1], intensity_offset=f["intensity"][0], intensity_type=f["intensity"][1]))
        parts.append(np.frombuffer(data, np.uint8))
        off += len(data)
    return np.concatenate(parts), descs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    args = ap.parse_args()
    rng = np.random.default_rng(1)
    res = {}
    for n in (10_000_000, 100_000_000):
        blob, descs = _scans(n, 100, rng)
        PB.bag_integrate(blob, descs, 0.002, 1.0)  # warm-up (pool, module load)
        best = None
        for _ in range(3):
            st = {}
            out = PB.bag_integrate(blob, descs, 0.002, 1.0, stats=st)
            tot = sum(st["stage_ms"])
            if best is None or tot < best[0]:
                best = (tot, st["stage_ms"])
        res[f"kernel_ms_{n}"] = round(best[0], 3)
        res[f"stage_ms_{n}"] = [round(v, 3) for v in best[1]]
        res[f"voxels_{n}"] = int(out.shape[0])
        if n == 10_000_000:
            t0 = time.perf_counter()
            BO.bag_integrate(blob, descs, 0.002, 1.0)
            res["checker_s_10000000"] = round(time.perf_counter() - t0, 3)
        del blob, descs
    # whole pipeline on a two-bag ROS 1 directory, 100 scans of 10^5 points each
    bag = S.make_bag("pinhole_640x480", "frustum", 1_000_000, config_index=9)
    with tempfile.TemporaryDirectory() as d:
        data = os.path.join(d, "bags")
        os.makedirs(data)
        K = bag["intrinsics"]
        k9 = [K[0], 0.0, K[2], 0.0, K[1], K[3], 0.0, 0.0, 1.0]
        for b in range(2):
            msgs = [("/ci", "sensor_msgs/CameraInfo", 1, BW.camera_info(1, 0, bag["width"], bag["height"], "plumb_bob", bag["distortion"], k9)),
                    ("/img", "sensor_msgs/Image", 1, BW.image(1, 0, bag["image"], "mono8"))]
            for k in range(100):
                sl = slice((k % 10) * 100_000, (k % 10 + 1) * 100_000)
                xyz = bag["points"][sl, :3].astype(np.float32) + np.float32(1e-3 * (k // 10))
                dat, fields, step = BW.cloud_bytes(xyz, bag["intensities"][sl].astype(np.float32), "<f4", "<f4")
                msgs.append(("/points", "sensor_msgs/PointCloud2", 2 + k, BW.point_cloud2(1 + k // 10, (k % 10) * 10**8, fields, dat, 100_000, point_step=step)))
            BW.write_ros1(os.path.join(data, f"bag{b}.bag"), msgs, per_chunk=10)
        st = {}
        t0 = time.perf_counter()
        PB.preprocess_bags(data, os.path.join(d, "out"), auto_topic=True, stats=st, log=lambda m: None)
        wall = time.perf_counter() - t0
    res["cli_wall_s_2x1e7"] = round(wall, 3)
    res["cli_io_s"] = round(st["io_s"], 3)
    res["cli_gpu_stage_s"] = round(st["gpu_s"], 3)
    res["cli_io_share"] = round(st["io_s"] / wall, 3)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
