"""Times the headless viewer's kernels (csrc/viewer.cu and the z-buffer passes of csrc/lidar_image.cu) at the C2 size
(10^6 points, 1920 x 1080 plumb_bob) and the C3 size (5 * 10^6 points, 3840 x 1920 equirectangular): the colourise
kernel, and the overlay (init + project + winner + compose) for point radius 0, 1 and 2, between CUDA events inside the
library, after a warm-up call of every shape.  The read-back of the colours (16 bytes per point) is timed on its own,
between CUDA events around a device-to-host copy of the same size, and is not part of any kernel time.  Prints one JSON
line per size with the GPU's name and power limit.  Fails without a GPU.

    python tools/viewer_probe.py [--repeats 7]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from direct_visual_lidar_calibration_b200 import PointsColorUpdater, create_camera, device_count, render_overlay  # noqa: E402
from direct_visual_lidar_calibration_b200 import synthetic as S  # noqa: E402

SIZES = {"C2": ("pinhole_1920x1080", "os1_64", 1_000_000), "C3": ("equirect_3840x1920", "avia", 5_000_000)}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def d2h_ms(nbytes, repeats):
    """Device-to-host copy of nbytes into pageable and into pinned memory, ms (median), between CUDA events."""
    import torch

    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = {}
    for kind, dst in (("pageable", torch.empty(nbytes, dtype=torch.uint8)), ("pinned", torch.empty(nbytes, dtype=torch.uint8).pin_memory())):
        ms = []
        for it in range(repeats + 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dst.copy_(src)
            b.record()
            b.synchronize()
            if it:  # the first copy warms up
                ms.append(a.elapsed_time(b))
        out[kind] = float(np.median(ms))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    if device_count() < 1:
        raise SystemExit("viewer_probe: no CUDA device visible; nothing to time")
    gpu = gpu_info()
    w = float(np.float32(0.7))
    for name, (camera_key, pattern, n) in SIZES.items():
        model, intr, dist, W, H = S.CAMERAS[camera_key]
        pts, inten = S.make_cloud(pattern, n, scene_seed=71, seed=72)
        image = np.random.default_rng(73).integers(0, 256, (H, W), dtype=np.uint8)
        T = S.gt_T_camera_lidar()
        cam = create_camera(model, intr, dist)
        upd = PointsColorUpdater(cam, image, pts, inten)
        colors = upd.update(T, w)  # warm-up (module load, pool)
        ms, wall = [], []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            again = upd.update(T, w)
            wall.append((time.perf_counter() - t0) * 1e3)
            ms.append(upd.kernel_ms)
            assert np.array_equal(again.view(np.uint32), colors.view(np.uint32))
        k = float(np.median(ms))
        row = {
            "gpu": gpu, "size": name, "model": model, "points": n, "image": [W, H], "coloured_fraction": float((colors[:, 3] != 0).mean()),
            "colorize_kernel_ms_median": k, "colorize_kernel_ms_min": float(np.min(ms)),
            # 16 B of float4 read and 16 B of RGBA written per point, one image byte gathered per coloured point
            "colorize_bytes_per_point": 32, "colorize_image_bytes": W * H, "colorize_GBps": (32.0 * n + W * H) / (k * 1e-3) / 1e9,
            "colorize_call_wall_ms_median": float(np.median(wall)),  # with the upload of cloud and image and the read-back
            "colors_d2h_ms": d2h_ms(16 * n, args.repeats), "colors_d2h_bytes": 16 * n,
        }
        for radius in (0, 1, 2):
            bgr, index, _ = render_overlay(cam, image, T, pts, inten, radius, w, return_kernel_ms=True)  # warm-up
            ms = []
            for _ in range(args.repeats):
                b2, i2, k = render_overlay(cam, image, T, pts, inten, radius, w, return_kernel_ms=True)
                assert np.array_equal(i2, index) and np.array_equal(b2, bgr)
                ms.append(k)
            row[f"overlay_r{radius}_kernels_ms_median"] = float(np.median(ms))
            row[f"overlay_r{radius}_kernels_ms_min"] = float(np.min(ms))
            row[f"overlay_r{radius}_covered_pixels"] = int((index >= 0).sum())
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
