"""Timing of preprocess_map's GPU stages on synthetic maps at a 2 mm leaf.

    python tools/preprocess_probe.py [--sizes 10000000,100000000] [--reps 5] [--oracle-size 10000000] [--out FILE]

Per map size: the kernel time of each stage between CUDA events (voxel grid keys / sort / runs / order, equalisation,
FoV grid), median of `reps` runs after one warm-up, and the wall time of the in-memory pipeline (voxel grid, equalisation,
FoV estimate with the host hull, LiDAR-image render; host<->device copies included, file I/O excluded).  Also the
single-thread time of the sequential CPU checker (tests/cpp/preprocess_oracle.c) for the same point stages on the
`--oracle-size` map, and the card name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def synthetic_map(n: int, seed: int = 0) -> np.ndarray:
    """A 40 x 40 x 8 m room: walls, floor and ceiling plus clutter inside, with 1.5 mm noise, float32 (n, 4).  At a 2 mm
    leaf almost every point keeps a voxel of its own, so the outputs are as large as the inputs."""
    rng = np.random.default_rng(seed)
    out = np.empty((n, 4), np.float32)
    chunk = 1 << 23
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        u = rng.random((m, 3), dtype=np.float32)
        face = rng.integers(0, 7, m)
        p = np.empty((m, 3), np.float32)
        p[:, 0] = (u[:, 0] - 0.5) * 40.0
        p[:, 1] = (u[:, 1] - 0.5) * 40.0
        p[:, 2] = (u[:, 2] - 0.3) * 8.0
        p[face == 0, 2], p[face == 1, 2] = -2.4, 5.6
        p[face == 2, 0], p[face == 3, 0] = -20.0, 20.0
        p[face == 4, 1], p[face == 5, 1] = -20.0, 20.0
        p[:, :] += rng.normal(0.0, 0.0015, (m, 3)).astype(np.float32)
        out[s : s + m, :3] = p
        out[s : s + m, 3] = rng.uniform(0.0, 255.0, m).astype(np.float32)
    return out


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def probe(n: int, reps: int):
    from direct_visual_lidar_calibration_b200 import create_camera, generate_lidar_image
    from direct_visual_lidar_calibration_b200 import preprocess as P

    cloud = synthetic_map(n)
    runs = []
    for r in range(reps + 1):
        t0 = time.perf_counter()
        avg, eq, fov = {}, {}, {}
        filtered = P.approximate_voxel_grid(cloud, 0.002, stats=avg)
        inten = P.equalize_intensities(filtered[:, 3], stats=eq)
        lidar_fov = P.estimate_lidar_fov(filtered[:, :3], stats=fov)
        model, intr, size, T = P.virtual_lidar_camera(lidar_fov)
        generate_lidar_image(create_camera(model, intr, []), size, T, filtered[:, :3].astype(np.float64), inten)
        wall = time.perf_counter() - t0
        if r:  # the first run warms up
            runs.append({"voxel_grid_ms": avg["stage_ms"], "equalize_ms": eq["kernel_ms"], "fov_grid_ms": fov["kernel_ms"], "wall_s": wall})
    med = lambda xs: float(np.median(xs))  # noqa: E731
    return {
        "points": n, "filtered": int(filtered.shape[0]), "fov_deg": float(np.degrees(lidar_fov)), "virtual_camera": model,
        "voxel_grid_stage_ms": {k: med([r["voxel_grid_ms"][i] for r in runs]) for i, k in enumerate(("keys", "sort", "runs", "order"))},
        "equalize_ms": med([r["equalize_ms"] for r in runs]), "fov_grid_ms": med([r["fov_grid_ms"] for r in runs]),
        "pipeline_wall_s": med([r["wall_s"] for r in runs]), "reps": reps,
    }


def oracle_time(n: int):
    import preprocess_oracle as PO

    cloud = synthetic_map(n)
    PO.lib()
    t0 = time.perf_counter()
    filtered = PO.approximate_voxel_grid(cloud, 0.002)
    t1 = time.perf_counter()
    PO.rank_equalize(filtered[:, 3])
    t2 = time.perf_counter()
    PO.voxel_grid_fov(filtered[:, :3])
    t3 = time.perf_counter()
    return {"points": n, "voxel_grid_s": t1 - t0, "equalize_s": t2 - t1, "fov_grid_s": t3 - t2, "total_s": t3 - t0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000000,100000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-size", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, limit = card()
    result = {"device": name, "power_limit": limit, "gpu": [probe(int(s), args.reps) for s in args.sizes.split(",")]}
    if args.oracle_size > 0:
        result["cpu_checker_single_thread"] = oracle_time(args.oracle_size)
    text = json.dumps(result, indent=2)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
