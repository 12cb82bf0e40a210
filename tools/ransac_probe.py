"""Times the RANSAC scoring launch of PoseEstimation (csrc/pose_estimation.cu) for 8192 hypotheses x M correspondences,
M in {1e3, 1e4, 1e5}, with CUDA events around the launch, next to the CPU checker (tests/cpp/pose_oracle.c, OpenMP) on
a subset of the same hypotheses, whose counts must agree.  Prints one JSON line per M with the GPU's name and power limit.

    python tools/ransac_probe.py [--model plumb_bob] [--repeats 5] [--oracle-hypotheses 256]"""
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

import pose_oracle  # noqa: E402
import util  # noqa: E402
from direct_visual_lidar_calibration_b200 import create_camera, device_count  # noqa: E402
from direct_visual_lidar_calibration_b200 import pose_estimation as PE  # noqa: E402
from direct_visual_lidar_calibration_b200 import synthetic as S  # noqa: E402
from oracle import oracle as O  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def problem(model, m, seed=0):
    intr, dist, (W, H) = util.CAMERAS[model]
    rng = np.random.default_rng(seed)
    T = S.gt_T_camera_lidar()
    pts = (S.lidar_directions("avia", m, rng) * rng.uniform(1.0, 30.0, (m, 1))).astype(np.float32).astype(np.float64)
    ocam = O.create_camera(model, intr, dist)
    kp = np.array([O.project(ocam, p) for p in pts @ T[:3, :3].T + T[:3, 3]]) + rng.normal(0.0, 1.0, (m, 2))
    out = rng.random(m) < 0.3
    kp[out] = rng.uniform([0, 0], [W, H], (int(out.sum()), 2))
    return intr, dist, kp, pts, ocam


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="plumb_bob", choices=util.MODELS)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--oracle-hypotheses", type=int, default=256)
    args = ap.parse_args()
    if device_count() < 1:
        raise SystemExit("ransac_probe: no CUDA device visible; nothing to time")
    gpu = gpu_info()
    pose_oracle.lib()  # compile the checker before anything is timed
    for m in (1_000, 10_000, 100_000):
        intr, dist, kp, pts, ocam = problem(args.model, m)
        cam = create_camera(args.model, intr, dist)
        pairs = PE.sample_pairs(m, 8192)
        timing = {}
        counts, _ = PE.score_pairs(cam, kp, pts, pairs, 5.0, timing=timing)  # warm-up (module load)
        ms = []
        for _ in range(args.repeats):
            c, _ = PE.score_pairs(cam, kp, pts, pairs, 5.0, timing=timing)
            assert np.array_equal(c, counts)
            ms.append(timing["kernel_ms"])
        sub = pairs[: args.oracle_hypotheses]
        t0 = time.perf_counter()
        ref, _, near = pose_oracle.score(ocam, kp, pts, sub, 5.0)
        cpu_s = time.perf_counter() - t0  # bearings (NelderMead per correspondence) and the scoring of the subset
        agree = bool(np.all(np.abs(counts[: sub.shape[0]].astype(np.int64) - ref) <= near))
        print(json.dumps({
            "gpu": gpu, "model": args.model, "hypotheses": 8192, "M": m, "kernel_ms_median": float(np.median(ms)), "kernel_ms_min": float(np.min(ms)),
            "projections_per_s": 8192 * m / (np.median(ms) * 1e-3), "cpu_oracle_hypotheses": int(sub.shape[0]), "cpu_oracle_s": cpu_s,
            "cpu_oracle_threads": os.cpu_count(), "counts_agree": agree, "best_count": int(counts.max()),
        }), flush=True)


if __name__ == "__main__":
    main()
