"""Measurements behind initial_guess_search (DESIGN.md section 4e), one command on one GPU:

    python tools/initial_guess_search_probe.py [--skip_crossover] [--skip_basins] [--skip_search]

1. the pose sweep kernel against vlcal_nid_score_poses (the persistent kernel's pose-list mode) on the same seeded inputs,
   alternating, N in {8 k, 16 k, 64 k, 256 k, 1 M} x P in {10^3, 10^5}: CUDA-event kernel time of the sweep, wall time of
   both calls (upload and download included, as a caller pays them), point-poses/s and the crossover N;
2. the NID basin around the ground truth at every level of the search, per rotation axis and per translation axis, for
   the synthetic pinhole and equirectangular bags: the half-width is the largest offset up to which the NID still grows
   monotonically away from the truth;
3. a full search without a prior on both bags: per-level pose count, kernel and wall time, and the error of the result.
Outputs are compared before any time is printed.  Fails without a GPU."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import direct_visual_lidar_calibration_b200 as V  # noqa: E402
from direct_visual_lidar_calibration_b200 import _lib  # noqa: E402
from direct_visual_lidar_calibration_b200 import initial_guess as ig  # noqa: E402
from direct_visual_lidar_calibration_b200 import initial_guess_search as igs  # noqa: E402
from direct_visual_lidar_calibration_b200 import io as vio  # noqa: E402
from direct_visual_lidar_calibration_b200 import synthetic as S  # noqa: E402
from direct_visual_lidar_calibration_b200.cost import score_poses  # noqa: E402

BAGS = {"pinhole": ("pinhole_1920x1080", "os1_64"), "equirectangular": ("equirect_3840x1920", "sphere")}


def card() -> str:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return out.stdout.strip().splitlines()[0]


def crossover():
    import util

    L = _lib.load_library()
    print("\n== sweep kernel vs vlcal_nid_score_poses (plumb_bob 640x480 at 16 bins; ms are medians of 3 alternating runs) ==")
    print(f"{'N':>8} {'P':>7} {'sweep kernel ms':>16} {'sweep call ms':>14} {'score_poses call ms':>20} {'sweep Gpp/s (kernel)':>21} {'score_poses Gpp/s (call)':>25}")
    wins = {}
    for n in (8192, 16384, 65536, 262144, 1048576):
        pr = util.random_problem("plumb_bob", n=n, seed=n)
        cam = V.create_camera(pr["model"], pr["intrinsics"], pr["distortion"])
        cost = V.CostCalculatorNID(cam, V.VisualLiDARData(pr["image"], pr["points"], pr["intensities"]))
        for P in (1000, 100000):
            if n * P > 3e10:  # the 1 M x 10^5 corner is minutes of the slower kernel; the trend is set below it
                continue
            rot = ig.rotation_set(3.0)
            Ts = rot.poses(np.random.default_rng(P).permutation(rot.n_poses)[:P])
            Ts[:, :3, 3] = pr["T"][:3, 3]
            a = ig.sweep_poses([cost], Ts, kernel_only=True)  # warm-up of both, and the comparison
            b = score_poses([cost], Ts)
            if not np.array_equal(a, b, equal_nan=True):
                raise SystemExit(f"sweep and score_poses differ at N={n} P={P}")
            tk, ts, tp = [], [], []
            for _ in range(3):
                t0 = time.perf_counter()
                ig.sweep_poses([cost], Ts, kernel_only=True)
                ts.append((time.perf_counter() - t0) * 1e3)
                tk.append(L.vlcal_nid_sweep_last_kernel_ms())
                t0 = time.perf_counter()
                score_poses([cost], Ts)
                tp.append((time.perf_counter() - t0) * 1e3)
            k, s, p = np.median(tk), np.median(ts), np.median(tp)
            print(f"{n:>8} {P:>7} {k:>16.2f} {s:>14.2f} {p:>20.2f} {n * P / k / 1e6:>21.2f} {n * P / p / 1e6:>25.2f}")
            wins[(n, P)] = s < p
        cost.close()
    for P in (1000, 100000):
        ns = sorted(n for (n, q) in wins if q == P)
        last = [n for n in ns if wins[(n, P)]]
        print(f"P = {P}: the sweep call is faster up to N = {max(last) if last else 'none'} of {ns}")
    print(f"threshold compiled into the library: {int(L.vlcal_nid_sweep_max_points())} points")


def basins(name, bag):
    scorer = igs.SweepScorer(bag["camera_model"], bag["intrinsics"], bag["distortion"], [V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])])
    rot_offsets = np.array([0.0, 0.25, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0, 8.0, 12.0])
    trans_offsets = np.array([0.0, 0.02, 0.05, 0.1, 0.15, 0.2, 0.3, 0.45, 0.6])
    print(f"\n== NID basin around the truth, {name} bag (half-width: offsets up to which NID grows monotonically, worst of +-) ==")
    for lv in igs.level_schedule(3.0, 0.3, 64):
        costs = scorer.costs(lv)
        line = [f"level {lv['index']} (1/{lv['scale']}, {min(lv['points'], bag['points'].shape[0])} pts):"]
        for kind, offsets, unit in (("rot", rot_offsets, "deg"), ("trans", trans_offsets, "m")):
            for axis in range(3):
                half = np.inf
                curve = None
                for sign in (1.0, -1.0):
                    Ts = []
                    for o in offsets:
                        v = np.zeros(3)
                        v[axis] = sign * o
                        Ts.append(S.perturb(bag["T_gt"], v if kind == "rot" else (0, 0, 0), v if kind == "trans" else (0, 0, 0)))
                    nid = ig.sweep_poses(costs, np.stack(Ts))
                    grow = np.diff(nid) > 0
                    stop = int(np.argmin(grow)) if not grow.all() else len(grow)
                    half = min(half, offsets[stop])
                    curve = nid if curve is None else curve
                line.append(f"{kind}{'xyz'[axis]} {half:g} {unit} (NID {curve[0]:.4f} -> {curve[-1]:.4f})")
        print("  " + "; ".join(line))
    scorer.close()


def full_search(name, bag):
    scorer = igs.SweepScorer(bag["camera_model"], bag["intrinsics"], bag["distortion"], [V.VisualLiDARData(bag["image"], bag["points"], bag["intensities"])])
    print(f"\n== full search without a prior, {name} bag ==")
    t0 = time.perf_counter()
    rep = igs.run_search(scorer, log=lambda *_: None)
    total = time.perf_counter() - t0
    scorer.close()
    for lv in rep["levels"]:
        pp = lv["poses"] * min(lv["points_per_bag"], bag["points"].shape[0])
        rate = f"{pp / lv['kernel_ms'] / 1e6:.1f} Gpp/s" if lv["kernel_ms"] > 0 else "persistent kernel"
        print(f"  level {lv['level']}: 1/{lv['scale']} step {lv['step_deg']:g} deg, {lv['poses']} poses, kernel {lv['kernel_ms']:.1f} ms ({rate}), wall {lv['wall_ms']:.1f} ms, best NID {lv['best_nid'][0]:.5f}")
    T = rep["T_camera_lidar"]
    err_r = float(ig.rotation_angle_deg(T[:3, :3], bag["T_gt"][:3, :3]))
    err_t = float(np.linalg.norm(vio.invert_isometry(T)[:3, 3] - vio.invert_isometry(bag["T_gt"])[:3, 3]))
    print(f"  total {total:.2f} s (contexts built on first use included); error {err_r:.3f} deg, {err_t * 100:.1f} cm; margin {rep['margin']}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip_crossover", action="store_true")
    ap.add_argument("--skip_basins", action="store_true")
    ap.add_argument("--skip_search", action="store_true")
    args = ap.parse_args()
    if V.device_count() < 1:
        raise SystemExit("no CUDA device: this probe measures on the GPU only")
    print(f"card: {card()}")
    if not args.skip_crossover:
        crossover()
    if not (args.skip_basins and args.skip_search):
        for name, (key, pattern) in BAGS.items():
            bag = S.make_bag(key, pattern, 200_000, config_index=9)
            if not args.skip_basins:
                basins(name, bag)
            if not args.skip_search:
                full_search(name, bag)


if __name__ == "__main__":
    main()
