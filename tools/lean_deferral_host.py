#!/usr/bin/env python
"""CPU prediction of the equirectangular deferral rate (tools/, no GPU): the bench.py C3 cloud (uncompressed, not culled)
at the solves' start poses, each with the batch of a Nelder-Mead iteration -- {xo, xr, xe, xc} = xo + {0, 1, 2, 1/2} diff
in the tangent space, |diff| = --diff rad and metres along a random direction -- through the host-compiled lean classifier
(tools/lean_deferral_host.cu): the share of point-poses deferred to the exact path with this tree's constants and with
those of the looser bound (arctangent charge --other turns, one ulp per FMA rounding), for the plain classifier and for
the delta step anchored at xo (pose 0) and at the pose lean_delta_anchor picks.  Prints one JSON line per --diff.
--batches FILE: the four-pose batches a solve recorded (tools/delta_probe.py --replay, batches.npz) instead."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", type=float, default=2.5e-7, help="arctangent charge to compare with, turns")
    ap.add_argument("--stride", type=int, default=5, help="every stride-th point per batch")
    ap.add_argument("--diff", type=float, nargs="+", default=[1e-3], help="|xr - xo| of the iterations, rad and metres")
    ap.add_argument("--directions", type=int, default=2, help="random directions per start pose")
    ap.add_argument("--batches", default=None, help="batches.npz of tools/delta_probe.py --replay")
    args = ap.parse_args()

    import bench
    from direct_visual_lidar_calibration_b200 import synthetic as S

    bag = bench.make_inputs(argparse.Namespace(config="C3", points=None), 0)
    rng = np.random.default_rng(5)

    def iteration_rows(size):
        rows = []
        for T0 in bag["starts"][:8]:
            for _ in range(args.directions):
                w, v = rng.normal(size=3), rng.normal(size=3)
                w *= size / np.linalg.norm(w)
                v *= size / np.linalg.norm(v)
                batch = [S.perturb(T0, tuple(np.degrees(s * w)), tuple(s * v)) for s in (0.0, 1.0, 2.0, 0.5)]
                rows.append(np.stack([T[:3, :4].reshape(12) for T in batch]))
        return np.ascontiguousarray(np.stack(rows), dtype=np.float64)

    pts = np.ascontiguousarray(np.asarray(bag["points"])[:, :3], dtype=np.float32)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    csrc = os.path.join(ROOT, "direct_visual_lidar_calibration_b200", "csrc")
    with tempfile.TemporaryDirectory() as tmp:
        exe, inp = os.path.join(tmp, "lean_deferral_host"), os.path.join(tmp, "in.bin")
        subprocess.run([nvcc, "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-Xcompiler", "-ffp-contract=off", f"-I{csrc}", f"-I{os.path.join(ROOT, 'include')}", "-o", exe,
                        os.path.join(ROOT, "tools", "lean_deferral_host.cu")], check=True)
        if args.batches:
            rec = np.load(args.batches)
            sets = [("recorded", rec["poses"][rec["counts"] == 4][:, :4])]
        else:
            sets = [(size, iteration_rows(size)) for size in args.diff]
        for size, rows in sets:
            rows = np.ascontiguousarray(rows, dtype=np.float64)
            with open(inp, "wb") as fh:
                fh.write(np.array([bag["width"], bag["height"], len(pts), len(rows)], dtype=np.int32).tobytes())
                fh.write(pts.tobytes())
                fh.write(rows.tobytes())
            out = subprocess.run([exe, inp, str(args.stride), repr(args.other)], check=True, capture_output=True, text=True).stdout
            print(json.dumps({"diff": size, **json.loads(out)}))


if __name__ == "__main__":
    main()
