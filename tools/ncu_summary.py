#!/usr/bin/env python
"""Summarise one `ncu --set full` capture of the persistent kernel into profiles/ncu_<config>.json (profiles/ is a local,
git-ignored directory) -- the figures that only a profiler gives, to be read beside bench.py's CUDA-event timings (never a
number measured under ncu as a bench value): DRAM traffic per pass over the cloud, executed warp instructions per point-pose, issue utilisation.

  python tools/ncu_summary.py <capture>.ncu-rep --config C3 --points 4902806 --poses 1055 --passes 261
(points = cloud size of the profiled context, poses / passes = point-pose passes the captured launch carried; the probe
tools print them)."""
import argparse
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("report")
    ap.add_argument("--config", required=True)
    ap.add_argument("--points", type=int, required=True)
    ap.add_argument("--poses", type=int, required=True, help="poses scored by the captured launch (sum over its passes)")
    ap.add_argument("--passes", type=int, required=True)
    ap.add_argument("--out", default=None)
    ap.add_argument("--note", default="")
    args = ap.parse_args()
    raw = subprocess.run(["ncu", "-i", args.report, "--page", "raw", "--csv"], check=True, capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, vals = rows[0], rows[1], rows[2]
    m = {h: (v, u) for h, u, v in zip(hdr, units, vals)}

    def num(name, scale_units=None):
        v, u = m[name]
        x = float(v.replace(",", ""))
        mult = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "ms": 1e-3, "us": 1e-6, "ns": 1e-9, "s": 1.0}.get(u, 1.0)
        return x * mult

    dram = num("dram__bytes_read.sum") + num("dram__bytes_write.sum")
    inst = num("smsp__inst_executed.sum")
    dur = num("gpu__time_duration.sum")
    out = {
        "source": f"{os.path.basename(args.report)} (ncu --set full --clock-control none, one launch of {m['Kernel Name'][0] if 'Kernel Name' in m else 'nid_persistent_kernel'})",
        "config": args.config, "points": args.points, "poses": args.poses, "passes": args.passes,
        "duration_under_ncu_ms": dur * 1e3,
        "dram_bytes_per_launch": dram, "dram_bytes_per_pass": dram / args.passes,
        "algorithmic_bytes_per_pass_cloud_only": 16 * args.points,
        "warp_inst_executed": inst, "warp_inst_per_pointpose": inst * 32.0 / (float(args.points) * args.poses),
        "issue_active_pct": num("smsp__issue_active.avg.pct_of_peak_sustained_active"),
        "registers_per_thread": num("launch__registers_per_thread"), "grid": num("launch__grid_size"),
        "l1_hit_pct": num("l1tex__t_sector_hit_rate.pct"), "l2_hit_pct": num("lts__t_sector_hit_rate.pct"),
        "sm_cycles_active_over_elapsed": num("sm__cycles_active.avg") / num("sm__cycles_elapsed.avg"),
        "stalls_per_issue": {k.split("issue_stalled_")[1].split("_per_issue")[0]: float(v[0]) for k, v in m.items() if k.startswith("smsp__average_warps_issue_stalled_") and k.endswith("_per_issue_active.ratio")},
        "note": args.note or "instruction count includes the spin-waits of the persistent kernel's barriers (thread 0 of every block polls) and the exact fp64 rechecks",
    }
    path = args.out or os.path.join(ROOT, "profiles", f"ncu_{args.config}.json")
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    json.dump(out, open(path, "w"), indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
