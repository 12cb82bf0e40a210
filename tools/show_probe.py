#!/usr/bin/env python
"""Compact view of a tools/pk_probe.py JSON-lines file (or a log that contains such lines)."""
import json
import sys

for line in open(sys.argv[1]):
    line = line.strip()
    if not line.startswith('{"config"'):
        if line and not line.startswith("."):
            print(line[:300])
        continue
    try:
        d = json.loads(line)
    except ValueError:
        print(line[:200])
        continue
    tag = d["tag"] or "default"
    if d["what"] == "solve":
        print(f'{d["config"]} {tag:12s} mode {d["mode"]} {d["ms_per_solve"]:8.3f} ms/solve {d["evals_per_s"]:9.0f} evals/s {d["us_per_batch"]:7.2f} us/batch same_as_first={d["same_as_first_mode"]}')
    elif d["what"] == "stamps_us_median":
        print("    stamps", {k: round(v, 1) for k, v in d["phases"].items()}, "period", round(d["batch_period_us"], 1))
    elif d["what"].startswith("pose_list"):
        print(f'    {d["config"]} {tag} {d["what"]} {d.get("cloud")} poses={d.get("poses")} {d["gpp_per_s"]:.1f} G point-poses/s')
    elif d["what"].startswith("block_times"):
        print("    main_duration p0/p10/p50/p90/p100", [round(x, 1) for x in d["main_duration"]], "arrived", [round(x, 1) for x in d["arrived"]])
    else:
        print("   ", d["what"])
