#!/usr/bin/env python
"""Executed-instruction breakdown of one persistent-kernel capture from `ncu -i <rep> --page source --csv`:
per code region (contiguous SASS ranges with similar execution counts) and per opcode, with the stall-sample share.

  ncu -i <capture>.ncu-rep --page source --csv > /tmp/source.csv
  python tools/ncu_instruction_mix.py /tmp/source.csv > profiles/<name>_instruction_mix.txt"""
import csv
import sys


def main():
    rows = list(csv.reader(open(sys.argv[1])))
    kernel = rows[0][1] if rows[0] and rows[0][0] == "Kernel Name" else "?"
    hdr, data = rows[1], rows[2:]
    isrc, ie, ismp = hdr.index("Source"), hdr.index("Instructions Executed"), hdr.index("# Samples")
    tot = sum(int(r[ie]) for r in data)
    tots = sum(int(r[ismp]) for r in data)
    print(f"kernel: {kernel}")
    print(f"executed warp instructions: {tot}   stall samples: {tots}")
    print()
    print("regions (contiguous SASS ranges whose per-line execution counts stay within 1.5x of each other; >= 0.4 % of the instructions)")
    print(f"{'lines':>13} {'n':>5} {'instr %':>8} {'samples %':>10} {'exec/line':>12}  first instruction")
    segs, cur = [], None
    for k, r in enumerate(data):
        e, s = int(r[ie]), int(r[ismp])
        if cur and ((e > 0 and cur["lo"] <= e * 1.5 and e <= cur["hi"] * 1.5) or (e == 0 and cur["hi"] == 0)):
            cur["n"] += 1
            cur["sum"] += e
            cur["smp"] += s
            cur["lo"], cur["hi"], cur["end"] = min(cur["lo"], e), max(cur["hi"], e), k
        else:
            cur = {"start": k, "end": k, "n": 1, "sum": e, "smp": s, "lo": e, "hi": e}
            segs.append(cur)
    covered = 0
    for s in segs:
        if s["sum"] > tot * 0.004:
            covered += s["sum"]
            print(f"{s['start']:6d}-{s['end']:6d} {s['n']:5d} {100 * s['sum'] / tot:8.1f} {100 * s['smp'] / max(tots, 1):10.1f} {s['sum'] // s['n']:12d}  {data[s['start']][isrc][:60]}")
    print(f"(listed regions cover {100 * covered / tot:.1f} % of the executed instructions)")
    print()
    print("opcodes (>= 0.5 % of the instructions)")
    ops = {}
    for r in data:
        parts = r[isrc].split()
        if not parts:
            continue
        op = parts[1] if parts[0].startswith("@") and len(parts) > 1 else parts[0]
        op = op.split(".")[0]
        o = ops.setdefault(op, [0, 0])
        o[0] += int(r[ie])
        o[1] += int(r[ismp])
    print(f"{'opcode':>12} {'instr %':>8} {'samples %':>10}")
    for op, (e, s) in sorted(ops.items(), key=lambda x: -x[1][0]):
        if e >= tot * 0.005:
            print(f"{op:>12} {100 * e / tot:8.1f} {100 * s / max(tots, 1):10.1f}")


if __name__ == "__main__":
    main()
