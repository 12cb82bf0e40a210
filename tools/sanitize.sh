#!/bin/bash
# compute-sanitizer memcheck + racecheck over tools/sanitize_workload.py (mode B: tools/sanitize_modeb.py).
# usage: tools/sanitize.sh [output directory, default: a new temporary directory]
OUT=${1:-$(mktemp -d)}; mkdir -p "$OUT"; echo "logs in $OUT"
for tool in memcheck racecheck; do
  echo "== compute-sanitizer --tool $tool"
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 9 python tools/sanitize_workload.py > $OUT/sanitize_$tool.log 2>&1; echo "rc=$?"
  grep -E "ERROR SUMMARY|SANITIZE_WORKLOAD_OK|RACECHECK SUMMARY|hazard" $OUT/sanitize_$tool.log | head -5
done
