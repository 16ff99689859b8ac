#!/bin/bash
# compute-sanitizer over tools/sanitize_small.py (all five estimators through both regimes of the iteration kernel, k-NN /
# radius search, VoxelDownSample, fused EstimateNormals, OccupancyGrid, FPFH, DBSCAN, filters).  Logs go to OUTDIR.
#   tools/gpu_sanitize.sh [OUTDIR]
OUT=${1:-sanitizer_logs}
mkdir -p "$OUT"
for tool in memcheck racecheck; do
  timeout 600 compute-sanitizer --tool $tool --print-limit 20 python tools/sanitize_small.py > "$OUT/sanitizer_$tool.log" 2>&1
  echo "== $tool"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|hazard|Invalid|fitness|occupancy|fpfh" "$OUT/sanitizer_$tool.log" | cut -c1-200 | head -30
done
