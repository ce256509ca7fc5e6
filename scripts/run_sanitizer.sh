#!/bin/bash
# compute-sanitizer memcheck + racecheck + synccheck over one small forward per GEMM path (GPU box).
# The input (1x3x32x128, x4) reaches every tensor-core GEMM variant: 64- and 128-wide tiles, K-sliced accumulation
# (layers in front of the VQ), F8 cross terms (behind it),
# sub-pixel upsample convs, stride-2 TMA, split-plane outputs, GroupNorm partials; plus attention / VQ / edge kernels.
# Usage: bash scripts/run_sanitizer.sh   -> gpurun_out/sanitizer_*.txt + gpurun_out/sanitizer_summary.txt
set -u
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
SUMMARY=gpurun_out/sanitizer_summary.txt
: > "$SUMMARY"
for tool in memcheck racecheck synccheck; do
  for path in 1 0; do
    if [ "$tool" != memcheck ] && [ "$path" = 0 ]; then continue; fi
    log=gpurun_out/sanitizer_${tool}_path${path}.txt
    FEMASR_GEMM_PATH=$path FEMASR_CUDA_GRAPH=0 timeout 1500 compute-sanitizer --tool $tool --print-limit 20 \
      python scripts/sanitizer_target.py > "$log" 2>&1
    rc=$?
    echo "== $tool gemm_path=$path rc=$rc" >> "$SUMMARY"
    grep -E "ERROR SUMMARY|RACECHECK SUMMARY|target:|Error|hazard" "$log" | head -12 >> "$SUMMARY"
  done
done
cat "$SUMMARY"
