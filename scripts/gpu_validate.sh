#!/bin/bash
# Full validation + evidence pass on one GPU: tests, bench lines, per-layer table, sanitizer, ncu launch
# list and DRAM/L2 traffic of the dominant kernel.  Outputs under gpurun_out/ (tag = $1, default "final").
set -u
cd "$(dirname "$0")/.."
TAG=${1:-final}
mkdir -p gpurun_out
rm -f gpurun_out/parity_report.json
python -m pytest tests -m gpu -q -s --maxfail=8 2>&1 | tail -150 > gpurun_out/pytest_$TAG.log
python bench.py --steps 10 --warmup 3 > gpurun_out/bench_$TAG.json 2> gpurun_out/bench_$TAG.err
for c in 3 5 2test; do python bench.py --config $c --steps 5 --warmup 3 --no-cpu-baseline > gpurun_out/bench_${TAG}_cfg$c.json 2> gpurun_out/bench_${TAG}_cfg$c.err; done
python scripts/profile_layers.py 32 > gpurun_out/layers_$TAG.txt 2>&1
python scripts/microbench_tc.py > gpurun_out/microbench_$TAG.txt 2>&1
python scripts/vq_stats.py > gpurun_out/vq_stats_$TAG.json 2>/dev/null
bash scripts/run_sanitizer.sh > /dev/null 2>&1
cp gpurun_out/sanitizer_summary.txt gpurun_out/sanitizer_$TAG.txt
# ncu: every launch of one eager step (shares), then DRAM / L2 bytes + tensor-pipe activity of the tc_igemm launches
FEMASR_CUDA_GRAPH=0 ncu --metrics gpu__time_duration.sum --clock-control none -s 840 -c 280 --csv \
  --log-file gpurun_out/launches_$TAG.csv python bench.py --steps 1 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_launches_$TAG.log 2>&1
FEMASR_CUDA_GRAPH=0 ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,lts__t_bytes.sum,gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active \
  --clock-control none -k regex:tc_igemm -s 402 -c 134 --csv --log-file gpurun_out/traffic_$TAG.csv \
  python bench.py --steps 1 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_traffic_$TAG.log 2>&1
grep -E "passed|failed" gpurun_out/pytest_$TAG.log | tail -2
cat gpurun_out/bench_$TAG.json | head -c 600
