#!/bin/bash
# ncu launch list of the default bench workload's training step (eager, no CUDA graph): per-launch device time and
# DRAM bytes (single replay pass; cold-cache serialised -> compare SHARES).  tools/conv_traffic_from_launchlist.py turns
# it into the conv-traffic record bench.py reports.  usage: bash tools/gpu_launchlist.sh [OUT_DIR]
OUT=${1:-launchlist_out}
mkdir -p "$OUT"
timeout 900 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none \
  --csv --log-file "$OUT/launches_resnet50.csv" python tools/one_step.py resnet50_uq8_dst_b128 2 > "$OUT/launchlist_bench.log" 2>&1
echo "ncu exit $?"; tail -2 "$OUT/launchlist_bench.log" | cut -c1-300
wc -l "$OUT/launches_resnet50.csv"
