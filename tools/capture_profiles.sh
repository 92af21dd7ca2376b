#!/bin/bash
# Run on a GPU machine: captures the ncu evidence that tools/summarize_profiles.py summarises under profiles/ (git-ignored).
#   1. launch list of the bench command (every kernel with its device time; cold-cache, serialised)
#   2. one --set full capture of the fused kernels of one step
set -e
TAG=${1:-r01}
mkdir -p profile_out
ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file profile_out/${TAG}_launches.csv \
    python bench.py --steps 2 --warmup 3 --no-cpu-baseline > profile_out/${TAG}_bench_under_ncu.log 2>&1 || true
ncu --set full --clock-control none --import-source on -k "regex:k_scan_aggregate" -s 8 -c 4 -o profile_out/${TAG}_scan \
    python tools/profile_scan.py --series 1000000 --steps 4 > profile_out/${TAG}_profile_scan.log 2>&1 || true
ncu -i profile_out/${TAG}_scan.ncu-rep --page raw --csv > profile_out/${TAG}_scan_raw.csv 2>/dev/null || true
python bench.py --steps 10 --warmup 3 > profile_out/${TAG}_bench.json 2> profile_out/${TAG}_bench.err || true
tail -c 600 profile_out/${TAG}_bench.json
