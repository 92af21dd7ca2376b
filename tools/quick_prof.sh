#!/bin/bash
# Run on the GPU box: parity tests, per-bin times of one C4 step (full size and 1/8 shard), and the instruction /
# issue counters of the fused kernels of one step (ncu, few metrics: cheap).
TAG=${1:-q}
mkdir -p profile_out
python -m pytest tests -m gpu -x -q 2>&1 | tail -3
TSKV_DEBUG_BINS=1 python tools/profile_scan.py --series 1000000 --steps 4 2>&1 | tail -5
TSKV_DEBUG_BINS=1 python tools/profile_scan.py --series 125000 --steps 4 2>&1 | tail -5
M="smsp__inst_executed.sum,gpu__time_duration.sum,smsp__issue_active.avg.pct_of_peak_sustained_active,launch__registers_per_thread,launch__grid_size,sm__warps_active.avg.pct_of_peak_sustained_active,dram__bytes_read.sum"
ncu --metrics $M --clock-control none -k "regex:k_scan_aggregate" -s 8 -c 4 --csv --log-file profile_out/${TAG}_inst.csv \
  python tools/profile_scan.py --series 1000000 --steps 3 > /dev/null 2>&1
python - <<PY
import csv
rows=list(csv.reader(open("profile_out/${TAG}_inst.csv")))
hdr=[i for i,r in enumerate(rows) if r and r[0]=="ID"][0]
H=rows[hdr]; 
out={}
for r in rows[hdr+1:]:
    d=dict(zip(H,r)); k=(d["ID"], d["Kernel Name"][:60]); out.setdefault(k,{})[d["Metric Name"]]=d["Metric Value"]
for k,v in out.items(): print(k, v)
PY
