M="smsp__inst_executed.sum,gpu__time_duration.sum,smsp__thread_inst_executed.sum,launch__registers_per_thread"
for cfg in "i64 0" "i64 1000" "f64b 0" "f64a 0"; do
  set -- $cfg
  echo "== kind=$1 jitter=$2"
  ncu --metrics $M --clock-control none -k "regex:k_scan_aggregate" -s 2 -c 1 python tools/profile_scan.py --series 1000000 --steps 3 --kind $1 --jitter $2 2>&1 | grep -E "smsp__|gpu__time|scan "
done
echo "== i64 count only"
ncu --metrics $M --clock-control none -k "regex:k_scan_aggregate" -s 2 -c 1 python tools/profile_scan.py --series 1000000 --steps 3 --kind i64 --jitter 0 --aggs count 2>&1 | grep -E "smsp__|gpu__time|scan "
