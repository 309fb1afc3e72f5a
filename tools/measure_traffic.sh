#!/bin/bash
# DRAM traffic of the training kernel at the bench's own step size (profiles/traffic.json): for each workload, bench.py's
# resident run under `ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum` (one pass, no replay), the first
# TIMED step's launch; tools/make_traffic_json.py pairs it with the positions that launch trained.
#   bash tools/measure_traffic.sh c2 c3 c4      -> gpurun_out/traffic_<w>.csv, gpurun_out/steps_<w>.json
set -u
mkdir -p gpurun_out
for w in "$@"; do
  W2B_BENCH_RESIDENT_ONLY=1 W2B_BENCH_STEP_LOG=gpurun_out/steps_$w.json timeout 900 \
    ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none \
        -k regex:train_warp -s 3 -c 1 --csv --log-file gpurun_out/traffic_$w.csv \
        python bench.py --workload $w --steps 1 --warmup 3 --no-cpu-baseline > gpurun_out/traffic_$w.log 2>&1
  echo "traffic $w: exit $?"
done
