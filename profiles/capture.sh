#!/bin/bash
# Captures the profiling artefacts of one round on an H100 (run from the repo root): bash profiles/capture.sh r03
# Outputs land in gpurun_out/<round>/ (scratch); profiles/collect.py turns them into the summaries under profiles/.
set -u
R=${1:-r02}
O=gpurun_out/$R/cap
mkdir -p $O
B="--steps 3 --warmup 3 --no-cpu --no-extra --e2e-steps 1"
if [ -z "${SKIP_NCU:-}" ]; then   # SKIP_NCU=1: only the plain bench lines (parts 3 and 4)
# 1. launch list: every kernel of a short headline run with its device time (cold-cache, serialised:
#    compare SHARES, not absolutes)
ncu --metrics gpu__time_duration.sum --clock-control none -k regex:"k_" -c 400 --csv \
    --log-file $O/launches.csv python bench.py --steps 3 --warmup 3 --no-cpu --no-extra --e2e-steps 0 > $O/launches.log 2>&1
# 2. full-set captures (one instance each) of the kernels of the headline step ...
ncu --set full --clock-control none --import-source on -k regex:"k_pipe_classify" -s 5 -c 1 -o $O/classify -f \
    python bench.py $B > $O/classify.log 2>&1
ncu --set full --clock-control none --import-source on -k regex:"k_resolve|k_rs_scatter|k_rs_hist|k_rs_scan|k_heads" -s 36 -c 9 -o $O/group_resolve -f \
    python bench.py $B > $O/group_resolve.log 2>&1
# ... and of the other programs' kernels
for spec in "dhcp k_dhcp_fastpath 4" "antispoof_64 k_antispoof 4" "nat_cold_64 k_resolve 4" "nat_steady_64 k_pipe_classify 5" "nat_ingress_64 k_nat_ingress 4"; do
    set -- $spec
    ncu --set full --clock-control none --import-source on -k regex:"$2" -s $3 -c 1 -o $O/$1 -f \
        python bench.py --workload $1 $B > $O/$1.log 2>&1
done
fi
# 3. clocks during a plain (unprofiled) run, next to the number itself
nvidia-smi --query-gpu=index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap \
    --format=csv -lms 200 > $O/clocks.csv &
SMI=$!
python bench.py > $O/bench.json 2> $O/bench.err
kill $SMI
python bench.py --impl reference --steps 5 --warmup 1 > $O/bench_reference.json 2> $O/bench_reference.err
for w in pipeline_64 nat_ingress_64 qos_64 qos_egress_64; do
    python bench.py --workload $w --steps 10 --no-extra --no-cpu > $O/bench_$w.json 2> $O/bench_$w.err
done
bash tools/batch_sweep.sh > $O/batch_sweep.log 2>&1
echo done
