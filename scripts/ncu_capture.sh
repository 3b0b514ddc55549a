#!/bin/bash
# ncu --set full capture of one kernel of the resident pass, exported as CSV (raw metrics + per-instruction source page) so that
# only text needs keeping, plus the FP64 instruction counters of the same launch.  The CSVs go to $NCU_OUT (default /tmp).
# usage: scripts/ncu_capture.sh <tag> <kernel-regex> <skip> [stage_bench args...]
tag=$1; kern=$2; skip=$3; shift 3
rep=/tmp/prof_$tag
out=${NCU_OUT:-/tmp}
ncu --set full --clock-control none --import-source on -k "regex:$kern" -s "$skip" -c 1 -f -o $rep python scripts/stage_bench.py --steps 1 "$@" > /dev/null 2>&1
ncu -i $rep.ncu-rep --page raw --csv > $out/ncu_raw_$tag.csv 2>/dev/null
ncu -i $rep.ncu-rep --page source --csv > $out/ncu_src_$tag.csv 2>/dev/null
ncu --clock-control none -k "regex:$kern" -s "$skip" -c 1 --csv --metrics smsp__sass_thread_inst_executed_op_dfma_pred_on.sum,smsp__sass_thread_inst_executed_op_dmul_pred_on.sum,smsp__sass_thread_inst_executed_op_dadd_pred_on.sum,gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum python scripts/stage_bench.py --steps 1 "$@" 2>/dev/null | grep -E '^"|^[0-9]' > $out/ncu_fp64_$tag.csv
ls -la $out/ncu_raw_$tag.csv $out/ncu_src_$tag.csv $out/ncu_fp64_$tag.csv
