#!/bin/bash
# Round-2 ncu evidence (run under gpurun, 1 GPU).  Output: gpurun_out/r2/*.csv / *.ncu-rep ; summaries are extracted with
# profiles/ncu_extract.py on the CPU box and committed as profiles/ncu_r2_*.txt.
set -x
O=gpurun_out/r2
mkdir -p $O
B="python bench.py --steps 1 --warmup 1 --no-e2e --no-cpu --no-mofa"
# every launch of one warm-up + one timed step with its device time (cold-cache, serialised: compare SHARES)
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 2500 --csv --log-file $O/launches_r2_cfg2.csv $B > $O/ncu_launches.log 2>&1
# full captures of the dominant kernels
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"tfidf_reduce_tiled|tfidf_apply|transpose_fill_pairs" -c 3 -o $O/prof_tfidf -f $B > $O/ncu_tfidf.log 2>&1
# the default LSI schedule starts with half-operand passes, so the first SpMM launches are the half instantiations
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"rowwarp_kernel" -c 3 -o $O/prof_spmm_half -f $B > $O/ncu_half.log 2>&1
ls -la $O
