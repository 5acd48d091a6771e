#!/bin/bash
# ncu evidence for the latency form of the kernel: one full capture of small_rs_hh_kernel at one block per SM (132 on an H100);
# results go to $OUT (default bench_out/)
cd "$(dirname "$0")/.."
O=${OUT:-bench_out}
mkdir -p "$O"
timeout 600 ncu --set full --clock-control none --import-source on -k regex:small_rs_hh -s 3 -c 1 -o "$O/prof_small" python tools/small_launch.py 132 > "$O/prof_small_run.log" 2>&1; echo "rc=$?"
tail -3 "$O/prof_small_run.log"; ls -la "$O/prof_small.ncu-rep"
