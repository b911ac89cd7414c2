#!/bin/bash
# two PIR server processes, one per GPU, at once (needs two GPUs)
mkdir -p gpurun_out
{
( timeout 120 python tools/diag_pir_threads.py plain 0 8 2>&1 | sed "s/^/[gpu0] /" ) &
( timeout 120 python tools/diag_pir_threads.py plain 1 8 2>&1 | sed "s/^/[gpu1] /" ); wait
nproc; cat /sys/fs/cgroup/cpu.max 2>/dev/null
} > gpurun_out/diag_pir_2proc.log 2>&1
grep -v Warning gpurun_out/diag_pir_2proc.log
