#!/bin/bash
# round-2 profiling pass: launch list of the headline bench, full captures of every kernel on the C2 and C3 paths and of
# the inner-product kernels.  Reports and their summaries land in the output directory the script creates.
mkdir -p gpurun_out
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/r02_launches.csv \
    python bench.py --steps 2 --warmup 3 --no-e2e --no-cpu-baseline > gpurun_out/ncu_launches.log 2>&1
echo "launch list rc=$?"
# one multiply chunk = lift, lift, ntt fwd, tensor, ntt inv, floor (6 launches); skip the 3 warm-up steps (2 chunks each)
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"ntt_rows_kernel|lift_kernel|tensor_kernel|floor_kernel" -s 36 -c 6 -f -o gpurun_out/r02_c2_kernels \
    python bench.py --steps 1 --warmup 3 --no-e2e --no-cpu-baseline > gpurun_out/ncu_c2.log 2>&1
echo "C2 kernels rc=$?"
timeout 600 ncu --set full --clock-control none -k regex:"ntt_rows_kernel|ks_mac|ks_finish|mod_switch" -s 10 -c 5 -f -o gpurun_out/r02_c3_kernels \
    python tools/prof_kernels.py c3 > gpurun_out/ncu_c3.log 2>&1
echo "C3 kernels rc=$?"
timeout 600 ncu --set full --clock-control none -k regex:"inner_product_plain|tensor_sum" -s 2 -c 2 -f -o gpurun_out/r02_ip_kernels \
    python tools/prof_kernels.py ip > gpurun_out/ncu_ip.log 2>&1
echo "inner-product kernels rc=$?"
ls -la gpurun_out/*.ncu-rep gpurun_out/r02_launches.csv
# summaries on the box (the reports together exceed what travels back); keep only the C2 report
for r in r02_c2_kernels r02_c3_kernels r02_ip_kernels; do python tools/summarize_ncu.py gpurun_out/$r.ncu-rep gpurun_out/$r.txt; done
python tools/summarize_ncu.py --launches gpurun_out/r02_launches.csv gpurun_out/r02_launches.txt
ncu -i gpurun_out/r02_c2_kernels.ncu-rep --page source --csv --kernel-name regex:ntt_rows_kernel --launch-skip 0 --launch-count 1 > gpurun_out/r02_ntt_fwd_source.csv 2>/dev/null
rm -f gpurun_out/r02_c3_kernels.ncu-rep gpurun_out/r02_ip_kernels.ncu-rep
ls -la gpurun_out/
