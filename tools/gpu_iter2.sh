#!/bin/bash
# quick development iteration: core parity, NTT-only timings (C2 extended base), a short bench
mkdir -p gpurun_out
timeout 900 python -m pytest tests/test_gpu_parity.py -x -q > gpurun_out/iter_pytest.log 2>&1
echo "pytest rc=$? $(tail -1 gpurun_out/iter_pytest.log)"
: > gpurun_out/ntt_exp.txt
for p in 256 1024; do python tools/bench_ntt.py $p >> gpurun_out/ntt_exp.txt 2>&1; done
cat gpurun_out/ntt_exp.txt
timeout 300 python bench.py --steps 5 --warmup 3 --no-cpu-baseline --no-e2e > gpurun_out/iter_bench.json 2> gpurun_out/iter_bench.err
echo "bench rc=$?"; cat gpurun_out/iter_bench.json | python -c "import sys,json; d=json.loads(sys.stdin.read()); print('value',d['value'],'ms',d['ms_per_step'],'ntt/s',d['roofline']['ntt_per_s'],'frac',d['roofline']['frac'], d['extra'].get('error'))"
