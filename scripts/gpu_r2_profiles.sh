#!/bin/bash
# one GPU call: the round's ncu captures (launch list, full sets of the OFDM kernel with the oscillator off / fast / exact, and of the
# MSC Viterbi launch)
set -u
mkdir -p gpurun_out

bash scripts/gpu_ncu.sh 8192
BENCH="python bench.py --batch 8192 --steps 3 --warmup 8 --no-cpu-baseline --no-e2e --no-other-configs"
ncu --set full --clock-control none --import-source on -k regex:ofdm_demod_kernel -s 39 -c 1 -o gpurun_out/prof_ofdm_fastnco -f $BENCH --cfo-hz 50 > gpurun_out/ncu_bench4.log 2>&1
ncu --set full --clock-control none --import-source on -k regex:ofdm_demod_kernel -s 24 -c 1 -o gpurun_out/prof_ofdm_exactnco -f $BENCH --cfo-hz 50 > gpurun_out/ncu_bench5.log 2>&1
ncu --set full --clock-control none --import-source on -k regex:viterbi_kernel -s 18 -c 1 -o gpurun_out/prof_viterbi_fic -f $BENCH --cfo-hz 0 > gpurun_out/ncu_bench6.log 2>&1
tail -n 2 gpurun_out/ncu_bench6.log
ls -la gpurun_out/*.ncu-rep
