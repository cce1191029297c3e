#!/bin/bash
# Nsight Compute captures of the preintegration and factor kernels (run from the repo root; OUT= sets the output directory)
set -x
OUT=${OUT:-ncu_out}
mkdir -p "$OUT"
B="python bench.py --no-e2e --no-cpu-baseline --no-clocks --no-configs"
NCU="ncu --set full --clock-control none --import-source on -k regex:k_preintegrate_tri -s 3 -c 1"
$NCU -o $OUT/prof_k1_tri_10k $B --steps 3 --warmup 3 > $OUT/ncu_k1.log 2>&1
$NCU -o $OUT/prof_k1_tri_125k $B --workload v1_125k_200 --distinct 12500 --steps 3 --warmup 3 > $OUT/ncu_k1_125k.log 2>&1
$NCU -o $OUT/prof_k2_tri_100k $B --workload v2_100k_400 --distinct 5000 --steps 3 --warmup 3 > $OUT/ncu_k2.log 2>&1
$NCU -o $OUT/prof_k1_tri_fp32_125k $B --workload v1_1m_200_fp32 --distinct 12500 --steps 3 --warmup 3 > $OUT/ncu_fp32.log 2>&1
CPI_B200_LIB=$PWD/cpi_b200/libcpi_b200_phase_load.so $NCU -o $OUT/prof_phase_load $B --steps 3 --warmup 3 > $OUT/ncu_load.log 2>&1
CPI_B200_LIB=$PWD/cpi_b200/libcpi_b200_phase_cov.so $NCU -o $OUT/prof_phase_cov $B --steps 3 --warmup 3 > $OUT/ncu_cov.log 2>&1
ncu --set full --clock-control none -k regex:k_factor_eval -s 3 -c 1 -o $OUT/prof_k3_factor_1m python bench.py --workload factor_1m --steps 3 --warmup 3 --no-cpu-baseline > $OUT/ncu_k3.log 2>&1
ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file $OUT/launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline > $OUT/launches.log 2>&1
ls -la $OUT/*.ncu-rep
