#!/bin/bash
# Profiling-only builds of the tri-lane kernels (never shipped, never loaded by the product):
#   cpi_b200/libcpi_b200_phase_load.so       sample-load phase alone (TMA staging, no arithmetic)
#   cpi_b200/libcpi_b200_phase_cov.so        covariance RK4 alone (constant inputs, no fetch, no front)
#   cpi_b200/libcpi_b200_phase_noprepass.so  constant scalar sets instead of the pre-pass (wrong output: bounds what hiding it can win)
# Loaded with CPI_B200_LIB=... (bench.py reports kernel_ms) to time each phase against the normal build.
set -e
cd "$(dirname "$0")/../cpi_b200/csrc"
make -s
others=$(ls *.o | grep -v '^preintegrate_tri\.o$')
tmp=$(mktemp -d)
for v in LOAD COV NOPREPASS; do
  lv=$(echo $v | tr A-Z a-z)
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -DCPI_TRI_PHASE_$v -c -o $tmp/tri_phase_$lv.o preintegrate_tri.cu
  nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../libcpi_b200_phase_$lv.so $others $tmp/tri_phase_$lv.o -lcudart -ldl
done
rm -rf $tmp
ls -la ../libcpi_b200_phase_*.so
