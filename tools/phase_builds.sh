#!/bin/bash
# Profiling-only builds of the tri-lane kernels (never shipped, never loaded by the product):
#   cpi_b200/libcpi_b200_phase_load.so  sample-load phase alone (TMA staging, no arithmetic)
#   cpi_b200/libcpi_b200_phase_cov.so   covariance RK4 alone (constant inputs, no fetch, no front)
# Used with CPI_B200_LIB=... under ncu to report achieved HBM GB/s of the load phase and fp64 FLOP/s of the covariance phase.
set -e
cd "$(dirname "$0")/../cpi_b200/csrc"
make -s
for v in LOAD COV; do
  lv=$(echo $v | tr A-Z a-z)
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -DCPI_TRI_PHASE_$v -c -o /tmp/tri_phase_$lv.o preintegrate_tri.cu
  nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../libcpi_b200_phase_$lv.so capi.o preintegrate.o /tmp/tri_phase_$lv.o factor.o shard.o windows.o solve.o -lcudart -ldl
done
ls -la ../libcpi_b200_phase_*.so
