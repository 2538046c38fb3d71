#!/bin/bash
# Builds libb200nuts.so for the H100 (sm_90a) in-tree.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -shared \
  ${B200_PTXAS_V:+-Xptxas -v} ${B200_PHASE_CLOCKS:+-DB200_PHASE_CLOCKS} \
  -o ${B200_OUT:-pymc_b200/libb200nuts.so} pymc_b200/csrc/b200nuts.cu
echo "built pymc_b200/libb200nuts.so"
