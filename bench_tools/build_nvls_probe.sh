#!/bin/bash
# Builds the standalone NVLS multicast probe (see nvls_probe_main.cu). The binary is git-ignored but travels to the
# GPU box with the gpurun snapshot.
set -e
cd "$(dirname "$0")/.."
mkdir -p bench_tools/bin
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -I dist_mnist_b200/csrc \
  dist_mnist_b200/csrc/nvls_sm90.cu bench_tools/nvls_probe_main.cu -o bench_tools/bin/nvls_probe
ls -l bench_tools/bin/nvls_probe
