#!/bin/bash
# builds tools/probe/probe (sm_90a); the binary is git-ignored
cd "$(dirname "$0")"
/usr/local/cuda/bin/nvcc -ccbin /usr/bin/g++ -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o probe probe.cu
