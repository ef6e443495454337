#!/bin/bash
# Development build of libb2gram with the ablation / timing knobs compiled in (-DB2_DEV_KNOBS):
#   B2_TC_DEBUG bits (skip MMAs / STS / LDS / proxy fence -- WRONG results, timing only; bit 8 = 256 keeps every
#   drained fp64 sum in L2 instead of registers / shared memory -- same results), B2_WAIT_HINT_NS, B2_SOLVE_TIMING.
#   The knobs cost registers: ptxas serialises the wgmma of this build's RAWB (bf16 rows, D = 128) kernels, so time
#   those with the product build.  Use with  B2_LIB_PATH=tools/bin/libb2gram_dev.so python bench.py ...
set -e
cd "$(dirname "$0")/../bodywork-mlops-demo_b200/csrc"
mkdir -p ../../tools/bin
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -shared -DB2_DEV_KNOBS \
     -o ../../tools/bin/libb2gram_dev.so *.cu -ldl
echo built tools/bin/libb2gram_dev.so
