#!/bin/bash
# Builds libkvidx.so (sm_90a only) in-tree.  Usage: ./build.sh [extra nvcc flags]
set -e
cd "$(dirname "$0")"
OUT=${KVIDX_OUT:-llm-d-kv-cache-manager_b200/lib}
mkdir -p $OUT
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall -shared \
     -Xptxas -v "$@" -o $OUT/libkvidx.so llm-d-kv-cache-manager_b200/csrc/kvidx.cu llm-d-kv-cache-manager_b200/host/kvhost.cpp 2>&1
# load generator for the concurrent-callers measurement (bench.py "concurrent_clients"): plain C++ against the C ABI
g++ -O2 -std=c++17 -pthread -o $OUT/kvidx_qps llm-d-kv-cache-manager_b200/tools/qps_clients.cpp -L$OUT -lkvidx -Wl,-rpath,'$ORIGIN' 2>&1
