#!/bin/bash
# Builds libmetrabs_b200.so in-tree for sm_90a (the only target).  Usage: build.sh [extra nvcc flags]
set -e
cd "$(dirname "$0")"
OUT=../libmetrabs_b200.so
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
  -Xcompiler -fPIC -shared -o $OUT engine.cu -ldl "$@"
echo "built $(realpath $OUT)"
