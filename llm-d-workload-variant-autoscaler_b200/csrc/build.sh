#!/bin/sh
# Builds csrc/libwva_b200.so for sm_90a (H100; called by __graft_entry__.build()).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
HOSTCXX=/usr/bin/g++
[ -x "$HOSTCXX" ] || HOSTCXX=g++
exec "$NVCC" -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
  -ccbin "$HOSTCXX" -Xcompiler -fPIC,-O2 --fmad=false -Xptxas -v \
  -shared -o libwva_b200.so capi.cu -lcudart "$@"
