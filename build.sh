#!/bin/bash
# Builds libtmac_b200.so (sm_90a only) in-tree. Usage: ./build.sh [extra nvcc flags]
# The translation units (host + gemv3/prefill kernels, sequence kernels) are compiled in parallel, then linked.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=${TMAC_B200_OUT:-t-mac_b200/libtmac_b200.so}
OBJ=$(mktemp -d)
trap 'rm -rf "$OBJ"' EXIT
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden,-O2"
PIDS=""
for tu in tmac_b200 tmac_seq tmac_chain_batch tmac_gemv_io tmac_gemv_experts tmac_prefill_experts; do
  $NVCC $FLAGS -c -o "$OBJ/$tu.o" t-mac_b200/csrc/$tu.cu "$@" &
  PIDS="$PIDS $!"
done
for p in $PIDS; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -cudart static -o "$OUT" "$OBJ"/*.o
echo "built $OUT"
