#!/bin/bash
# Builds helix-db_b200/libhelix_b200.so for sm_90a (H100), in-tree.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
OUT="$HERE/libhelix_b200.so"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-O2,-Wall,-Wno-unused-function
       --fmad=false -Xptxas -v)
SRCS=("$HERE/csrc/hx_api.cu" "$HERE/csrc/k_build.cu" "$HERE/csrc/k_dense.cu" "$HERE/csrc/hx_shard.cu")
mkdir -p "$HERE/_obj"
OBJS=()
PIDS=()
for s in "${SRCS[@]}"; do
  o="$HERE/_obj/$(basename "${s%.cu}").o"
  if [[ ! -f "$o" || "$s" -nt "$o" || -n "$(find "$HERE/csrc" "$HERE/../include" -newer "$o" \( -name '*.cuh' -o -name '*.hpp' -o -name '*.h' -o -name '*.inl' \) -print -quit)" ]]; then
    ( "$NVCC" "${FLAGS[@]}" -c "$s" -o "$o.tmp" 2> "$o.log" && mv "$o.tmp" "$o" || { cat "$o.log"; rm -f "$o.tmp"; exit 1; } ) &
    PIDS+=($!)
  fi
  OBJS+=("$o")
done
for p in "${PIDS[@]}"; do wait "$p" || exit 1; done
"$NVCC" -gencode arch=compute_90a,code=sm_90a -shared -o "$OUT" "${OBJS[@]}" -lcudart -ldl
echo "built $OUT"
# C++ host harness over the C ABI (host/vector_index.hpp): N concurrent one-query callers, linked against the library
g++ -O2 -std=c++17 -shared -fPIC -pthread -Wall "$HERE/host/hx_callers.cpp" -I"$HERE/host" -L"$HERE" -lhelix_b200 \
    -Wl,-rpath,'$ORIGIN' -o "$HERE/libhx_callers.so"
echo "built $HERE/libhx_callers.so"
