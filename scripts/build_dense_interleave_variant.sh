#!/bin/bash
# A/B build of libhelix_b200.so with another value of HXD_INTERLEAVE [and HXD_T] (csrc/k_dense.cu) -> helix-db_b200/_variants/
# usage: build_dense_interleave_variant.sh <interleave 0|1> [top-T]
set -euo pipefail
ROOT="$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)"
HERE="$ROOT/helix-db_b200"
VAL="${1:-1}"
TOPT="${2:-8}"
TAG="il${VAL}"; [[ "$TOPT" != 8 ]] && TAG="il${VAL}_t${TOPT}"
mkdir -p "$HERE/_variants"
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-O2,-Wall,-Wno-unused-function \
  --fmad=false -DHXD_INTERLEAVE="$VAL" -DHXD_T="$TOPT" -Xptxas -v -c "$HERE/csrc/k_dense.cu" -o "$HERE/_variants/k_dense_$TAG.o"
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o "$HERE/_variants/libhelix_b200_$TAG.so" \
  "$HERE/_obj/hx_api.o" "$HERE/_obj/k_build.o" "$HERE/_obj/hx_shard.o" "$HERE/_variants/k_dense_$TAG.o" -lcudart -ldl
echo "built $HERE/_variants/libhelix_b200_$TAG.so"
