#!/bin/bash
# HOST code of the product library under AddressSanitizer + UBSan (device code untouched): builds
# helix-db_b200/_variants/libhelix_b200_asan.so, then runs the device-free ABI / codec / host-logic tests and a byte-level
# fuzz of the row and key decoders on it.  CPU only.
set -euo pipefail
ROOT="$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)"
HERE="$ROOT/helix-db_b200"
cd "$ROOT"
mkdir -p "$HERE/_variants"
[[ -f "$HERE/_obj/k_build.o" ]] || bash "$HERE/build.sh" > /dev/null
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O1 -g -lineinfo -std=c++17 --fmad=false \
  -Xcompiler -fPIC,-O1,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer -c "$HERE/csrc/hx_api.cu" -o "$HERE/_variants/hx_api_asan.o" 2> /dev/null
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -Xcompiler -fsanitize=address,-fsanitize=undefined \
  -o "$HERE/_variants/libhelix_b200_asan.so" "$HERE/_variants/hx_api_asan.o" "$HERE/_obj/k_build.o" "$HERE/_obj/k_dense.o" "$HERE/_obj/hx_shard.o" -lcudart -ldl
export HELIX_B200_LIB="$HERE/_variants/libhelix_b200_asan.so"
export ASAN_OPTIONS=detect_leaks=0:abort_on_error=1:protect_shadow_gap=0
export LD_PRELOAD="$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so)"
python -m pytest tests/test_row_codecs.py tests/test_host_logic.py tests/test_abi_surface.py -q -m "not gpu" -p no:cacheprovider \
  -k "not library_exports and not no_torch_or_oracle and not cpp_host" 2>&1 | tail -3
python scripts/codec_fuzz.py 2>&1 | tail -3
