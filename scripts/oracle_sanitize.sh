#!/bin/bash
# The CPU oracle (the parity checker) under AddressSanitizer + UBSan: its known-answer suite, the golden fixture and a
# randomised mutation stress.  CPU only.
set -euo pipefail
ROOT="$(cd "$(dirname "${BASH_SOURCE[0]}")/.." && pwd)"
cd "$ROOT"
make -C oracle -s asan
export HXO_ORACLE_SO="$ROOT/oracle/_build/libhx_oracle_asan.so"
export ASAN_OPTIONS=detect_leaks=0:abort_on_error=1
export LD_PRELOAD="$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so)"
python -m pytest tests/test_oracle_kat.py tests/test_golden.py -q -m "not gpu" -p no:cacheprovider 2>&1 | tail -3
python scripts/oracle_mutation_stress.py 2>&1 | tail -8
