#!/bin/bash
# Host-side memory / UB check: build libacb200 with AddressSanitizer + UBSan and run the CPU test-suite against it
# (ACB_LIB selects the library).  No GPU needed; the device code is compiled but never launched.
set -e
cd "$(dirname "$0")/.."
OUT=${1:-/tmp/libacb200_asan.so}
( cd pyahocorasick_b200/csrc && nvcc -O1 -g -std=c++17 -gencode arch=compute_90a,code=sm_90a \
    -Xcompiler -fPIC,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer -shared \
    -o "$OUT" acb_host.cpp acb_device.cu -Xlinker -lasan -Xlinker -lubsan )
ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1 \
LD_PRELOAD=$(gcc -print-file-name=libasan.so) ACB_LIB="$OUT" \
python -m pytest tests -q -m "not gpu" -p no:cacheprovider \
    --deselect tests/test_cabi.py::test_header_is_plain_c_and_links_from_c --deselect tests/test_bench_contract.py
