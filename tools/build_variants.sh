#!/bin/bash
# Build libdhqr.so with several DHQR_PANEL_VARIANT values into build/ (git-ignored) for tools/gpu_ab.py:
#   bash tools/build_variants.sh 4 12 && python tools/gpu_ab.py build/libdhqr_v4.so build/libdhqr_v12.so 2
# A variant that has never run on a GPU must pass the parity tests first, e.g.
#   cp build/libdhqr_v12.so distributedhouseholderqr.jl_b200/libdhqr.so && python -m pytest tests -m gpu -k "panel or golden or fast"
set -e
cd "$(dirname "$0")/../distributedhouseholderqr.jl_b200/csrc"
mkdir -p ../../build
for v in "$@"; do
  nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -shared -DDHQR_PANEL_VARIANT=$v \
       -o ../../build/libdhqr_v$v.so dhqr_api.cu -I../../include -lcudart -ldl
  echo "built build/libdhqr_v$v.so"
done
