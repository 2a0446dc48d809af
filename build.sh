#!/usr/bin/env bash
# Build the C-ABI library (sm_90a, H100) in-tree: vit.cpp_b200/libvitb200.so
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=vit.cpp_b200/libvitb200.so
$NVCC -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo \
      -Xcompiler -fPIC -Xptxas -v -shared -o "$OUT" vit.cpp_b200/csrc/engine.cu 2> build.log || { cat build.log; exit 1; }
grep -E "error|warning" build.log | grep -v "ptxas info" | head -20 || true
echo "built $OUT"
