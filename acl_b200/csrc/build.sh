#!/bin/sh
# Builds acl_b200/libaclb200.so for sm_90a (H100; no other architecture, no PTX fallback path for other GPUs).
# Used by __graft_entry__.build(); nvcc cross-compiles without a GPU.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="${ACLB200_OUT:-$HERE/../libaclb200.so}"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"$NVCC" -std=c++17 -O3 -lineinfo \
  -gencode arch=compute_90a,code=sm_90a \
  --fmad=false -Xptxas -v \
  -Xcompiler -fPIC,-fvisibility=hidden,-Wall -shared -cudart static \
  -o "$OUT" \
  "$HERE/kernels.cu" "$HERE/pipeline.cu" "$HERE/bones.cu" "$HERE/root_motion.cu" "$HERE/features.cu" "$HERE/feature_search.cu" "$HERE/inertialization.cu" "$HERE/mirror.cu" "$HERE/error_metric.cu" "$HERE/clipset.cpp" "$HERE/database.cpp" "$HERE/api.cpp" "$@"
echo "built $OUT"
