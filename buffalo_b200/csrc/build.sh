#!/bin/bash
# Builds libbuffalo_b200.so (sm_90a only) next to the Python package.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../libbuffalo_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
SRCS="$HERE/bfl_common.cu $HERE/als.cu"
[ -f "$HERE/sgd.cu" ] && SRCS="$SRCS $HERE/sgd.cu"
[ -f "$HERE/topk.cu" ] && SRCS="$SRCS $HERE/topk.cu"
[ -f "$HERE/serve.cu" ] && SRCS="$SRCS $HERE/serve.cu"
[ -f "$HERE/ivf.cu" ] && SRCS="$SRCS $HERE/ivf.cu"
[ -f "$HERE/candidates.cu" ] && SRCS="$SRCS $HERE/candidates.cu"
[ -f "$HERE/rerank.cu" ] && SRCS="$SRCS $HERE/rerank.cu"
[ -f "$HERE/category.cu" ] && SRCS="$SRCS $HERE/category.cu"
[ -f "$HERE/evaluate.cu" ] && SRCS="$SRCS $HERE/evaluate.cu"
[ -f "$HERE/offline_eval.cu" ] && SRCS="$SRCS $HERE/offline_eval.cu"
[ -f "$HERE/ingest.cu" ] && SRCS="$SRCS $HERE/ingest.cu"
[ -f "$HERE/plsi.cu" ] && SRCS="$SRCS $HERE/plsi.cu"
[ -f "$HERE/mm_ingest.cu" ] && SRCS="$SRCS $HERE/mm_ingest.cu"
[ -f "$HERE/stream_ingest.cu" ] && SRCS="$SRCS $HERE/stream_ingest.cu"
[ -f "$HERE/explain.cu" ] && SRCS="$SRCS $HERE/explain.cu"
"$NVCC" -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
    -ccbin /usr/bin/g++ -Xcompiler -fPIC,-O3,-Wall -shared \
    ${BFL_PTXAS_V:+-Xptxas -v} -o "$OUT" $SRCS
echo "built $OUT"
