#!/usr/bin/env bash
# Builds libsemtools_b200.so for sm_90a (cross-compiles without a GPU).
# STB_NVCC_EXTRA adds compiler flags (e.g. -DSTB_SHADOW_F16=0), STB_LIB_OUT redirects the output
# (load such a library with STB_LIB_PATH).
set -euo pipefail
cd "$(dirname "$0")/.."
mkdir -p semtools_b200/lib
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
  -ccbin /usr/bin/g++ -Xcompiler -fPIC -shared ${STB_NVCC_EXTRA:-} \
  -o ${STB_LIB_OUT:-semtools_b200/lib/libsemtools_b200.so} \
  semtools_b200/csrc/api.cu semtools_b200/csrc/scan_topk.cu \
  semtools_b200/csrc/hits_merge.cu semtools_b200/csrc/embed_pool.cu \
  semtools_b200/csrc/batch_scan.cu semtools_b200/csrc/ivfpq.cu \
  semtools_b200/csrc/corpus_update.cu semtools_b200/csrc/batch_threshold.cu "$@"
