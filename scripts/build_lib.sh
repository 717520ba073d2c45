#!/usr/bin/env bash
# Builds libsemtools_b200.so for sm_90a (cross-compiles without a GPU).
# STB_NVCC_EXTRA adds compiler flags (e.g. -DSTB_SHADOW_F16=0), STB_LIB_OUT redirects the output
# (load such a library with STB_LIB_PATH).
# The C++ host's tokenizer (HfTokenizer, with the files that define the JSON reader and the lowercase tables it
# uses) is compiled in with hidden visibility: stb_tokenizer_load parses tokenizer.json with it, and the
# host programs that link the library keep their own copy of those classes.
set -euo pipefail
cd "$(dirname "$0")/.."
mkdir -p semtools_b200/lib
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OBJ=$(mktemp -d)
trap 'rm -rf "$OBJ"' EXIT
for f in semtools_tokenizer semtools_store semtools_host; do
  /usr/bin/g++ -std=c++17 -O2 -fPIC -fvisibility=hidden -c semtools_b200/host/$f.cpp -o "$OBJ/$f.o"
done
$NVCC -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 \
  -ccbin /usr/bin/g++ -Xcompiler -fPIC -shared ${STB_NVCC_EXTRA:-} \
  -o ${STB_LIB_OUT:-semtools_b200/lib/libsemtools_b200.so} \
  semtools_b200/csrc/api.cu semtools_b200/csrc/scan_topk.cu \
  semtools_b200/csrc/hits_merge.cu semtools_b200/csrc/embed_pool.cu \
  semtools_b200/csrc/batch_scan.cu semtools_b200/csrc/ivfpq.cu \
  semtools_b200/csrc/corpus_update.cu semtools_b200/csrc/batch_threshold.cu \
  semtools_b200/csrc/tokenize.cu "$OBJ"/*.o "$@"
