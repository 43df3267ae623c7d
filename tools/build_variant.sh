#!/bin/bash
# tools/build_variant.sh NAME [-DFLAG=VALUE ...]  ->  build_variants/lib_NAME.so  (A/B experiments; load with
# CUTADAPT_B200_LIB=build_variants/lib_NAME.so).  The sources are the library's, __graft_entry__.SOURCES.
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p build_variants
srcs=$(python3 -c "import __graft_entry__ as g; g.write_jit_embed(); print(' '.join('cutadapt_b200/csrc/' + s for s in g.SOURCES))")
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared "$@" \
  -Xcompiler -pthread -o build_variants/lib_$name.so $srcs -lpthread -ldl
