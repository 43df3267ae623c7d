#!/bin/bash
# tools/build_variant.sh NAME [-DFLAG=VALUE ...]  ->  build_variants/lib_NAME.so  (A/B experiments; load with
# CUTADAPT_B200_LIB=build_variants/lib_NAME.so)
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p build_variants
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared "$@" \
  -Xcompiler -pthread -o build_variants/lib_$name.so cutadapt_b200/csrc/cg_kernels.cu cutadapt_b200/csrc/cg_fastq.cu \
  cutadapt_b200/csrc/cg_api.cu cutadapt_b200/csrc/cg_setbuild.cpp cutadapt_b200/csrc/cg_host_algos.cpp \
  cutadapt_b200/csrc/cg_hostpack.cpp cutadapt_b200/csrc/cg_jit.cpp -lpthread -ldl
