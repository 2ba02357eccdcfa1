#!/bin/bash
# build a tuning variant of the library: tools/build_variant.sh NAME -DF2_TC=.. -DF2_S=..   -> build/variants/libdfm_NAME.so
cd "$(dirname "$0")/.."
mkdir -p build/variants
name=$1; shift
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr "$@" \
  -shared dynamic_factor_models_b200/csrc/dfm_api.cu -o build/variants/libdfm_$name.so -lcudart -ldl
