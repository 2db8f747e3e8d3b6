#!/bin/bash
# Development aid for A/B timing on the GPU box: build mozjpeg_b200/variants/libb200jpeg_<name>.so with extra -D flags
# for kernels.cu (encoder.o / params.o are reused).  bench.py / the binding load it when B200JPEG_LIB_VARIANT=<name>.
#   tools/build_variant.sh halfrate -DTRELLIS_RATE_F32=0
set -e
cd "$(dirname "$0")/.."
NAME=$1; shift
mkdir -p build/variants mozjpeg_b200/variants
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Iinclude -Imozjpeg_b200/csrc -fmad=false "$@" \
  -c mozjpeg_b200/csrc/kernels.cu -o build/variants/kernels_$NAME.o
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o mozjpeg_b200/variants/libb200jpeg_$NAME.so build/variants/kernels_$NAME.o \
  build/encoder.cu.o build/params.cpp.o -lcudart_static -ldl -lrt -lpthread
ls -la mozjpeg_b200/variants/libb200jpeg_$NAME.so
