#!/bin/bash
# builds experimental kernel variants into gpurun-shipped .so files: tools/variants/libmec_<name>.so
cd "$(dirname "$0")/../minio_b200/csrc"
mkdir -p ../../tools/variants
build() { name=$1; shift; d=/tmp/mecv_$name; mkdir -p $d
  nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC "$@" -c ec_engine.cu -o $d/ec_engine.o &&
  nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC "$@" -c ec_api.cu -o $d/ec_api.o &&
  nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -x cu -c rs_matrix.cc -o $d/rs_matrix.o &&
  nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -x cu -c ec_numa.cc -o $d/ec_numa.o &&
  nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../tools/variants/libmec_$name.so $d/ec_engine.o $d/ec_api.o $d/rs_matrix.o $d/ec_numa.o -cudart static -ldl -lpthread && echo built $name; }
for spec in "$@"; do name=${spec%%:*}; flags=${spec#*:}; build $name $flags & done; wait
