#!/bin/bash
# build ubench2 variants: tools/build_ub.sh "name:flags" ...
cd "$(dirname "$0")/.."
mkdir -p tools/ub
for spec in "$@"; do n=${spec%%:*}; fl=${spec#*:}; nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I minio_b200/csrc $fl -o tools/ub/u_$n tools/ubench2.cu 2>&1 | grep -E "error" & done; wait
ls tools/ub
