#!/bin/bash
# Compile-time variant of the engine for same-box A/B runs: scripts/build_variant.sh NAME -DFLAG [-DFLAG2 ...]
#   -> howtotrainyourmamlpytorch_b200/lib/libmaml_b200_NAME.so   (select with MAML_B200_LIB=<path>)
set -e
cd "$(dirname "$0")/../howtotrainyourmamlpytorch_b200"
NAME=$1; shift
mkdir -p lib/var_$NAME
for f in kernels_conv kernels_bn kernels_head kernels_param kernels_tc engine; do
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC "$@" -c csrc/$f.cu -o lib/var_$NAME/$f.o &
done
wait
nvcc -shared -o lib/libmaml_b200_$NAME.so lib/var_$NAME/*.o -lcudart
echo lib/libmaml_b200_$NAME.so
