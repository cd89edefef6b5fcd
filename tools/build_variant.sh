#!/bin/bash
# Builds a variant of the library with extra nvcc defines for A/B runs: tools/build_variant.sh <name> [-DNR_...=..]
# -> neuray_b200/libneuray_b200_<name>.so (select with NEURAY_B200_LIB=<path>)
set -e
name=$1; shift
cd "$(dirname "$0")/../neuray_b200/csrc"
mkdir -p /tmp/nrvar_$name
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -O2 $@"
for f in nr_ops nr_pack nr_point_kernel nr_ray_kernel nr_tc_test nr_train nr_tape_gemm nr_encoder nr_losses nr_mvs; do
  nvcc $FLAGS -c $f.cu -o /tmp/nrvar_$name/$f.o &
done
wait
nvcc -shared -o ../libneuray_b200_$name.so /tmp/nrvar_$name/*.o -gencode arch=compute_90a,code=sm_90a
echo ../libneuray_b200_$name.so
