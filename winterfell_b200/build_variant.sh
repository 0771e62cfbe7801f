#!/bin/bash
# build_variant.sh <name> <extra nvcc flags...> : experiment build into _var/<name>/lib.so
set -e
cd "$(dirname "$0")"
name=$1; shift
mkdir -p _var/$name
NVCC=/usr/local/cuda/bin/nvcc
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --use_fast_math -ccbin /usr/bin/g++ -w -I_build"
for f in ntt ntt2 commit fri layout capi prover jit auxbuild; do $NVCC $FLAGS "$@" -c csrc/$f.cu -o _var/$name/$f.o & done; wait
$NVCC -shared -Xlinker --version-script=exports.map -o _var/$name/lib.so _var/$name/*.o -lcudart -ldl -ccbin /usr/bin/g++
echo built _var/$name/lib.so
