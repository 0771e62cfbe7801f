#!/bin/bash
# Host-side code of the product library (C ABI argument checks, AIR description parser, option parsing, opening planner,
# host transcript, JIT source generation) and the oracle under AddressSanitizer + UBSan, driven by the CPU test suite.
# Device code is compiled as usual (it does not run here). Builds into winterfell_b200/_var/asan and oracle/_build/asan.
set -e
cd "$(dirname "$0")/.."
NVCC=/usr/local/cuda/bin/nvcc
mkdir -p winterfell_b200/_var/asan
( cd winterfell_b200
  FLAGS="-gencode arch=compute_90a,code=sm_90a -O1 -g -std=c++17 -Xcompiler -fPIC,-fsanitize=address,-fsanitize=undefined,-fno-omit-frame-pointer --use_fast_math -ccbin /usr/bin/g++ -w -I_build"
  for f in ntt ntt2 commit fri layout capi prover jit auxbuild validate verify; do $NVCC $FLAGS -c csrc/$f.cu -o _var/asan/$f.o & done; wait
  $NVCC -Wno-deprecated-gpu-targets -shared -Xlinker --version-script=exports.map -Xcompiler -fsanitize=address,-fsanitize=undefined \
        -o _var/asan/libwinterfell_b200.so _var/asan/*.o -lcudart -ldl -ccbin /usr/bin/g++ )
export ASAN_OPTIONS=detect_leaks=0:halt_on_error=1:protect_shadow_gap=0 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1
export LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)"
WF_LIB_PATH=$PWD/winterfell_b200/_var/asan/libwinterfell_b200.so python -m pytest tests -x -q -m "not gpu" -p no:cacheprovider \
    -k "not bench_reference and not soundness and not sass"
