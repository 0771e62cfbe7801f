#!/bin/bash
# build_variant.sh <name> <extra nvcc flags...> : experiment build into _var/<name>/lib.so (load it with WF_LIB_PATH).
# Compiles the same sources as build.sh, so that the variant exports every symbol the Python bindings declare.
set -e
cd "$(dirname "$0")"
name=$1; shift
mkdir -p _var/$name _build
NVCC=/usr/local/cuda/bin/nvcc
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --use_fast_math -ccbin /usr/bin/g++ -w -I_build"
# jit.cu includes the NVRTC header strings that build.sh generates: write them when a fresh tree has none
[ -f _build/jit_headers.inc ] || python3 - <<'PY'
import os
def lit(path):
    return "".join('"' + l.rstrip("\n").replace("\\", "\\\\").replace('"', '\\"') + '\\n"\n' for l in open(path))
out = "".join("static const char %s[] =\n%s;\n" % (name, lit(os.path.join("csrc", f)))
              for name, f in (("JIT_SRC_GL64", "gl64.cuh"), ("JIT_SRC_COMMIT", "commit.cuh"), ("JIT_SRC_GENERIC", "constraints_generic.cuh")))
open("_build/jit_headers.inc", "w").write(out)
PY
pids=()
for f in ntt ntt2 commit fri layout capi prover jit auxbuild validate verify; do
  $NVCC $FLAGS "$@" -c csrc/$f.cu -o _var/$name/$f.o &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared -Xlinker --version-script=exports.map -o _var/$name/lib.so _var/$name/*.o -lcudart -ldl -ccbin /usr/bin/g++
echo built _var/$name/lib.so
