#!/bin/bash
# Builds the product library in-tree: winterfell_b200/libwinterfell_b200.so (sm_90a only).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-Wno-deprecated-gpu-targets -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall -Xcompiler -Wno-unknown-pragmas --use_fast_math -ccbin /usr/bin/g++ -I_build"
mkdir -p _build
# the three headers NVRTC needs to compile a constraint kernel at run time (csrc/jit.cu), as string literals
python3 - <<'PY'
import os
def lit(path):
    return "".join('"' + l.rstrip("\n").replace("\\", "\\\\").replace('"', '\\"') + '\\n"\n' for l in open(path))
out = "".join("static const char %s[] =\n%s;\n" % (name, lit(os.path.join("csrc", f)))
              for name, f in (("JIT_SRC_GL64", "gl64.cuh"), ("JIT_SRC_COMMIT", "commit.cuh"), ("JIT_SRC_GENERIC", "constraints_generic.cuh")))
old = open("_build/jit_headers.inc").read() if os.path.exists("_build/jit_headers.inc") else None
if out != old:
    open("_build/jit_headers.inc", "w").write(out)
PY
pids=()
for f in ntt ntt2 commit fri layout capi prover jit auxbuild validate verify ${EXTRA_SRCS}; do
  if [ ! -f _build/$f.o ] || [ csrc/$f.cu -nt _build/$f.o ] || [ -n "$(find csrc include ../include -newer _build/$f.o \( -name '*.cuh' -o -name '*.hpp' -o -name '*.h' -o -name '*.inc' \) 2>/dev/null | head -1)" ]; then
    $NVCC $FLAGS ${PTXAS_V:+-Xptxas -v} -c csrc/$f.cu -o _build/$f.o &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
# linked beside its final place and renamed: a reader (or a snapshot of the tree) never sees a half-written library
$NVCC -Wno-deprecated-gpu-targets -shared -Xlinker --version-script=exports.map -o _build/libwinterfell_b200.so.new _build/*.o -lcudart -ldl -ccbin /usr/bin/g++
mv -f _build/libwinterfell_b200.so.new libwinterfell_b200.so
echo "built $(pwd)/libwinterfell_b200.so"
# the C++ mirror of the reference's plugin interface (include/winterfell_b200.hpp) + its driver: plain
# g++ over the C ABI, proving the header has no CUDA dependency
/usr/bin/g++ -O2 -std=c++17 -Wall -Wextra -I../include ../tests/shim/generate_proof_main.cpp -o _build/generate_proof_main \
  -L. -lwinterfell_b200 -Wl,-rpath,'$ORIGIN/..' -Wl,-rpath-link,/usr/local/cuda/lib64
echo "built $(pwd)/_build/generate_proof_main"
