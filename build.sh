#!/bin/bash
# Builds libbm.so (sm_90a) in-tree next to the Python package.  nvcc cross-compiles without a GPU.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
SRC="$HERE/boltzmann-machines_b200/csrc"
OUT="$HERE/boltzmann-machines_b200/boltzmann_machines/libbm.so"
OBJ="$HERE/boltzmann-machines_b200/build"
mkdir -p "$OBJ"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --cudart static"
pids=()
for f in "$SRC"/*.cu; do
  o="$OBJ/$(basename "${f%.cu}").o"
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ "$HERE/build.sh" -nt "$o" ] || [ -n "$(find "$SRC" -name '*.h' -newer "$o" -o -name '*.cuh' -newer "$o")" ]; then
    $NVCC $FLAGS ${BM_PTXAS_V:+-Xptxas -v} -c "$f" -o "$o" &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared --cudart static -gencode arch=compute_90a,code=sm_90a -o "$OUT" "$OBJ"/*.o -ldl -lpthread -lrt
echo "built $OUT"
