#!/bin/bash
# TEST INFRASTRUCTURE: links libbm's own objects (built by ../../build.sh for sm_90a) against tests/hostsim/fake_cudart.cpp
# instead of libcudart -> tests/hostsim/_build/libbm_hostsim.so: the host side of the library runs without a GPU
# (kernel launches are recorded and skipped; see fake_cudart.cpp for what is checked).
# Safe to call from several processes at once (pytest-xdist workers): one builds under a lock, outputs appear by rename, and nothing
# is rebuilt while it is newer than its inputs.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OBJ="$ROOT/boltzmann-machines_b200/build"
OUT="$HERE/_build"
ls "$OBJ"/*.o > /dev/null
mkdir -p "$OUT"
exec 9> "$OUT/.lock"
flock 9
fresh=1
for f in "$OUT/libbm_hostsim.so" "$OUT/libfakenccl.so"; do [ -f "$f" ] || fresh=0; done
if [ $fresh = 1 ]; then
    for src in "$OBJ"/*.o "$HERE/fake_cudart.cpp" "$HERE/kernels_cpu.cpp" "$HERE/fake_nccl.cpp" "$HERE/build.sh" "$ROOT"/boltzmann-machines_b200/csrc/*.h; do
        [ "$src" -nt "$OUT/libbm_hostsim.so" ] && fresh=0
    done
fi
if [ $fresh = 0 ]; then
    g++ -O1 -g -std=c++17 -fPIC -I/usr/local/cuda/include -c "$HERE/fake_cudart.cpp" -o "$OUT/fake_cudart.o"
    g++ -O2 -g -std=c++17 -fPIC -I/usr/local/cuda/include -c "$HERE/kernels_cpu.cpp" -o "$OUT/kernels_cpu.o"
    g++ -O2 -g -std=c++17 -fPIC -shared -o "$OUT/libfakenccl.so.tmp" "$HERE/fake_nccl.cpp" -lrt -lpthread
    mv -f "$OUT/libfakenccl.so.tmp" "$OUT/libfakenccl.so"
    g++ -shared -Wl,-Bsymbolic -o "$OUT/libbm_hostsim.so.tmp" "$OBJ"/*.o "$OUT/fake_cudart.o" "$OUT/kernels_cpu.o" -ldl -lpthread -lrt -lstdc++
    mv -f "$OUT/libbm_hostsim.so.tmp" "$OUT/libbm_hostsim.so"
fi
echo "built $OUT/libbm_hostsim.so"
