#!/bin/bash
# TEST INFRASTRUCTURE: the stand-in-runtime library of build.sh plus the CPU restatements of the exact log Z / log p*(v)
# enumeration's kernels (kernels_dbm_exact_cpu.cpp) -> tests/hostsim/_build/libbm_hostsim_dbm_exact.so.  kernels_cpu.cpp is
# compiled again with its dispatcher renamed to execute_base, to which the restatement's dispatcher falls back.
# Safe to call from several processes at once; nothing is rebuilt while it is newer than its inputs.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OBJ="$ROOT/boltzmann-machines_b200/build"
OUT="$HERE/_build"
LIB="$OUT/libbm_hostsim_dbm_exact.so"
bash "$HERE/build.sh" > /dev/null                     # fake_cudart.o and the library's objects
exec 8> "$OUT/.lock_dbm_exact"
flock 8
fresh=1
[ -f "$LIB" ] || fresh=0
if [ $fresh = 1 ]; then
    for src in "$OBJ"/*.o "$OUT/fake_cudart.o" "$HERE/kernels_cpu.cpp" "$HERE/kernels_dbm_exact_cpu.cpp" "$HERE/build_dbm_exact.sh" \
               "$ROOT"/boltzmann-machines_b200/csrc/*.h "$ROOT"/boltzmann-machines_b200/csrc/*.cuh; do
        [ "$src" -nt "$LIB" ] && fresh=0
    done
fi
if [ $fresh = 0 ]; then
    F="-O2 -g -std=c++17 -fPIC -I/usr/local/cuda/include"
    g++ $F -Dexecute=execute_base -c "$HERE/kernels_cpu.cpp" -o "$OUT/kernels_cpu_base_exact.o"
    g++ $F -c "$HERE/kernels_dbm_exact_cpu.cpp" -o "$OUT/kernels_dbm_exact_cpu.o"
    g++ -shared -Wl,-Bsymbolic -o "$LIB.tmp" "$OBJ"/*.o "$OUT/fake_cudart.o" "$OUT/kernels_cpu_base_exact.o" \
        "$OUT/kernels_dbm_exact_cpu.o" -ldl -lpthread -lrt -lstdc++
    mv -f "$LIB.tmp" "$LIB"
fi
echo "built $LIB"
