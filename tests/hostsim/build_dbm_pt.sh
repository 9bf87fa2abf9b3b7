#!/bin/bash
# TEST INFRASTRUCTURE: the stand-in-runtime library of build.sh plus the CPU restatement of what parallel tempering adds to the
# tensor-core DBM engine (kernels_dbm_pt_cpu.cpp) -> tests/hostsim/_build/libbm_hostsim_dbm_pt.so.
# kernels_cpu.cpp is compiled again with its dispatcher renamed to execute_base, which the new dispatcher falls back to.
# Safe to call from several processes at once; nothing is rebuilt while it is newer than its inputs.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OBJ="$ROOT/boltzmann-machines_b200/build"
OUT="$HERE/_build"
LIB="$OUT/libbm_hostsim_dbm_pt.so"
bash "$HERE/build.sh" > /dev/null                     # fake_cudart.o and the library's objects
exec 8> "$OUT/.lock_dbm_pt"
flock 8
fresh=1
[ -f "$LIB" ] || fresh=0
if [ $fresh = 1 ]; then
    for src in "$OBJ"/*.o "$OUT/fake_cudart.o" "$HERE/kernels_cpu.cpp" "$HERE/kernels_dbm_pt_cpu.cpp" "$HERE/build_dbm_pt.sh" \
               "$ROOT"/boltzmann-machines_b200/csrc/*.h; do
        [ "$src" -nt "$LIB" ] && fresh=0
    done
fi
if [ $fresh = 0 ]; then
    g++ -O2 -g -std=c++17 -fPIC -I/usr/local/cuda/include -Dexecute=execute_base -c "$HERE/kernels_cpu.cpp" -o "$OUT/kernels_cpu_base_pt.o"
    g++ -O2 -g -std=c++17 -fPIC -I/usr/local/cuda/include -c "$HERE/kernels_dbm_pt_cpu.cpp" -o "$OUT/kernels_dbm_pt_cpu.o"
    g++ -shared -Wl,-Bsymbolic -o "$LIB.tmp" "$OBJ"/*.o "$OUT/fake_cudart.o" "$OUT/kernels_cpu_base_pt.o" "$OUT/kernels_dbm_pt_cpu.o" \
        -ldl -lpthread -lrt -lstdc++
    mv -f "$LIB.tmp" "$LIB"
fi
echo "built $LIB"
