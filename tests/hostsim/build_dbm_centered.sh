#!/bin/bash
# TEST INFRASTRUCTURE: the stand-in-runtime library of build.sh plus the CPU restatement of what centering adds to the tensor-core
# DBM engine (kernels_dbm_centered_cpu.cpp) -> tests/hostsim/_build/libbm_hostsim_dbm_centered.so.  Centering runs with parallel
# tempering and multinomial layers, so their restatements are linked too: kernels_dbm_pt_cpu.cpp with its dispatcher renamed to
# execute_pt and its fall-back to execute_multinomial, kernels_dbm_multinomial_cpu.cpp renamed to execute_multinomial, and
# kernels_cpu.cpp renamed to execute_base; each dispatcher falls back to the next.
# Safe to call from several processes at once; nothing is rebuilt while it is newer than its inputs.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OBJ="$ROOT/boltzmann-machines_b200/build"
OUT="$HERE/_build"
LIB="$OUT/libbm_hostsim_dbm_centered.so"
bash "$HERE/build.sh" > /dev/null                     # fake_cudart.o and the library's objects
exec 8> "$OUT/.lock_dbm_centered"
flock 8
fresh=1
[ -f "$LIB" ] || fresh=0
if [ $fresh = 1 ]; then
    for src in "$OBJ"/*.o "$OUT/fake_cudart.o" "$HERE/kernels_cpu.cpp" "$HERE/kernels_dbm_multinomial_cpu.cpp" "$HERE/kernels_dbm_pt_cpu.cpp" \
               "$HERE/kernels_dbm_centered_cpu.cpp" "$HERE/build_dbm_centered.sh" "$ROOT"/boltzmann-machines_b200/csrc/*.h; do
        [ "$src" -nt "$LIB" ] && fresh=0
    done
fi
if [ $fresh = 0 ]; then
    CXX="g++ -O2 -g -std=c++17 -fPIC -ffp-contract=off -I/usr/local/cuda/include"
    $CXX -Dexecute=execute_base -c "$HERE/kernels_cpu.cpp" -o "$OUT/kernels_cpu_base_cen.o"
    $CXX -Dexecute=execute_multinomial -c "$HERE/kernels_dbm_multinomial_cpu.cpp" -o "$OUT/kernels_dbm_multinomial_cen.o"
    $CXX -Dexecute=execute_pt -Dexecute_base=execute_multinomial -c "$HERE/kernels_dbm_pt_cpu.cpp" -o "$OUT/kernels_dbm_pt_cen.o"
    $CXX -c "$HERE/kernels_dbm_centered_cpu.cpp" -o "$OUT/kernels_dbm_centered_cpu.o"
    g++ -shared -Wl,-Bsymbolic -o "$LIB.tmp" "$OBJ"/*.o "$OUT/fake_cudart.o" "$OUT/kernels_cpu_base_cen.o" "$OUT/kernels_dbm_multinomial_cen.o" \
        "$OUT/kernels_dbm_pt_cen.o" "$OUT/kernels_dbm_centered_cpu.o" -ldl -lpthread -lrt -lstdc++
    mv -f "$LIB.tmp" "$LIB"
fi
echo "built $LIB"
