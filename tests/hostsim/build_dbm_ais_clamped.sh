#!/bin/bash
# TEST INFRASTRUCTURE: the stand-in-runtime library of build_dbm_ais_base.sh plus the CPU restatement of the clamped AIS
# ladder's operand kernel (kernels_dbm_ais_clamped_cpu.cpp) -> tests/hostsim/_build/libbm_hostsim_dbm_ais_clamped.so.
# kernels_cpu.cpp is compiled with its dispatcher renamed to execute_base, the multinomial restatement to execute_multinomial,
# the depth restatement to execute_ais_depth and the base-rate restatement to execute_ais_base; each dispatcher falls back to
# the next.  Safe to call from several processes at once; nothing is rebuilt while it is newer than its inputs.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OBJ="$ROOT/boltzmann-machines_b200/build"
OUT="$HERE/_build"
LIB="$OUT/libbm_hostsim_dbm_ais_clamped.so"
bash "$HERE/build.sh" > /dev/null                     # fake_cudart.o and the library's objects
exec 8> "$OUT/.lock_dbm_ais_clamped"
flock 8
fresh=1
[ -f "$LIB" ] || fresh=0
if [ $fresh = 1 ]; then
    for src in "$OBJ"/*.o "$OUT/fake_cudart.o" "$HERE/kernels_cpu.cpp" "$HERE/kernels_dbm_multinomial_cpu.cpp" \
               "$HERE/kernels_dbm_ais_depth_cpu.cpp" "$HERE/kernels_dbm_ais_base_cpu.cpp" "$HERE/kernels_dbm_ais_clamped_cpu.cpp" \
               "$HERE/build_dbm_ais_clamped.sh" "$ROOT"/boltzmann-machines_b200/csrc/*.h; do
        [ "$src" -nt "$LIB" ] && fresh=0
    done
fi
if [ $fresh = 0 ]; then
    F="-O2 -g -std=c++17 -fPIC -I/usr/local/cuda/include"
    g++ $F -Dexecute=execute_base -c "$HERE/kernels_cpu.cpp" -o "$OUT/kernels_cpu_base_ais_clamped.o"
    g++ $F -Dexecute=execute_multinomial -c "$HERE/kernels_dbm_multinomial_cpu.cpp" -o "$OUT/kernels_dbm_multinomial_ais_clamped.o"
    g++ $F -Dexecute=execute_ais_depth -c "$HERE/kernels_dbm_ais_depth_cpu.cpp" -o "$OUT/kernels_dbm_ais_depth_ais_clamped.o"
    g++ $F -Dexecute=execute_ais_base -c "$HERE/kernels_dbm_ais_base_cpu.cpp" -o "$OUT/kernels_dbm_ais_base_ais_clamped.o"
    g++ $F -c "$HERE/kernels_dbm_ais_clamped_cpu.cpp" -o "$OUT/kernels_dbm_ais_clamped_cpu.o"
    g++ -shared -Wl,-Bsymbolic -o "$LIB.tmp" "$OBJ"/*.o "$OUT/fake_cudart.o" "$OUT/kernels_cpu_base_ais_clamped.o" \
        "$OUT/kernels_dbm_multinomial_ais_clamped.o" "$OUT/kernels_dbm_ais_depth_ais_clamped.o" \
        "$OUT/kernels_dbm_ais_base_ais_clamped.o" "$OUT/kernels_dbm_ais_clamped_cpu.o" -ldl -lpthread -lrt -lstdc++
    mv -f "$LIB.tmp" "$LIB"
fi
echo "built $LIB"
