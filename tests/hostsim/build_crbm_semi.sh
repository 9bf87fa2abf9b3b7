#!/bin/bash
# TEST INFRASTRUCTURE: the stand-in-runtime library of build.sh plus the CPU restatements of the classification RBM's kernels
# with the semi-supervised terms of rows labelled -1 (kernels_crbm_semi_cpu.cpp) and of the multinomial row kernel that draws
# its label (kernels_dbm_multinomial_cpu.cpp) -> tests/hostsim/_build/libbm_hostsim_crbm_semi.so.  Dispatch chain:
# kernels_crbm_semi_cpu.cpp's execute -> execute_multinomial (the row kernel's file, its dispatcher renamed) -> execute_base
# (kernels_cpu.cpp, its dispatcher renamed).  kernels_crbm_cpu.cpp (build_crbm.sh) restates the same kernels for labelled
# batches only.
# Safe to call from several processes at once; nothing is rebuilt while it is newer than its inputs.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OBJ="$ROOT/boltzmann-machines_b200/build"
OUT="$HERE/_build"
LIB="$OUT/libbm_hostsim_crbm_semi.so"
bash "$HERE/build.sh" > /dev/null                     # fake_cudart.o and the library's objects
exec 7> "$OUT/.lock_crbm_semi"
flock 7
fresh=1
[ -f "$LIB" ] || fresh=0
if [ $fresh = 1 ]; then
    for src in "$OBJ"/*.o "$OUT/fake_cudart.o" "$HERE/kernels_cpu.cpp" "$HERE/kernels_dbm_multinomial_cpu.cpp" \
               "$HERE/kernels_crbm_semi_cpu.cpp" "$HERE/build_crbm_semi.sh" "$ROOT"/boltzmann-machines_b200/csrc/*.h \
               "$ROOT"/boltzmann-machines_b200/csrc/*.cuh; do
        [ "$src" -nt "$LIB" ] && fresh=0
    done
fi
if [ $fresh = 0 ]; then
    F="-O2 -g -std=c++17 -fPIC -I/usr/local/cuda/include"
    g++ $F -Dexecute=execute_base -c "$HERE/kernels_cpu.cpp" -o "$OUT/kernels_cpu_base_crbm_semi.o"
    g++ $F -Dexecute=execute_multinomial -c "$HERE/kernels_dbm_multinomial_cpu.cpp" -o "$OUT/kernels_dbm_multinomial_chained_semi.o"
    g++ $F -c "$HERE/kernels_crbm_semi_cpu.cpp" -o "$OUT/kernels_crbm_semi_cpu.o"
    g++ -shared -Wl,-Bsymbolic -o "$LIB.tmp" "$OBJ"/*.o "$OUT/fake_cudart.o" "$OUT/kernels_cpu_base_crbm_semi.o" \
        "$OUT/kernels_dbm_multinomial_chained_semi.o" "$OUT/kernels_crbm_semi_cpu.o" -ldl -lpthread -lrt -lstdc++
    mv -f "$LIB.tmp" "$LIB"
fi
echo "built $LIB"
