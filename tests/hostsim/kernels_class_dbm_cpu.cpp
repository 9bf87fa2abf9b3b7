// TEST INFRASTRUCTURE ONLY -- CPU restatement of cdbm_clamp_labels_kernel (csrc/bm_dbm_tc.cuh), the label clamp of the classification
// DBM, for the stand-in runtime (fake_cudart.cpp).
//
// build_class_dbm.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base and kernels_dbm_multinomial_cpu.cpp with
// its dispatcher renamed to execute_multinomial, and links this file in front of both: `execute` below interprets the clamp and
// hands every other launch to the multinomial row kernel's restatement, which hands the rest to kernels_cpu.cpp.
#include <cuda_runtime_api.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstring>
#include <string>

namespace fakecuda {
bool execute_multinomial(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_dbm_multinomial_cpu.cpp

template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }

// cdbm_clamp_labels_kernel(labels, rows, cols, out, ld, slot_stride): rows with label t >= 0 become e_t in every slot (grid.y)
static void k_cdbm_clamp_labels(void** a, dim3 grid) {
    const int* labels = arg<const int*>(a, 0); const int rows = arg<int>(a, 1), cols = arg<int>(a, 2);
    __nv_bfloat16* out = arg<__nv_bfloat16*>(a, 3); const int ld = arg<int>(a, 4); const size_t stride = arg<size_t>(a, 5);
    const unsigned short one = 0x3f80, zero = 0;                // bf16 1.0 and +0.0
    for (unsigned s = 0; s < grid.y; ++s)
        for (int r = 0; r < rows; ++r) {
            const int t = labels[r];
            if (t < 0) continue;
            __nv_bfloat16* row = out + (size_t)s * stride + (size_t)r * ld;
            for (int c = 0; c < cols; ++c) memcpy(&row[c], c == t ? &one : &zero, 2);
        }
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("cdbm_clamp_labels_kernel") != std::string::npos) { k_cdbm_clamp_labels(args, grid); return true; }
    return execute_multinomial(name, grid, block, args);
}

}  // namespace fakecuda
