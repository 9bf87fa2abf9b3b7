// TEST INFRASTRUCTURE ONLY -- CPU restatement of the row kernel of the tensor-core DBM's variational bound at depths other than 2
// (csrc/bm_dbm_tc.cuh, DESIGN.md §5.4c) for the stand-in runtime (fake_cudart.cpp):
//
//   * dbm_bound_layer_rows_kernel: out[r] (+)= t.mu + mu.c + H(clip(mu)) of one hidden layer, plus X.b_v for the first.
//
// build_dbm_ais_depth.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base and kernels_dbm_multinomial_cpu.cpp
// with its dispatcher renamed to execute_multinomial, and links this file in front of them: `execute` below interprets the row
// kernel and hands every other launch down the chain.
#include <cuda_runtime_api.h>
#include <cmath>
#include <cstdint>
#include <string>

namespace fakecuda {
bool execute_multinomial(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_dbm_multinomial_cpu.cpp

template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }

// dbm_bound_layer_rows_kernel(X, V, vb, mu, t, hb, H, first, rows, out)
static void k_bound_layer_rows(void** a) {
    const float* X = arg<const float*>(a, 0); const int V = arg<int>(a, 1); const float* vb = arg<const float*>(a, 2);
    const float* mu = arg<const float*>(a, 3); const float* t = arg<const float*>(a, 4); const float* hb = arg<const float*>(a, 5);
    const int H = arg<int>(a, 6), first = arg<int>(a, 7), rows = arg<int>(a, 8); double* out = arg<double*>(a, 9);
    for (int r = 0; r < rows; ++r) {
        double acc = 0.0;
        for (int j = 0; j < H; ++j) {
            const double m = (double)mu[(size_t)r * H + j];
            acc += (double)t[(size_t)r * H + j] * m + m * (double)hb[j];
            const double s = (double)fminf(fmaxf((float)m, 1e-7f), 1.0f - 1e-7f);
            acc += -s * std::log(s) - (1.0 - s) * std::log(1.0 - s);
        }
        if (first)
            for (int j = 0; j < V; ++j) acc += (double)X[(size_t)r * V + j] * (double)vb[j];
        out[r] = first ? acc : out[r] + acc;
    }
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("dbm_bound_layer_rows_kernel") != std::string::npos) { k_bound_layer_rows(args); return true; }
    return execute_multinomial(name, grid, block, args);
}

}  // namespace fakecuda
