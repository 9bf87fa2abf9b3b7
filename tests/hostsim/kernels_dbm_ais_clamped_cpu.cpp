// TEST INFRASTRUCTURE ONLY -- CPU restatement of the operand kernel of AIS with v clamped (csrc/bm_dbm_tc.cuh, DESIGN.md §5.4g)
// for the stand-in runtime (fake_cudart.cpp):
//
//   * ais_clamp_rows_kernel: chain i of a slice reads row (c0 + i) / n_runs of X; out [n, ldo] bf16, the padding columns zero.
//
// build_dbm_ais_clamped.sh links this file in front of the base-rate restatement (kernels_dbm_ais_base_cpu.cpp, dispatcher
// renamed to execute_ais_base), which falls back to the depth, the multinomial and then kernels_cpu.cpp's restatements.
#include <cuda_runtime_api.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstring>
#include <string>

namespace fakecuda {
bool execute_ais_base(const std::string& name, dim3 grid, dim3 block, void** args);      // kernels_dbm_ais_base_cpu.cpp

template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }

static inline __nv_bfloat16 f2bf(float f) {           // round to nearest even, as kernels_cpu.cpp
    unsigned u; memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) { u |= 0x00400000u; } else { u += 0x7fffu + ((u >> 16) & 1u); }
    unsigned short b = (unsigned short)(u >> 16); __nv_bfloat16 v; memcpy(&v, &b, 2); return v;
}

// ais_clamp_rows_kernel(X, V, c0, n_runs, out, ldo, n)
static void k_clamp_rows(void** a) {
    const float* X = arg<const float*>(a, 0); const int V = arg<int>(a, 1); const long long c0 = arg<long long>(a, 2);
    const int n_runs = arg<int>(a, 3); __nv_bfloat16* out = arg<__nv_bfloat16*>(a, 4);
    const int ldo = arg<int>(a, 5), n = arg<int>(a, 6);
    for (int i = 0; i < n; ++i) {
        const float* x = X + (size_t)((c0 + i) / n_runs) * V;
        for (int c = 0; c < ldo; ++c) out[(size_t)i * ldo + c] = f2bf(c < V ? x[c] : 0.f);
    }
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("ais_clamp_rows_kernel") != std::string::npos) { k_clamp_rows(args); return true; }
    return execute_ais_base(name, grid, block, args);
}

}  // namespace fakecuda
