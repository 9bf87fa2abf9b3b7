// TEST INFRASTRUCTURE ONLY -- CPU restatement of the clamped Gibbs chains' kernels (csrc/bm_dbm.cu, DESIGN.md §5.9) for the
// stand-in runtime (fake_cudart.cpp):
//
//   * dbm_fill_clamp_kernel<S>: v[r, c] <- X[r, c] wherever mask[r, c] is set (S = bf16, float, double);
//   * dbm_fill_out_kernel<S, T>: out[r, c] = mask ? X[r, c] : T(mean[r, c]).
//
// build_dbm_fill.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base, kernels_dbm_multinomial_cpu.cpp with its
// dispatcher renamed to execute_multinomial and kernels_class_dbm_cpu.cpp with its dispatcher renamed to execute_class_dbm, and
// links this file in front of them: `execute` below interprets the two kernels and hands every other launch down the chain.
#include <cuda_runtime_api.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstring>
#include <string>

namespace fakecuda {
bool execute_class_dbm(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_class_dbm_cpu.cpp

template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }

static inline float widen(__nv_bfloat16 b) { unsigned short s; memcpy(&s, &b, 2); unsigned u = (unsigned)s << 16; float f; memcpy(&f, &u, 4); return f; }
static inline float widen(float x) { return x; }
static inline double widen(double x) { return x; }

// dbm_fill_clamp_kernel<S>(mask, X, ldx, v, ldv, rows, cols)
template <class S>
static void k_fill_clamp(void** a) {
    const uint8_t* mask = arg<const uint8_t*>(a, 0); const S* X = arg<const S*>(a, 1); const int ldx = arg<int>(a, 2);
    S* v = arg<S*>(a, 3); const int ldv = arg<int>(a, 4), rows = arg<int>(a, 5), cols = arg<int>(a, 6);
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c)
            if (mask[(size_t)r * cols + c]) v[(size_t)r * ldv + c] = X[(size_t)r * ldx + c];
}
// dbm_fill_out_kernel<S, T>(mask, X, mean, ldm, out, rows, cols)
template <class S, class T>
static void k_fill_out(void** a) {
    const uint8_t* mask = arg<const uint8_t*>(a, 0); const T* X = arg<const T*>(a, 1); const S* mean = arg<const S*>(a, 2);
    const int ldm = arg<int>(a, 3); T* out = arg<T*>(a, 4); const int rows = arg<int>(a, 5), cols = arg<int>(a, 6);
    for (int r = 0; r < rows; ++r)
        for (int c = 0; c < cols; ++c) {
            const size_t i = (size_t)r * cols + c;
            out[i] = mask[i] ? X[i] : (T)widen(mean[(size_t)r * ldm + c]);
        }
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    auto has = [&](const char* s) { return name.find(s) != std::string::npos; };
    // the instantiation from the mangled name: "I13__nv_bfloat16E", "IfE", "IdE"; the out kernel's pair "I13__nv_bfloat16fE", ...
    if (has("dbm_fill_clamp_kernelI13__nv_bfloat16E")) { k_fill_clamp<__nv_bfloat16>(args); return true; }
    if (has("dbm_fill_clamp_kernelIfE")) { k_fill_clamp<float>(args); return true; }
    if (has("dbm_fill_clamp_kernelIdE")) { k_fill_clamp<double>(args); return true; }
    if (has("dbm_fill_out_kernelI13__nv_bfloat16fE")) { k_fill_out<__nv_bfloat16, float>(args); return true; }
    if (has("dbm_fill_out_kernelIffE")) { k_fill_out<float, float>(args); return true; }
    if (has("dbm_fill_out_kernelIddE")) { k_fill_out<double, double>(args); return true; }
    return execute_class_dbm(name, grid, block, args);
}

}  // namespace fakecuda
