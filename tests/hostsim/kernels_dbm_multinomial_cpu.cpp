// TEST INFRASTRUCTURE ONLY -- CPU restatement of dbm_multinomial_rows_kernel (csrc/bm_dbm_tc.cuh), the multinomial row kernel of
// the tensor-core DBM engine, for the stand-in runtime (fake_cudart.cpp).
//
// build_dbm_multinomial.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base and links this file in front of it:
// `execute` below interprets the row kernel and hands every other launch to kernels_cpu.cpp's restatements unchanged.
#include <cuda_runtime_api.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>
#undef __host__
#undef __device__
#undef __forceinline__
#include "../../boltzmann-machines_b200/csrc/bm_internal.h"   // RngKey, site_block (bm_rng.cuh defines the qualifiers away on the host)

namespace fakecuda {
bool execute_base(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_cpu.cpp's dispatcher

static inline __nv_bfloat16 f2bf(float f) {           // round to nearest even, as __float2bfloat16_rn
    unsigned u; memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) { u |= 0x00400000u; } else { u += 0x7fffu + ((u >> 16) & 1u); }
    unsigned short b = (unsigned short)(u >> 16); __nv_bfloat16 v; memcpy(&v, &b, 2); return v;
}
template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }

// dbm_multinomial_rows_kernel: softmax_rows_kernel<float> then multinomial_rows_kernel<float> on each row (one block per row), the
// result in bf16 and (optionally) fp32; the double sum of the exponentials in the kernel's order (256 strided partials, then its tree)
static void k_dbm_multinomial_rows(void** a, dim3 grid) {
    const float* pre = arg<const float*>(a, 0); const int ldp = arg<int>(a, 1), cols = arg<int>(a, 2); const float scale = arg<float>(a, 3);
    const int n_draws = arg<int>(a, 4); __nv_bfloat16* out = arg<__nv_bfloat16*>(a, 5); const int ldo = arg<int>(a, 6);
    float* out_f32 = arg<float*>(a, 7); const int ldf = arg<int>(a, 8); const bm::RngKey rng = arg<bm::RngKey>(a, 9);
    std::vector<float> x(cols); std::vector<double> sh(256), cdf(cols); std::vector<int> cnt(cols);
    for (unsigned r = 0; r < grid.x; ++r) {
        const float* row = pre + (size_t)r * ldp;
        double mx = -1e300;
        for (int c = 0; c < cols; ++c) { x[c] = row[c]; mx = std::fmax(mx, (double)row[c]); }
        const float m = (float)mx;
        std::fill(sh.begin(), sh.end(), 0.0);
        for (int c = 0; c < cols; ++c) { x[c] = expf(x[c] - m); sh[c % 256] += (double)x[c]; }
        for (int o = 128; o > 0; o >>= 1) for (int t = 0; t < o; ++t) sh[t] += sh[t + o];
        const float tot = (float)sh[0];
        for (int c = 0; c < cols; ++c) x[c] = scale * x[c] / tot;
        if (n_draws > 0) {
            double t = 0.0; for (int c = 0; c < cols; ++c) t += (double)x[c];
            double run = 0.0;
            for (int c = 0; c < cols; ++c) { run += (double)(float)((double)x[c] / t); cdf[c] = run; }
            const double last = cdf[cols - 1];
            for (int c = 0; c < cols; ++c) { cdf[c] = cdf[c] / last; cnt[c] = 0; }
            for (int d = 0; d < n_draws; ++d) {
                const bm::U4 w = bm::site_block(rng, r, (uint32_t)(d >> 2));
                const uint32_t words[4] = {w.x, w.y, w.z, w.w};
                const double u = (double)bm::u32_to_unit_float(words[d & 3]);
                int lo = 0, hi = cols;
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (cdf[mid] > u) hi = mid; else lo = mid + 1; }
                cnt[lo < cols ? lo : cols - 1]++;
            }
            for (int c = 0; c < cols; ++c) x[c] = (float)cnt[c];
        }
        for (int c = 0; c < cols; ++c) {
            out[(size_t)r * ldo + c] = f2bf(x[c]);
            if (out_f32) out_f32[(size_t)r * ldf + c] = x[c];
        }
    }
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("dbm_multinomial_rows_kernel") != std::string::npos) { k_dbm_multinomial_rows(args, grid); return true; }
    return execute_base(name, grid, block, args);
}

}  // namespace fakecuda
