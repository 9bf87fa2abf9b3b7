// TEST INFRASTRUCTURE ONLY -- CPU restatement of what centering adds to the tensor-core DBM engine (csrc/bm_dbm_tc.cuh,
// DESIGN.md §5.8), for the stand-in runtime (fake_cudart.cpp):
//
//   * dbm_center_stats_kernel: s_j, the first step's offsets and the moved offsets;
//   * dbm_centered_grad_combine_kernel: the split-K combine with the rank-2 (+ rank-1) correction;
//   * dbm_coupling_kernel: c_j = W_{j-1}' o_{j-1} + W_j o_{j+1} in the kernel's fp32 order (fma column partials over rows
//     y, y + 8, ...; fma lane partials over k = l, l + 32, ... and the xor tree), stored or taken out of b_j.
//
// build_dbm_centered.sh chains the dispatchers: this file -> kernels_dbm_pt_cpu.cpp (execute_pt) -> kernels_dbm_multinomial_cpu.cpp
// (execute_multinomial) -> kernels_cpu.cpp (execute_base).
#include <cuda_runtime_api.h>
#include <cmath>
#include <cstring>
#include <string>

namespace fakecuda {
bool execute_pt(const std::string& name, dim3 grid, dim3 block, void** args);

template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }

// csrc/bm_dbm_tc.cuh::CenterArgs and CouplingArgs, field for field
struct CenterArgs {
    int n_layers;
    int n[9];
    const float* dsum[9];
    const float* psum[9];
    float* o[9];
    float* o_next[9];
    float* s[9];
    float rows, inv_n, inv_m, keep, rate;
    int init;
};
struct CouplingArgs {
    int n_layers;
    int n[9];
    const float* W[8];
    const float* o[9];
    float* cpl[9];
    float* b[9];
    int mode;
};

static void k_center_stats(void** args) {
    const CenterArgs& a = *reinterpret_cast<const CenterArgs*>(args[0]);
    for (int j = 0; j < a.n_layers; ++j)
        for (int u = 0; u < a.n[j]; ++u) {
            const float d = a.dsum[j][u], mean = d / a.rows;
            float o = a.o[j][u];
            if (a.init) { o = mean; a.o[j][u] = o; }
            const float x = d * a.inv_n, y = a.psum[j][u] * a.inv_m;
            a.s[j][u] = x - y;
            const float k = a.keep * o, r = a.rate * mean;
            a.o_next[j][u] = k + r;
        }
}

static void k_centered_combine(void** a) {
    const float* pos = arg<const float*>(a, 0); const int sp = arg<int>(a, 1); const float* neg = arg<const float*>(a, 2);
    const int sn = arg<int>(a, 3); const size_t stride = arg<size_t>(a, 4); const float inv_n = arg<float>(a, 5), inv_m = arg<float>(a, 6);
    const int H = arg<int>(a, 7);
    const float* o_in = arg<const float*>(a, 8); const float* s_in = arg<const float*>(a, 9);
    const float* o_out = arg<const float*>(a, 10); const float* s_out = arg<const float*>(a, 11);
    const float corr = arg<float>(a, 12); float* G = arg<float*>(a, 13); const size_t n = arg<size_t>(a, 14);
    for (size_t i = 0; i < n; ++i) {
        float x = 0.f, y = 0.f;
        for (int s = 0; s < sp; ++s) x += pos[(size_t)s * stride + i];
        for (int s = 0; s < sn; ++s) y += neg[(size_t)s * stride + i];
        const size_t r = i / (size_t)H, c = i % (size_t)H;
        float g = x * inv_n - y * inv_m;                      // as kernels_cpu.cpp restates dbm_grad_combine_kernel
        float t = o_in[r] * s_out[c]; g = g - t;
        t = s_in[r] * o_out[c]; g = g - t;
        t = o_in[r] * o_out[c]; t = corr * t; g = g + t;
        G[i] = g;
    }
}

static void k_coupling(void** args) {
    const CouplingArgs& a = *reinterpret_cast<const CouplingArgs*>(args[0]);
    for (int j = 0; j < a.n_layers; ++j) {
        const int n = a.n[j];
        for (int u = 0; u < n; ++u) {
            float colp[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (j > 0)
                for (int y = 0; y < 8; ++y)
                    for (int r = y; r < a.n[j - 1]; r += 8) colp[y] = std::fmaf(a.W[j - 1][(size_t)r * n + u], a.o[j - 1][r], colp[y]);
            float lane[32] = {0.f};
            if (j + 1 < a.n_layers) {
                const int m = a.n[j + 1];
                for (int l = 0; l < 32; ++l)
                    for (int k = l; k < m; k += 32) lane[l] = std::fmaf(a.W[j][(size_t)u * m + k], a.o[j + 1][k], lane[l]);
            }
            for (int o = 16; o > 0; o >>= 1) {
                float t[32];
                for (int l = 0; l < 32; ++l) t[l] = lane[l] + lane[l ^ o];
                memcpy(lane, t, sizeof(t));
            }
            float c = 0.f;
            for (int y = 0; y < 8; ++y) c = c + colp[y];
            c = c + lane[0];
            if (a.mode == 0) a.cpl[j][u] = c;
            else { const float d = c - a.cpl[j][u]; a.b[j][u] = a.b[j][u] - d; }
        }
    }
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("dbm_center_stats_kernel") != std::string::npos) { k_center_stats(args); return true; }
    if (name.find("dbm_centered_grad_combine_kernel") != std::string::npos) { k_centered_combine(args); return true; }
    if (name.find("dbm_coupling_kernel") != std::string::npos) { k_coupling(args); return true; }
    return execute_pt(name, grid, block, args);
}

}  // namespace fakecuda
