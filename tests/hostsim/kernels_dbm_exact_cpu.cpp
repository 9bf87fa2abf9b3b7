// TEST INFRASTRUCTURE ONLY -- CPU restatements of the kernels of the exact log Z / log p*(v) enumeration
// (csrc/bm_dbm_exact.cuh, DESIGN.md §5.4f) for the stand-in runtime (fake_cudart.cpp):
//
//   * dbm_exact_states_kernel: per state s, z = (sum of the hi terms of the bits set) + (sum of the lo terms) in fp32, + bias;
//     the softplus of each column pair in fp32 added to a float64 row sum; log p* = c.x + all columns, g = c.x + the columns
//     before n_rest; per CTA of 512 states the pair (max, sum exp(log p* - max));
//   * dbm_exact_rows_kernel: per row r and CTA of 8192 states, the running (max, sum) of q_r.x_1 + g (q_r's three bf16 terms
//     summed in fp32, the exponentials in fp32, the sum in float64);
//   * dbm_exact_merge_kernel, dbm_exact_query_kernel: as the kernels, in float64.
//
// build_dbm_exact.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base and links this file in front of it:
// `execute` below interprets these kernels and hands every other launch down.
#include <cuda_runtime_api.h>
#include <cuda_bf16.h>
#include <vector_functions.h>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace fakecuda {
bool execute_base(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_cpu.cpp

namespace {
template <class T> inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }

// the argument structs of csrc/bm_dbm_exact.cuh, field for field
struct ExactStatesArgs {
    const uint32_t* B; const float* bias; const double* c; int ks; int n_pad, n_rest; int n_bits; uint32_t s0, n;
    double* g; double2* part;
};
struct ExactRowsArgs { const uint32_t* Q; const double* g; int ks1; int rows; uint32_t s0, n; double2* part; };

inline float bf(uint16_t h) { uint32_t u = (uint32_t)h << 16; float f; std::memcpy(&f, &u, 4); return f; }
inline float softplus(float z) { return std::fmax(z, 0.f) + log1pf(expf(-std::fabs(z))); }
inline void merge(double& m, double& s, double m2, double s2) {
    const double M = std::max(m, m2);
    if (M == -INFINITY) return;
    s = s * std::exp(m - M) + s2 * std::exp(m2 - M);
    m = M;
}

void k_states(void** a_, dim3 grid) {
    const ExactStatesArgs a = arg<ExactStatesArgs>(a_, 0);
    const int KB = 16 * a.ks;
    const uint16_t* B = reinterpret_cast<const uint16_t*>(a.B);
    std::vector<double> lp(512);
    for (unsigned b = 0; b < grid.x; ++b) {
        double mx = -INFINITY;
        for (int i = 0; i < 512; ++i) {
            const uint32_t off = b * 512u + (uint32_t)i;
            lp[i] = -INFINITY;
            if (off >= a.n) continue;
            const uint32_t s = a.s0 + off;
            double tot = 0.0, rest = 0.0;
            for (int n0 = 0; n0 < a.n_pad; n0 += 2) {
                if (n0 == a.n_rest) rest = tot;
                float sp[2];
                for (int j = 0; j < 2; ++j) {
                    const uint16_t* col = B + (size_t)(n0 + j) * 2 * KB;
                    float acc = 0.f;
                    for (int k = 0; k < KB; ++k) if ((s >> k) & 1u) acc += bf(col[k]);
                    for (int k = 0; k < KB; ++k) if ((s >> k) & 1u) acc += bf(col[KB + k]);
                    sp[j] = softplus(acc + a.bias[n0 + j]);
                }
                tot += (double)(sp[0] + sp[1]);
            }
            double lin = 0.0;
            for (int k = 0; k < a.n_bits; ++k) if ((s >> k) & 1u) lin += a.c[k];
            lp[i] = lin + tot;
            if (a.g) a.g[off] = lin + rest;
            mx = std::max(mx, lp[i]);
        }
        double S = 0.0;
        if (mx != -INFINITY)
            for (int i = 0; i < 512; ++i) if (lp[i] != -INFINITY) S += std::exp(lp[i] - mx);
        a.part[b] = make_double2(mx, S);
    }
}

void k_rows(void** a_, dim3 grid) {
    const ExactRowsArgs a = arg<ExactRowsArgs>(a_, 0);
    const int KB1 = 16 * a.ks1;
    const uint16_t* Q = reinterpret_cast<const uint16_t*>(a.Q);
    for (int r = 0; r < a.rows; ++r) {
        const uint16_t* q = Q + (size_t)r * 3 * KB1;
        for (unsigned b = 0; b < grid.x; ++b) {
            const uint32_t lo = b * 8192u, hi = std::min(lo + 8192u, a.n);
            double m = -INFINITY, s = 0.0;
            for (uint32_t t = lo; t < hi; ++t) {
                const uint32_t key = a.s0 + t;
                float acc = 0.f;
                for (int p = 0; p < 3; ++p)
                    for (int k = 0; k < KB1; ++k) if ((key >> k) & 1u) acc += bf(q[p * KB1 + k]);
                const double v = (double)acc + a.g[t];
                if (v > m) { s = s * (double)expf((float)(m - v)) + 1.0; m = v; }
                else s += (double)expf((float)(v - m));
            }
            a.part[(size_t)r * grid.x + b] = make_double2(m, s);
        }
    }
}

// dbm_exact_merge_kernel(part, n, acc)
void k_merge(void** a, dim3 grid) {
    const double2* part = arg<const double2*>(a, 0); const int n = arg<int>(a, 1); double2* acc = arg<double2*>(a, 2);
    for (unsigned r = 0; r < grid.x; ++r) {
        double m = -INFINITY, s = 0.0;
        for (int i = 0; i < n; ++i) merge(m, s, part[(size_t)r * n + i].x, part[(size_t)r * n + i].y);
        double2 t = acc[r];
        merge(t.x, t.y, m, s);
        acc[r] = t;
    }
}

// dbm_exact_query_kernel(X, V, W0, n1, vb, kb1, Q, bv)
void k_query(void** a, dim3 grid) {
    const float* X = arg<const float*>(a, 0); const int V = arg<int>(a, 1); const float* W0 = arg<const float*>(a, 2);
    const int n1 = arg<int>(a, 3); const float* vb = arg<const float*>(a, 4); const int kb1 = arg<int>(a, 5);
    __nv_bfloat16* Q = arg<__nv_bfloat16*>(a, 6); double* bv = arg<double*>(a, 7);
    for (unsigned r = 0; r < grid.x; ++r) {
        const float* x = X + (size_t)r * V;
        for (int i = 0; i < kb1; ++i) {
            double q = 0.0;
            if (i < n1) for (int v = 0; v < V; ++v) q += (double)x[v] * (double)W0[(size_t)v * n1 + i];
            const __nv_bfloat16 h = __float2bfloat16_rn((float)q);
            const double r1 = q - (double)__bfloat162float(h);
            const __nv_bfloat16 md = __float2bfloat16_rn((float)r1);
            const __nv_bfloat16 l = __float2bfloat16_rn((float)(r1 - (double)__bfloat162float(md)));
            __nv_bfloat16* row = Q + (size_t)r * 3 * kb1;
            row[i] = h; row[kb1 + i] = md; row[2 * kb1 + i] = l;
        }
        double b = 0.0;
        for (int v = 0; v < V; ++v) b += (double)x[v] * (double)vb[v];
        bv[r] = b;
    }
}
}  // namespace

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("dbm_exact_states_kernel") != std::string::npos) { k_states(args, grid); return true; }
    if (name.find("dbm_exact_rows_kernel") != std::string::npos) { k_rows(args, grid); return true; }
    if (name.find("dbm_exact_merge_kernel") != std::string::npos) { k_merge(args, grid); return true; }
    if (name.find("dbm_exact_query_kernel") != std::string::npos) { k_query(args, grid); return true; }
    return execute_base(name, grid, block, args);
}

}  // namespace fakecuda
