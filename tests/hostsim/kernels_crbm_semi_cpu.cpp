// TEST INFRASTRUCTURE ONLY -- CPU restatements of the classification RBM's kernels (csrc/bm_crbm_tc.cuh) for the stand-in runtime
// (fake_cudart.cpp): crbm_posterior_rows_kernel, crbm_columns_kernel, crbm_chain_stats_kernel and crbm_update_kernel, with the
// semi-supervised terms of rows labelled -1 (the start-label draw, the beta-weighted columns and separate chain statistics).
// kernels_crbm_cpu.cpp restates the same kernels for labelled batches only; on such batches the two agree.
//
// build_crbm_semi.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base and kernels_dbm_multinomial_cpu.cpp
// (the label's row kernel) with its dispatcher renamed to execute_multinomial, and links this file in front of both: `execute`
// below interprets the four kernels and hands every other launch down the chain unchanged.
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
bool execute_multinomial(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_dbm_multinomial_cpu.cpp

static inline float bf2f(__nv_bfloat16 v) { unsigned short b; memcpy(&b, &v, 2); unsigned u = (unsigned)b << 16; float f; memcpy(&f, &u, 4); return f; }
static inline __nv_bfloat16 f2bf(float f) {           // round to nearest even, as __float2bfloat16_rn
    unsigned u; memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) { u |= 0x00400000u; } else { u += 0x7fffu + ((u >> 16) & 1u); }
    unsigned short b = (unsigned short)(u >> 16); __nv_bfloat16 v; memcpy(&v, &b, 2); return v;
}
template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }
static inline float softplus_f(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
static inline float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// one 256-thread block per row: thread t sums j = t, t + 256, ... in double; per warp the xor butterfly (every lane ends with the
// same value; lane 0's is kept), then the 8 warp sums in warp order
static void k_posterior(void** a, dim3 grid) {
    const float* A = arg<const float*>(a, 0); const int H = arg<int>(a, 1); const float* U1 = arg<const float*>(a, 2);
    const int C = arg<int>(a, 3); const float* hb = arg<const float*>(a, 4); const float* yb = arg<const float*>(a, 5);
    const int* labels = arg<const int*>(a, 6); float* P = arg<float*>(a, 7); double* nll = arg<double*>(a, 8); int* correct = arg<int*>(a, 9);
    const bm::RngKey yrng = arg<bm::RngKey>(a, 10); int* y0 = arg<int*>(a, 11);
    std::vector<double> acc(256), lane(32), F(C);
    for (unsigned r = 0; r < grid.x; ++r) {
        std::vector<double> part((size_t)8 * C);
        for (int y = 0; y < C; ++y) {
            for (int t = 0; t < 256; ++t) {
                double s = 0.0;
                for (int j = t; j < H; j += 256) {
                    const float av = A[(size_t)r * H + j] + hb[j];
                    s += (double)softplus_f(av + U1[(size_t)j * C + y]);
                }
                acc[t] = s;
            }
            for (int w = 0; w < 8; ++w) {
                for (int l = 0; l < 32; ++l) lane[l] = acc[w * 32 + l];
                for (int o = 16; o > 0; o >>= 1) {
                    std::vector<double> nx(32);
                    for (int l = 0; l < 32; ++l) nx[l] = lane[l] + lane[l ^ o];
                    lane = nx;
                }
                part[(size_t)w * C + y] = lane[0];
            }
        }
        double m = -1e300; int best = 0;
        for (int y = 0; y < C; ++y) {
            double s = 0.0;
            for (int w = 0; w < 8; ++w) s += part[(size_t)w * C + y];
            F[y] = (double)yb[y] + s;
            if (F[y] > m) { m = F[y]; best = y; }
        }
        double z = 0.0;
        for (int y = 0; y < C; ++y) z += exp(F[y] - m);
        const double logz = m + log(z);
        for (int y = 0; y < C; ++y) P[(size_t)r * C + y] = (float)exp(F[y] - logz);
        if (labels) {
            const int t = labels[r];
            if (t < 0) {                 // unlabelled: the chain's start label, one categorical draw from the float32 row
                const float* pr = P + (size_t)r * C;
                double tot = 0.0, last = 0.0, run = 0.0;
                for (int y = 0; y < C; ++y) tot += (double)pr[y];
                for (int y = 0; y < C; ++y) last += (double)(float)((double)pr[y] / tot);
                const double u = (double)bm::u32_to_unit_float(bm::site_block(yrng, r, 0u).x);
                int pick = C - 1;
                for (int y = 0; y < C; ++y) {
                    run += (double)(float)((double)pr[y] / tot);
                    if (run / last > u) { pick = y; break; }
                }
                y0[r] = pick;
                continue;
            }
            double Ft = 0.0;
            for (int y = 0; y < C; ++y) if (y == t) Ft = F[y];
            nll[r] = logz - Ft;
            correct[r] = best == t ? 1 : 0;
        }
    }
}

static void k_columns(void** a, dim3 grid, dim3 block) {
    const float* A = arg<const float*>(a, 0); const int H = arg<int>(a, 1); const float* U1 = arg<const float*>(a, 2);
    const int C = arg<int>(a, 3); const float* hb = arg<const float*>(a, 4); const float* P = arg<const float*>(a, 5);
    const int* labels = arg<const int*>(a, 6); const int rows = arg<int>(a, 7), rps = arg<int>(a, 8); const float alpha = arg<float>(a, 9);
    __nv_bfloat16* G = arg<__nv_bfloat16*>(a, 10); const int ldg = arg<int>(a, 11); __nv_bfloat16* h0 = arg<__nv_bfloat16*>(a, 12);
    const int ldh = arg<int>(a, 13); const int sample_h = arg<int>(a, 14); const bm::RngKey rng = arg<bm::RngKey>(a, 15);
    float* Sh = arg<float*>(a, 16); float* gU = arg<float*>(a, 17); float* ghb = arg<float*>(a, 18); float* gyb = arg<float*>(a, 19);
    const int* y0 = arg<const int*>(a, 20); const float beta = arg<float>(a, 21);
    const float pos = 1.0f + alpha;
    std::vector<float> gu(C);
    for (unsigned s = 0; s < grid.y; ++s) {
        const int r0 = (int)s * rps, r1 = std::min(rows, r0 + rps);
        for (unsigned bx = 0; bx < grid.x; ++bx)
            for (unsigned tx = 0; tx < block.x; ++tx) {
                const int j = (int)(bx * block.x + tx);
                const bool col = j < H, ycol = gyb && bx == 0 && (int)tx < C;
                if (!col && !ycol) continue;
                std::fill(gu.begin(), gu.end(), 0.f);
                float hsum = 0.f, ysum = 0.f;
                for (int r = r0; r < r1; ++r) {
                    const float* pr = P + (size_t)r * C;
                    const int t = labels ? labels[r] : -1;
                    const bool unl = y0 && t < 0;
                    const int ts = unl ? y0[r] : t;
                    if (col) {
                        const float av = A[(size_t)r * H + j] + hb[j];
                        float sh = 0.f, st = 0.f;
                        for (int y = 0; y < C; ++y) {
                            const float sy = sigmoid_f(av + U1[(size_t)j * C + y]);
                            sh += pr[y] * sy;
                            if (y == ts) st = sy;
                            if (gU) gu[y] += (unl ? beta * pr[y] : (y == t ? pos : 0.f) - pr[y]) * sy;
                        }
                        if (Sh) Sh[(size_t)r * H + j] = sh;
                        if (G) { const float g = unl ? beta * sh : pos * st - sh; G[(size_t)r * ldg + j] = f2bf(g); hsum += g; }
                        if (h0) {
                            float h = st;
                            if (sample_h) {
                                const bm::U4 w = bm::site_block(rng, (uint32_t)r, (uint32_t)(j >> 2));
                                const uint32_t words[4] = {w.x, w.y, w.z, w.w};
                                h = bm::u32_to_unit_float(words[j & 3]) < st ? 1.f : 0.f;
                            }
                            h0[(size_t)r * ldh + j] = f2bf(h);
                        }
                    }
                    if (ycol) ysum += unl ? beta * pr[tx] : ((int)tx == t ? pos : 0.f) - pr[tx];
                }
                if (col && gU) for (int y = 0; y < C; ++y) gU[((size_t)s * C + y) * H + j] = gu[y];
                if (col && ghb) ghb[(size_t)s * H + j] = hsum;
                if (ycol) gyb[(size_t)s * C + tx] = ysum;
            }
    }
}

static void k_chain_stats(void** a, dim3 grid, dim3 block) {
    const __nv_bfloat16* Hk = arg<const __nv_bfloat16*>(a, 0); const int ldh = arg<int>(a, 1);
    const __nv_bfloat16* Yk = arg<const __nv_bfloat16*>(a, 2); const int ldy = arg<int>(a, 3), C = arg<int>(a, 4);
    const __nv_bfloat16* X = arg<const __nv_bfloat16*>(a, 5); const __nv_bfloat16* Xk = arg<const __nv_bfloat16*>(a, 6);
    const int ldx = arg<int>(a, 7), V = arg<int>(a, 8), H = arg<int>(a, 9), rows = arg<int>(a, 10), rps = arg<int>(a, 11);
    const float alpha = arg<float>(a, 12); __nv_bfloat16* aH = arg<__nv_bfloat16*>(a, 13);
    float* yh = arg<float*>(a, 14); float* hk = arg<float*>(a, 15); float* xd = arg<float*>(a, 16); float* yk = arg<float*>(a, 17);
    const int* labels = arg<const int*>(a, 18); const float beta = arg<float>(a, 19);
    float* outs[2][4] = {{yh, hk, xd, yk}, {arg<float*>(a, 20), arg<float*>(a, 21), arg<float*>(a, 22), arg<float*>(a, 23)}};
    const int passes = outs[1][0] ? 2 : 1;     // pass 0: labelled rows (alpha), pass 1: unlabelled rows (beta)
    std::vector<float> acc(C);
    for (unsigned s = 0; s < grid.y; ++s) {
        const int r0 = (int)s * rps, r1 = std::min(rows, r0 + rps);
        for (unsigned bx = 0; bx < grid.x; ++bx)
            for (unsigned tx = 0; tx < block.x; ++tx)
                for (int pass = 0; pass < passes; ++pass) {
                    const float w = pass ? beta : alpha;
                    float *oyh = outs[pass][0], *ohk = outs[pass][1], *oxd = outs[pass][2], *oyk = outs[pass][3];
                    const int j = (int)(bx * block.x + tx);
                    const bool hcol = j < H, xcol = j < V, ycol = bx == 0 && (int)tx < C;
                    std::fill(acc.begin(), acc.end(), 0.f);
                    float hs = 0.f, xs = 0.f, ys = 0.f;
                    for (int r = r0; r < r1; ++r) {
                        if (passes == 2 && (labels[r] < 0) != (pass == 1)) continue;
                        const __nv_bfloat16* yr = Yk + (size_t)r * ldy;
                        if (hcol) {
                            const float h = bf2f(Hk[(size_t)r * ldh + j]);
                            hs += h;
                            aH[(size_t)r * ldh + j] = f2bf(w * h);
                            for (int y = 0; y < C; ++y) acc[y] += bf2f(yr[y]) * h;
                        }
                        if (xcol) xs += bf2f(X[(size_t)r * ldx + j]) - bf2f(Xk[(size_t)r * ldx + j]);
                        if (ycol) ys += bf2f(yr[tx]);
                    }
                    if (hcol) {
                        for (int y = 0; y < C; ++y) oyh[((size_t)s * C + y) * H + j] = acc[y];
                        ohk[(size_t)s * H + j] = hs;
                    }
                    if (xcol) oxd[(size_t)s * V + j] = xs;
                    if (ycol) oyk[(size_t)s * C + tx] = ys;
                }
    }
}

struct CrbmUpdate {      // the kernel's by-value argument (csrc/bm_crbm_tc.cuh), field for field
    int V, H, C, ld1, ld2;
    float *W, *dW, *U1, *dU1, *vb, *dvb, *hb, *dhb, *yb, *dyb;
    __nv_bfloat16 *Wb, *U1b, *UbT;
    const float *Wp; int s1; size_t wstride;
    const float *gU, *ghb, *gyb; int s2;
    const float *yh, *hk, *xd, *yk; int s3;
    float alpha, N, l2, lr, mom;
    const float *yhu, *hku, *xdu, *yku; int s4;
    float beta;
};
static inline float split_sum(const float* p, int n, size_t stride, size_t i) {
    float b = 0.f;
    for (int s = 0; s < n; ++s) b += p[(size_t)s * stride + i];
    return b;
}
static void k_update(void** a) {
    const CrbmUpdate u = arg<CrbmUpdate>(a, 0);
    const size_t nW = (size_t)u.V * u.H, nU = (size_t)u.C * u.H;
    const size_t n = nW + nU + u.V + u.H + u.C;
    for (size_t i = 0; i < n; ++i) {
        float g, *th, *d;
        if (i < nW) {
            float s = 0.f;
            for (int k = 0; k < u.s1; ++k) s += u.Wp[(size_t)k * u.wstride + i];
            th = u.W + i; d = u.dW + i;
            g = s / u.N - u.l2 * *th;
        } else if (i < nW + nU) {
            const size_t k = i - nW;
            const int y = (int)(k / u.H), j = (int)(k % u.H);
            float s = 0.f, b = 0.f;
            for (int q = 0; q < u.s2; ++q) s += u.gU[(size_t)q * nU + k];
            for (int q = 0; q < u.s3; ++q) b += u.yh[(size_t)q * nU + k];
            th = u.U1 + (size_t)j * u.C + y; d = u.dU1 + (size_t)j * u.C + y;
            float c = s - u.alpha * b;
            if (u.s4) c -= u.beta * split_sum(u.yhu, u.s4, nU, k);
            g = c / u.N - u.l2 * *th;
        } else if (i < nW + nU + u.V) {
            const int j = (int)(i - nW - nU);
            float b = 0.f;
            for (int q = 0; q < u.s3; ++q) b += u.xd[(size_t)q * u.V + j];
            th = u.vb + j; d = u.dvb + j;
            float c = u.alpha * b;
            if (u.s4) c += u.beta * split_sum(u.xdu, u.s4, u.V, j);
            g = c / u.N;
        } else if (i < nW + nU + u.V + u.H) {
            const int j = (int)(i - nW - nU - u.V);
            float s = 0.f, b = 0.f;
            for (int q = 0; q < u.s2; ++q) s += u.ghb[(size_t)q * u.H + j];
            for (int q = 0; q < u.s3; ++q) b += u.hk[(size_t)q * u.H + j];
            th = u.hb + j; d = u.dhb + j;
            float c = s - u.alpha * b;
            if (u.s4) c -= u.beta * split_sum(u.hku, u.s4, u.H, j);
            g = c / u.N;
        } else {
            const int y = (int)(i - nW - nU - u.V - u.H);
            float s = 0.f, b = 0.f;
            for (int q = 0; q < u.s2; ++q) s += u.gyb[(size_t)q * u.C + y];
            for (int q = 0; q < u.s3; ++q) b += u.yk[(size_t)q * u.C + y];
            th = u.yb + y; d = u.dyb + y;
            float c = s - u.alpha * b;
            if (u.s4) c -= u.beta * split_sum(u.yku, u.s4, u.C, y);
            g = c / u.N;
        }
        const float dd = u.lr * (u.mom * *d + g);
        *d = dd;
        const float v = *th + dd;
        *th = v;
        if (i < nW) u.Wb[(i / u.H) * u.ld1 + i % u.H] = f2bf(v);
        else if (i < nW + nU) {
            const size_t k = i - nW, y = k / u.H, j = k % u.H;
            u.U1b[j * u.ld2 + y] = f2bf(v);
            u.UbT[y * u.ld1 + j] = f2bf(v);
        }
    }
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("crbm_posterior_rows_kernel") != std::string::npos) { k_posterior(args, grid); return true; }
    if (name.find("crbm_columns_kernel") != std::string::npos) { k_columns(args, grid, block); return true; }
    if (name.find("crbm_chain_stats_kernel") != std::string::npos) { k_chain_stats(args, grid, block); return true; }
    if (name.find("crbm_update_kernel") != std::string::npos) { k_update(args); return true; }
    return execute_multinomial(name, grid, block, args);
}

}  // namespace fakecuda
