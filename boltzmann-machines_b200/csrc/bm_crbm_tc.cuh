// Classification RBM (Larochelle & Bengio, ICML 2008) on the tensor cores: included by bm_dbm.cu after bm_dbm_tc.cuh.
//
// Units x in {0,1}^V, a one-of-C label y and h in {0,1}^H; energy E = -x'W h - e_y'U h - vb'x - hb'h - yb'e_y.  The class
// posterior is exact:
//   o[b,y,j] = hb_j + U[y,j] + (x_b W)_j,   F[b,y] = yb_y + sum_j softplus(o[b,y,j]),   p(y|x_b) = softmax_y F[b,.]
// and a training step takes grad = g_disc + alpha g_gen - l2 theta (l2 on W and U), then d <- lr (momentum d + grad),
// theta += d.  g_disc is the gradient of the batch mean of log p(t|x); g_gen is CD-k on the joint p(x, y).
//
// The joint is an x - h - y chain, i.e. a two-layer DBM whose top layer is a multinomial group with n_samples = 1 and whose
// W_1 is U^T ([H, C]).  ClassRbmTC therefore IS a DbmTC of that shape: it keeps DbmTC's variables, bf16 shadows and op builders
// (hidden_gemm: h | x, y as one two-pair op; visible_gemm: x | h; hidden_tc(1): y | h as a raw fp32 op followed by
// dbm_multinomial_rows_kernel) and adds what no DBM op computes -- the posterior and the discriminative gradient:
//   forward   A = X W                                   MODE_RAW_F32 tensor-core op (fp32 out, no bias)
//   posterior crbm_posterior_rows_kernel               F, p, -log p(t|x), correctness (one block per row)
//   columns   crbm_columns_kernel                      G = (1+alpha) S_t - S^ (bf16 operand), the h0 the chain starts from,
//                                                        split partials of g_U, g_hb, g_yb (or S^ = E[h|x] for transform)
//   chain     alpha > 0 only: k sweeps x | h, y | h, h | x, y (DbmTC's builders), then crbm_chain_stats_kernel
//   dW        ONE split-K op X^T G (- X_k^T (alpha H_k) as a negated second pair when alpha > 0)
//   update    crbm_update_kernel: every variable, its momentum and its bf16 shadows
// with s[b,y,j] = sigmoid(o[b,y,j]), S_t[b,j] = s[b,t_b,j] (the positive hidden means of the joint) and
// S^[b,j] = sum_y p[b,y] s[b,y,j].
//
// Semi-supervised rows (Larochelle, Mandel, Pascanu & Bengio, JMLR 2012): with beta > 0 a row labelled -1 adds
// beta * CD-k of log p(x) instead.  Its positive phase is exact (x S^, p s, S^, p, x); its chain starts from a label y0 drawn
// from p(y|x) by the posterior kernel and h0 ~ S_{y0}; its negative phase is the last sweep of the same chain with weight beta.
// The chain runs when alpha > 0 or a row is unlabelled; a batch without an unlabelled row runs exactly the labelled-only step.
//
// Draws (Philox, make_rng(seed, site, t, tick, 0)): an unlabelled row's start label SITE_CRBM_Y0 (t = 0); h0 states SITE_H0
// (t = 0); sweep s = 1..k draws x at SITE_V, the label at SITE_CRBM_Y and h at SITE_H, all with t = s (DESIGN.md §3).
#pragma once

namespace bm {

constexpr int CRBM_MIN_CLASSES = 2, CRBM_MAX_CLASSES = 64;
constexpr int CRBM_COLS = 128;                   // columns (threads) per block of the column-tiled kernels
constexpr int CRBM_ROWS_PER_SPLIT = 64;          // batch rows per split of the column-tiled kernels' partial sums

__device__ __forceinline__ float crbm_softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float crbm_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// F[r, y] for all classes of row r = blockIdx.x (256 threads), then p = softmax(F), -log p(t|x) and whether argmax F == t
// (a tie goes to the lowest class).  Thread `tid` adds softplus(o[r,y,j]) for j = tid, tid + 256, ... in double; the 256
// partials of each class are reduced by a fixed xor tree per warp and the 8 warp sums in warp order, so F depends on H alone,
// never on how many rows a launch has.  U1 is W_1 = U^T [H, C].  CM: classes held in registers (C <= CM).
// A row labelled -1 (unlabelled) gets no NLL or correctness; instead y0[r] = the label its chain starts from, one categorical
// draw from the row's float32 p at `yrng` (word 0 of column block 0; the first y whose float64 CDF exceeds u, the CDF formed
// as dbm_multinomial_rows_kernel forms it).
template <int CM>
__global__ void __launch_bounds__(256) crbm_posterior_rows_kernel(const float* __restrict__ A, int H, const float* __restrict__ U1,
                                                                   int C, const float* __restrict__ hb, const float* __restrict__ yb,
                                                                   const int* __restrict__ labels, float* __restrict__ P,
                                                                   double* __restrict__ nll, int* __restrict__ correct,
                                                                   RngKey yrng, int* __restrict__ y0) {
    const int r = blockIdx.x, tid = threadIdx.x;
    double acc[CM];
#pragma unroll
    for (int y = 0; y < CM; ++y) acc[y] = 0.0;
    for (int j = tid; j < H; j += 256) {
        const float a = A[(size_t)r * H + j] + hb[j];
        const float* u = U1 + (size_t)j * C;
#pragma unroll
        for (int y = 0; y < CM; ++y)
            if (y < C) acc[y] += (double)crbm_softplus(a + u[y]);
    }
    __shared__ double part[8][CM];
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int y = 0; y < CM; ++y) {
        if (y >= C) break;
        double v = acc[y];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) part[warp][y] = v;
    }
    __syncthreads();
    if (tid != 0) return;
    double F[CM];
    double m = -1e300;
    int best = 0;
#pragma unroll
    for (int y = 0; y < CM; ++y) {
        if (y >= C) break;
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += part[w][y];
        F[y] = (double)yb[y] + s;
        if (F[y] > m) { m = F[y]; best = y; }
    }
    double z = 0.0;
#pragma unroll
    for (int y = 0; y < CM; ++y) { if (y >= C) break; z += exp(F[y] - m); }
    const double logz = m + log(z);
#pragma unroll
    for (int y = 0; y < CM; ++y) { if (y >= C) break; P[(size_t)r * C + y] = (float)exp(F[y] - logz); }
    if (labels) {
        const int t = labels[r];
        if (t < 0) {
            const float* pr = P + (size_t)r * C;
            double tot = 0.0, last = 0.0;
            for (int y = 0; y < C; ++y) tot += (double)pr[y];
            for (int y = 0; y < C; ++y) last += (double)(float)((double)pr[y] / tot);
            const double u = (double)u32_to_unit_float(site_block(yrng, (uint32_t)r, 0u).x);
            double run = 0.0;
            int pick = C - 1;
            for (int y = 0; y < C; ++y) {
                run += (double)(float)((double)pr[y] / tot);
                if (run / last > u) { pick = y; break; }
            }
            y0[r] = pick;
            return;
        }
        double Ft = 0.0;
#pragma unroll
        for (int y = 0; y < CM; ++y) if (y == t) Ft = F[y];
        nll[r] = logz - Ft;
        correct[r] = best == t ? 1 : 0;
    }
}

// Column pass over rows [s * rps, min(rows, (s + 1) * rps)) of split s = blockIdx.y; thread column j = blockIdx.x * 128 + tid.
// Every output is optional (nullptr: not written):
//   G  [r, j]  = bf16((1 + alpha) S_t - S^)                          the W-gradient operand (ldg)
//   h0 [r, j]  = sample ? (u < S_t) : S_t, bf16                       the chain's start (ldh; u from rng at (r, j))
//   Sh [r, j]  = S^ (fp32, [rows, H])                                  E[h|x], for transform
//   gU [s, y, j] = sum_r ((1 + alpha) [y == t_r] - p[r, y]) s[r, y, j]
//   ghb[s, j]  = sum_r G (fp32, before rounding)
//   gyb[s, y]  = sum_r ((1 + alpha) [y == t_r] - p[r, y])            (block column 0 only)
// The sums run over the split's rows in order, in fp32.  A row labelled -1 (unlabelled; y0 given) takes the semi-supervised
// terms with weight beta instead: G = bf16(beta S^), gU += beta p[r, y] s[r, y, j], gyb += beta p[r, y], and its h0 comes
// from S_{y0[r]}, the label drawn by the posterior kernel.
template <int CM>
__global__ void __launch_bounds__(CRBM_COLS) crbm_columns_kernel(const float* __restrict__ A, int H, const float* __restrict__ U1, int C,
                                                                 const float* __restrict__ hb, const float* __restrict__ P,
                                                                 const int* __restrict__ labels, int rows, int rps, float alpha,
                                                                 bf16_t* __restrict__ G, int ldg, bf16_t* __restrict__ h0, int ldh,
                                                                 int sample_h, RngKey rng, float* __restrict__ Sh,
                                                                 float* __restrict__ gU, float* __restrict__ ghb, float* __restrict__ gyb,
                                                                 const int* __restrict__ y0, float beta) {
    const int j = blockIdx.x * CRBM_COLS + threadIdx.x, s = blockIdx.y;
    const int r0 = s * rps, r1 = min(rows, r0 + rps);
    const bool col = j < H;
    const float pos = 1.0f + alpha;
    float u[CM], gu[CM];
#pragma unroll
    for (int y = 0; y < CM; ++y) { u[y] = (col && y < C) ? U1[(size_t)j * C + y] : 0.f; gu[y] = 0.f; }
    const float b = col ? hb[j] : 0.f;
    const bool ycol = gyb && blockIdx.x == 0 && (int)threadIdx.x < C;
    float hsum = 0.f, ysum = 0.f;
    for (int r = r0; r < r1; ++r) {
        const float* pr = P + (size_t)r * C;
        const int t = labels ? labels[r] : -1;
        const bool unl = y0 && t < 0;
        const int ts = unl ? y0[r] : t;                   // the label the chain starts from
        if (col) {
            const float a = A[(size_t)r * H + j] + b;
            float sh = 0.f, st = 0.f;
#pragma unroll
            for (int y = 0; y < CM; ++y) {
                if (y >= C) break;
                const float sy = crbm_sigmoid(a + u[y]);
                sh += pr[y] * sy;
                if (y == ts) st = sy;
                if (gU) gu[y] += (unl ? beta * pr[y] : (y == t ? pos : 0.f) - pr[y]) * sy;
            }
            if (Sh) Sh[(size_t)r * H + j] = sh;
            if (G) {
                const float g = unl ? beta * sh : pos * st - sh;
                G[(size_t)r * ldg + j] = __float2bfloat16_rn(g);
                hsum += g;
            }
            if (h0) {
                float h = st;
                if (sample_h) {
                    const U4 w = site_block(rng, (uint32_t)r, (uint32_t)(j >> 2));
                    const int l = j & 3;
                    h = u32_to_unit_float(l == 0 ? w.x : l == 1 ? w.y : l == 2 ? w.z : w.w) < st ? 1.f : 0.f;
                }
                h0[(size_t)r * ldh + j] = __float2bfloat16_rn(h);
            }
        }
        if (ycol) ysum += unl ? beta * pr[threadIdx.x] : ((int)threadIdx.x == t ? pos : 0.f) - pr[threadIdx.x];
    }
    if (col && gU) {
#pragma unroll
        for (int y = 0; y < CM; ++y) if (y < C) gU[((size_t)s * C + y) * H + j] = gu[y];
    }
    if (col && ghb) ghb[(size_t)s * H + j] = hsum;
    if (ycol) gyb[(size_t)s * C + threadIdx.x] = ysum;
}

// After the chain, over the rows of split s = blockIdx.y, thread column j:
//   aH [r, j]  = bf16(w_r H_k)                                        the negated second pair's operand (ldh)
//   yh [s, y, j] = sum_r Y_k[r, y] H_k[r, j]      hk[s, j] = sum_r H_k[r, j]          (j < H)
//   xd [s, j]  = sum_r X[r, j] - X_k[r, j]                                             (j < V)
//   yk [s, y]  = sum_r Y_k[r, y]                                                       (block column 0)
// The sums of pass 0 run over the labelled rows (w_r = alpha) into yh, hk, xd, yk; when yh_u is given, pass 1 runs over the
// unlabelled rows (label -1, w_r = beta) into yh_u, hk_u, xd_u, yk_u.  Without unlabelled rows pass 0 adds every row in order.
// one pass: the rows of [r0, r1) whose label is (unl ? -1 : not -1), or every row when labels is null
template <int CM>
__device__ __forceinline__ void crbm_chain_stats_pass(const bf16_t* __restrict__ Hk, int ldh, const bf16_t* __restrict__ Yk, int ldy,
                                                      int C, const bf16_t* __restrict__ X, const bf16_t* __restrict__ Xk, int ldx,
                                                      int V, int H, int r0, int r1, int s, int j, const int* __restrict__ labels,
                                                      bool unl, float w, bf16_t* __restrict__ aH, float* __restrict__ yh,
                                                      float* __restrict__ hk, float* __restrict__ xd, float* __restrict__ yk) {
    const bool hcol = j < H, xcol = j < V, ycol = blockIdx.x == 0 && (int)threadIdx.x < C;
    float acc[CM];
#pragma unroll
    for (int y = 0; y < CM; ++y) acc[y] = 0.f;
    float hs = 0.f, xs = 0.f, ys = 0.f;
    for (int r = r0; r < r1; ++r) {
        if (labels && (labels[r] < 0) != unl) continue;
        const bf16_t* yr = Yk + (size_t)r * ldy;
        if (hcol) {
            const float h = __bfloat162float(Hk[(size_t)r * ldh + j]);
            hs += h;
            aH[(size_t)r * ldh + j] = __float2bfloat16_rn(w * h);
#pragma unroll
            for (int y = 0; y < CM; ++y) { if (y >= C) break; acc[y] += __bfloat162float(yr[y]) * h; }
        }
        if (xcol) xs += __bfloat162float(X[(size_t)r * ldx + j]) - __bfloat162float(Xk[(size_t)r * ldx + j]);
        if (ycol) ys += __bfloat162float(yr[threadIdx.x]);
    }
    if (hcol) {
#pragma unroll
        for (int y = 0; y < CM; ++y) if (y < C) yh[((size_t)s * C + y) * H + j] = acc[y];
        hk[(size_t)s * H + j] = hs;
    }
    if (xcol) xd[(size_t)s * V + j] = xs;
    if (ycol) yk[(size_t)s * C + threadIdx.x] = ys;
}
template <int CM>
__global__ void __launch_bounds__(CRBM_COLS) crbm_chain_stats_kernel(const bf16_t* __restrict__ Hk, int ldh, const bf16_t* __restrict__ Yk,
                                                                     int ldy, int C, const bf16_t* __restrict__ X, const bf16_t* __restrict__ Xk,
                                                                     int ldx, int V, int H, int rows, int rps, float alpha,
                                                                     bf16_t* __restrict__ aH, float* __restrict__ yh, float* __restrict__ hk,
                                                                     float* __restrict__ xd, float* __restrict__ yk,
                                                                     const int* __restrict__ labels, float beta, float* __restrict__ yh_u,
                                                                     float* __restrict__ hk_u, float* __restrict__ xd_u, float* __restrict__ yk_u) {
    const int j = blockIdx.x * CRBM_COLS + threadIdx.x, s = blockIdx.y;
    const int r0 = s * rps, r1 = min(rows, r0 + rps);
    if (!yh_u) {            // every row labelled: one pass over all of them
        crbm_chain_stats_pass<CM>(Hk, ldh, Yk, ldy, C, X, Xk, ldx, V, H, r0, r1, s, j, nullptr, false, alpha, aH, yh, hk, xd, yk);
        return;
    }
    crbm_chain_stats_pass<CM>(Hk, ldh, Yk, ldy, C, X, Xk, ldx, V, H, r0, r1, s, j, labels, false, alpha, aH, yh, hk, xd, yk);
    crbm_chain_stats_pass<CM>(Hk, ldh, Yk, ldy, C, X, Xk, ldx, V, H, r0, r1, s, j, labels, true, beta, aH, yh_u, hk_u, xd_u, yk_u);
}

// The hybrid step's update of every variable (one thread per element of [W | U | vb | hb | yb]):
//   grad = (disc + alpha gen sums) / N  [- l2 theta for W and U];   d = lr (mom d + grad);   theta += d;  bf16 shadows refreshed.
// Sums over s1 split-K slices (W) or s2 / s3 / s4 row splits; the gen-only terms are read when s3 > 0, and the unlabelled
// rows' chain statistics (weight beta, yhu / hku / xdu / yku) when s4 > 0.
struct CrbmUpdate {
    int V, H, C, ld1, ld2;
    float *W, *dW, *U1, *dU1, *vb, *dvb, *hb, *dhb, *yb, *dyb;
    bf16_t *Wb, *U1b, *UbT;
    const float *Wp; int s1; size_t wstride;
    const float *gU, *ghb, *gyb; int s2;
    const float *yh, *hk, *xd, *yk; int s3;
    float alpha, N, l2, lr, mom;
    const float *yhu, *hku, *xdu, *yku; int s4;
    float beta;
};
__device__ __forceinline__ float crbm_split_sum(const float* p, int n, size_t stride, size_t i) {
    float b = 0.f;
    for (int s = 0; s < n; ++s) b += p[(size_t)s * stride + i];
    return b;
}
__global__ void crbm_update_kernel(CrbmUpdate u) {
    const size_t nW = (size_t)u.V * u.H, nU = (size_t)u.C * u.H;
    const size_t n = nW + nU + u.V + u.H + u.C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float g, *th, *d;
        if (i < nW) {
            float a = 0.f;
            for (int s = 0; s < u.s1; ++s) a += u.Wp[(size_t)s * u.wstride + i];
            th = u.W + i; d = u.dW + i;
            g = a / u.N - u.l2 * *th;
        } else if (i < nW + nU) {
            const size_t k = i - nW;                          // k = y * H + j
            const int y = (int)(k / u.H), j = (int)(k % u.H);
            float a = 0.f, b = 0.f;
            for (int s = 0; s < u.s2; ++s) a += u.gU[(size_t)s * nU + k];
            for (int s = 0; s < u.s3; ++s) b += u.yh[(size_t)s * nU + k];
            th = u.U1 + (size_t)j * u.C + y; d = u.dU1 + (size_t)j * u.C + y;
            float c = a - u.alpha * b;
            if (u.s4) c -= u.beta * crbm_split_sum(u.yhu, u.s4, nU, k);
            g = c / u.N - u.l2 * *th;
        } else if (i < nW + nU + u.V) {
            const int j = (int)(i - nW - nU);
            float b = 0.f;
            for (int s = 0; s < u.s3; ++s) b += u.xd[(size_t)s * u.V + j];
            th = u.vb + j; d = u.dvb + j;
            float c = u.alpha * b;
            if (u.s4) c += u.beta * crbm_split_sum(u.xdu, u.s4, u.V, j);
            g = c / u.N;
        } else if (i < nW + nU + u.V + u.H) {
            const int j = (int)(i - nW - nU - u.V);
            float a = 0.f, b = 0.f;
            for (int s = 0; s < u.s2; ++s) a += u.ghb[(size_t)s * u.H + j];
            for (int s = 0; s < u.s3; ++s) b += u.hk[(size_t)s * u.H + j];
            th = u.hb + j; d = u.dhb + j;
            float c = a - u.alpha * b;
            if (u.s4) c -= u.beta * crbm_split_sum(u.hku, u.s4, u.H, j);
            g = c / u.N;
        } else {
            const int y = (int)(i - nW - nU - u.V - u.H);
            float a = 0.f, b = 0.f;
            for (int s = 0; s < u.s2; ++s) a += u.gyb[(size_t)s * u.C + y];
            for (int s = 0; s < u.s3; ++s) b += u.yk[(size_t)s * u.C + y];
            th = u.yb + y; d = u.dyb + y;
            float c = a - u.alpha * b;
            if (u.s4) c -= u.beta * crbm_split_sum(u.yku, u.s4, u.C, y);
            g = c / u.N;
        }
        const float dd = u.lr * (u.mom * *d + g);
        *d = dd;
        const float v = *th + dd;
        *th = v;
        if (i < nW) u.Wb[(i / u.H) * u.ld1 + i % u.H] = __float2bfloat16_rn(v);
        else if (i < nW + nU) {
            const size_t k = i - nW;
            const size_t y = k / u.H, j = k % u.H;
            u.U1b[j * u.ld2 + y] = __float2bfloat16_rn(v);
            u.UbT[y * u.ld1 + j] = __float2bfloat16_rn(v);
        }
    }
}

static inline bm_dbm_cfg crbm_as_dbm(const bm_crbm_cfg& f, int32_t* Hs, int32_t* kinds, double* ns, int32_t* smp, double* spt, double* spc) {
    bm_dbm_cfg d;
    memset(&d, 0, sizeof(d));
    Hs[0] = f.n_hidden; Hs[1] = f.n_classes;
    kinds[0] = BM_UNIT_BERNOULLI; kinds[1] = BM_UNIT_MULTINOMIAL;
    ns[0] = 1.0; ns[1] = 1.0;                                   // the label: one draw of a one-of-C group
    smp[0] = f.sample_h; smp[1] = f.sample_v;                   // sample_v_states governs both visible groups
    spt[0] = spt[1] = 0.1; spc[0] = spc[1] = 0.0;
    d.n_layers = 2; d.n_visible = f.n_visible; d.n_hiddens = Hs; d.v_kind = BM_UNIT_BERNOULLI; d.h_kinds = kinds; d.h_n_samples = ns;
    d.dtype = BM_DTYPE_F32; d.compute = BM_COMPUTE_BF16;
    d.n_particles = f.max_batch; d.batch_size = f.max_batch; d.max_mf_updates = 1;
    d.sample_v = f.sample_v; d.sample_h = smp;
    d.mf_tol = 0.0; d.l2 = f.l2; d.max_norm = 1e300; d.sparsity_damping = 0.9;
    d.sparsity_target = spt; d.sparsity_cost = spc;
    return d;
}

struct CrbmShape {       // the arrays a bm_dbm_cfg points into, alive while DbmTC's constructor reads them
    int32_t Hs[2], kinds[2], smp[2];
    double ns[2], spt[2], spc[2];
};

// ---------------------------------------------------------------------------------------------
struct ClassRbmTC : DbmTC {
    int C, H;
    float alpha, beta;
    int smp_v, smp_h;
    DevBuf<float> A, P, Sh, part;
    DevBuf<double> nll;
    DevBuf<int> correct, lab, y0;
    DevBuf<bf16_t> Gb, aHb;
    // what the last hybrid_step left for debug_last_step: its rows (0: none since the last predict), chain length, whether
    // the chain ran, and the buffer holding its last sweep's h
    int last_rows = 0, last_k = 0;
    bool last_gen = false;
    const bf16_t* last_hk = nullptr;

    // refusals name the option (BM_EUNSUPPORTED); shapes and classes are BM_EINVAL
    static void check_cfg(Ctx* ctx, const bm_crbm_cfg& f) {
        BM_REQUIRE(f.n_visible > 0 && f.n_hidden > 0 && f.max_batch > 0, "bad classification RBM shape");
        BM_REQUIRE(f.n_classes >= CRBM_MIN_CLASSES && f.n_classes <= CRBM_MAX_CLASSES, "n_classes must be in [2, 64]");
        BM_REQUIRE(f.alpha >= 0.0, "alpha must be non-negative");
        BM_REQUIRE(f.beta >= 0.0 && std::isfinite(f.beta), "beta must be finite and non-negative");
        if (f.dtype != BM_DTYPE_F32) throw Error(BM_EUNSUPPORTED, "classification RBMs support float32 models only (dtype float64 requested)");
        if (f.compute != BM_COMPUTE_BF16) throw Error(BM_EUNSUPPORTED, "classification RBMs run on the tensor-core engine only (compute fp32 requested)");
        if (f.dropout_keep >= 0.0) throw Error(BM_EUNSUPPORTED, "classification RBMs do not support dropout");
        if (f.sparsity_cost != 0.0) throw Error(BM_EUNSUPPORTED, "classification RBMs do not support a sparsity cost");
        if (f.dbm_first || f.dbm_last) throw Error(BM_EUNSUPPORTED, "classification RBMs do not support dbm_first / dbm_last");
        if (ctx->nranks > 1) throw Error(BM_EUNSUPPORTED, "classification RBMs do not support a context with a communicator");
    }
    ClassRbmTC(Ctx* c, const bm_crbm_cfg& f, CrbmShape& s)
        : DbmTC(c, crbm_as_dbm(f, s.Hs, s.kinds, s.ns, s.smp, s.spt, s.spc)) {
        C = f.n_classes; H = f.n_hidden; alpha = (float)f.alpha; beta = (float)f.beta; smp_v = f.sample_v; smp_h = f.sample_h;
        A.ensure((size_t)B * H); P.ensure((size_t)B * C); Sh.ensure((size_t)B * H);
        nll.ensure(B); correct.ensure(B); lab.ensure(B); y0.ensure(B);
        Gb.ensure((size_t)B * ldn[1]); aHb.ensure((size_t)B * ldn[1]);
        for (DevBuf<bf16_t>* b : {&Gb, &aHb}) b->zero(ctx->stream);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    int splits(int rows) const { return (rows + CRBM_ROWS_PER_SPLIT - 1) / CRBM_ROWS_PER_SPLIT; }

    // ---- variables: W, U [C, H], vb, hb, yb and their momenta (U is W_1^T of the DBM underneath) --------------
    static std::string dbm_name(const std::string& n) {
        if (n == "yb") return "hb_1";
        if (n == "dyb") return "dhb_1";
        if (n == "U") return "W_1";
        if (n == "dU") return "dW_1";
        if (n == "W" || n == "vb" || n == "hb" || n == "dW" || n == "dvb" || n == "dhb") return n;
        throw Error(BM_EINVAL, "unknown variable '" + n + "'");
    }
    void set_param(const char* name, const void* host, size_t bytes) override {
        const std::string n(name);
        if (n == "U" || n == "dU") {
            BM_REQUIRE(bytes == (size_t)C * H * sizeof(float), "size mismatch for '" + n + "'");
            const float* src = static_cast<const float*>(host);
            std::vector<float> t((size_t)H * C);
            for (int y = 0; y < C; ++y) for (int j = 0; j < H; ++j) t[(size_t)j * C + y] = src[(size_t)y * H + j];
            DbmTC::set_param(dbm_name(n).c_str(), t.data(), bytes);
            return;
        }
        DbmTC::set_param(dbm_name(n).c_str(), host, bytes);
    }
    void get_param(const char* name, void* host, size_t bytes) override {
        const std::string n(name);
        if (n == "U" || n == "dU") {
            BM_REQUIRE(bytes == (size_t)C * H * sizeof(float), "size mismatch for '" + n + "'");
            std::vector<float> t((size_t)H * C);
            DbmTC::get_param(dbm_name(n).c_str(), t.data(), bytes);
            float* dst = static_cast<float*>(host);
            for (int y = 0; y < C; ++y) for (int j = 0; j < H; ++j) dst[(size_t)y * H + j] = t[(size_t)j * C + y];
            return;
        }
        DbmTC::get_param(dbm_name(n).c_str(), host, bytes);
    }
    // W <- N(0, stddev) with tf.random_normal's stream of op seed seed_w; U likewise from seed_u (drawn [C, H])
    void init_weights(double stddev, uint64_t seed_w, uint64_t seed_u) {
        launch_tf_normal_fill<float>(ctx, W[0].p, (size_t)V * H, stddev, seed_w);
        DevBuf<float> u;
        u.ensure((size_t)C * H);
        launch_tf_normal_fill<float>(ctx, u.p, (size_t)C * H, stddev, seed_u);
        std::vector<float> hu((size_t)C * H);
        BM_CUDA(cudaMemcpyAsync(hu.data(), u.p, hu.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        set_param("U", hu.data(), hu.size() * sizeof(float));      // also refreshes every bf16 shadow
    }

    // ---- posterior ------------------------------------------------------------------------------------------
    void forward(int rows) {                                   // A = X W (fp32, bias-free)
        linear_tc(Xb.p, ldn[0], rows, V, Wb[0].p, V, H, ldn[1], true, H, nullptr, A.p);
    }
    // yrng: the draw site of the chain's start label for rows labelled -1
    void posterior(int rows, const int* labels, RngKey yrng = RngKey{}) {
        if (C <= 16)
            crbm_posterior_rows_kernel<16><<<rows, 256, 0, ctx->stream>>>(A.p, H, W[1].p, C, hb[0].p, hb[1].p, labels, P.p, nll.p, correct.p,
                                                                          yrng, y0.p);
        else
            crbm_posterior_rows_kernel<64><<<rows, 256, 0, ctx->stream>>>(A.p, H, W[1].p, C, hb[0].p, hb[1].p, labels, P.p, nll.p, correct.p,
                                                                          yrng, y0.p);
        count_launch(ctx);
    }
    // semi: the batch holds rows labelled -1, whose chain starts from y0 (written by `posterior`)
    void columns(int rows, const int* labels, bf16_t* G, bf16_t* h0, RngKey rng, float* sh, float* gU, float* ghb, float* gyb,
                 bool semi = false) {
        const dim3 grid((H + CRBM_COLS - 1) / CRBM_COLS, splits(rows));
        const int* start = semi ? y0.p : nullptr;
        if (C <= 16)
            crbm_columns_kernel<16><<<grid, CRBM_COLS, 0, ctx->stream>>>(A.p, H, W[1].p, C, hb[0].p, P.p, labels, rows, CRBM_ROWS_PER_SPLIT, alpha,
                                                                         G, ldn[1], h0, ldn[1], smp_h, rng, sh, gU, ghb, gyb, start, beta);
        else
            crbm_columns_kernel<64><<<grid, CRBM_COLS, 0, ctx->stream>>>(A.p, H, W[1].p, C, hb[0].p, P.p, labels, rows, CRBM_ROWS_PER_SPLIT, alpha,
                                                                         G, ldn[1], h0, ldn[1], smp_h, rng, sh, gU, ghb, gyb, start, beta);
        count_launch(ctx);
    }
    void check_rows(int rows) const { BM_REQUIRE(rows >= 1 && rows <= B, "a batch must have 1..max_batch rows"); }

    // ---- one hybrid step --------------------------------------------------------------------------------------
    void hybrid_step(const void* Xh, const int32_t* labels, int rows, double lr, double mom, int k, uint64_t seed, uint32_t tick,
                    int want, double* out) {
        check_rows(rows);
        BM_REQUIRE(labels, "null labels");
        int unlabelled = 0;
        for (int r = 0; r < rows; ++r) {
            if (labels[r] == -1 && beta > 0.f) { ++unlabelled; continue; }
            if (labels[r] < 0 || labels[r] >= C)
                throw Error(BM_EINVAL, "label " + std::to_string(labels[r]) + " of row " + std::to_string(r) + " is outside [0, n_classes)" +
                                           (labels[r] == -1 ? " (-1 marks an unlabelled row only when beta > 0)" : ""));
        }
        const bool semi = unlabelled > 0;
        const bool gen = alpha > 0.f || semi;                    // the chain runs for the generative terms of either kind
        BM_REQUIRE(!gen || k >= 1, "n_gibbs_steps must be at least 1 when alpha > 0 or a row is unlabelled");
        BM_REQUIRE(!want || out, "metrics requested without a buffer");
        last_rows = 0;
        upload_tc(Xh, rows);
        BM_CUDA(cudaMemcpyAsync(lab.p, labels, (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        forward(rows);
        posterior(rows, lab.p, make_rng(seed, SITE_CRBM_Y0, 0, tick, 0));
        // partials: [W slices | gU | ghb | gyb] then, with the chain, [yh | hk | xd | yk] and, with unlabelled rows,
        // [yhu | hku | xdu | yku]
        const int s2 = splits(rows), s3 = gen ? s2 : 0, s4 = semi ? s2 : 0;
        const int total_pairs = ctx->sm_count / 2;
        const int pair_tiles = ((V + 255) / 256) * ((H + 255) / 256);
        const int s1 = std::max(1, std::min(total_pairs / std::max(pair_tiles, 1), (rows + 63) / 64));
        const size_t wstride = (size_t)V * H, nU = (size_t)C * H;
        const size_t per = nU + H + C, per_gen = nU + H + V + C;
        part.ensure((size_t)s1 * wstride + (size_t)s2 * per + (size_t)(s3 + s4) * per_gen);
        float* Wp = part.p;
        float* gU = Wp + (size_t)s1 * wstride;
        float* ghb = gU + (size_t)s2 * nU;
        float* gyb = ghb + (size_t)s2 * H;
        float* yh = gyb + (size_t)s2 * C;
        float* hk = yh + (size_t)s3 * nU;
        float* xd = hk + (size_t)s3 * H;
        float* yk = xd + (size_t)s3 * V;
        float* yhu = yk + (size_t)s3 * C;
        float* hku = yhu + (size_t)s4 * nU;
        float* xdu = hku + (size_t)s4 * H;
        float* yku = xdu + (size_t)s4 * V;
        columns(rows, lab.p, Gb.p, gen ? h_b[0].p : nullptr, make_rng(seed, SITE_H0, 0, tick, 0), nullptr, gU, ghb, gyb, semi);
        bf16_t* hc = h_b[0].p;
        if (gen) {
            bf16_t* hn = h2_b[0].p;
            for (int s = 1; s <= k; ++s) {                          // x | h, y | h, then h | x, y
                visible_tc(hc, v_b.p, smp_v != 0, rows, make_rng(seed, SITE_V, (uint32_t)s, tick, 0));
                hidden_tc(1, hc, nullptr, h_b[1].p, smp_v != 0, rows, 1.f, 1.f, make_rng(seed, SITE_CRBM_Y, (uint32_t)s, tick, 0));
                hidden_tc(0, v_b.p, h_b[1].p, hn, smp_h != 0 && s < k, rows, 1.f, 1.f, make_rng(seed, SITE_H, (uint32_t)s, tick, 0));
                std::swap(hc, hn);
            }
            const dim3 grid((std::max(V, H) + CRBM_COLS - 1) / CRBM_COLS, s3);
            float* const uyh = semi ? yhu : nullptr;
            if (C <= 16)
                crbm_chain_stats_kernel<16><<<grid, CRBM_COLS, 0, ctx->stream>>>(hc, ldn[1], h_b[1].p, ldn[2], C, Xb.p, v_b.p, ldn[0], V, H, rows,
                                                                                 CRBM_ROWS_PER_SPLIT, alpha, aHb.p, yh, hk, xd, yk,
                                                                                 lab.p, beta, uyh, hku, xdu, yku);
            else
                crbm_chain_stats_kernel<64><<<grid, CRBM_COLS, 0, ctx->stream>>>(hc, ldn[1], h_b[1].p, ldn[2], C, Xb.p, v_b.p, ldn[0], V, H, rows,
                                                                                 CRBM_ROWS_PER_SPLIT, alpha, aHb.p, yh, hk, xd, yk,
                                                                                 lab.p, beta, uyh, hku, xdu, yku);
            count_launch(ctx);
        }
        last_rows = rows; last_k = k; last_gen = gen; last_hk = hc;
        {   // X^T G [- X_k^T (alpha H_k)]: one split-K op over the batch rows
            TcGemm g;
            g.M = V; g.N = H;
            g.A[0] = mat(Xb.p, rows, V, ldn[0]); g.a_t[0] = true;        // stored [K = rows, M = V]
            g.B[0] = mat(Gb.p, rows, H, ldn[1]); g.b_t[0] = true;        // stored [K = rows, N = H]
            g.K[0] = rows;
            if (gen) {
                g.n_pairs = 2;
                g.A[1] = mat(v_b.p, rows, V, ldn[0]); g.a_t[1] = true;
                g.B[1] = mat(aHb.p, rows, H, ldn[1]); g.b_t[1] = true;
                g.K[1] = rows; g.neg[1] = true;
            }
            g.splits = s1; g.split_stride = wstride;
            g.out_f32 = Wp; g.ld_f32 = H;
            launch_tc_gemm(ctx, g);
        }
        if (want) {         // the pre-update posterior of this batch's labelled rows (NaN for a batch without one)
            std::vector<double> hn(rows);
            std::vector<int> hc_(rows);
            BM_CUDA(cudaMemcpyAsync(hn.data(), nll.p, (size_t)rows * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaMemcpyAsync(hc_.data(), correct.p, (size_t)rows * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
            double a = 0.0, c = 0.0;
            for (int r = 0; r < rows; ++r) if (labels[r] >= 0) { a += hn[r]; c += hc_[r]; }
            const int n = rows - unlabelled;
            out[0] = n ? a / n : std::nan(""); out[1] = n ? c / n : std::nan("");
        }
        CrbmUpdate u;
        u.V = V; u.H = H; u.C = C; u.ld1 = ldn[1]; u.ld2 = ldn[2];
        u.W = W[0].p; u.dW = dW[0].p; u.U1 = W[1].p; u.dU1 = dW[1].p; u.vb = vb.p; u.dvb = dvb.p;
        u.hb = hb[0].p; u.dhb = dhb[0].p; u.yb = hb[1].p; u.dyb = dhb[1].p;
        u.Wb = Wb[0].p; u.U1b = Wb[1].p; u.UbT = WbT[1].p;
        u.Wp = Wp; u.s1 = s1; u.wstride = wstride;
        u.gU = gU; u.ghb = ghb; u.gyb = gyb; u.s2 = s2;
        u.yh = yh; u.hk = hk; u.xd = xd; u.yk = yk; u.s3 = s3;
        u.alpha = alpha; u.N = (float)rows; u.l2 = (float)l2; u.lr = (float)lr; u.mom = (float)mom;
        u.yhu = yhu; u.hku = hku; u.xdu = xdu; u.yku = yku; u.s4 = s4; u.beta = beta;
        const size_t n = wstride + nU + V + H + C;
        crbm_update_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, 4096), 256, 0, ctx->stream>>>(u);
        count_launch(ctx);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // p(y|x) [rows, C] / E[h|x] = S^ [rows, H], in chunks of max_batch rows
    void predict(const void* Xh, int rows, float* out, bool hidden) {
        BM_REQUIRE(rows >= 1, "empty batch");
        const float* X = static_cast<const float*>(Xh);
        const int w = hidden ? H : C;
        last_rows = 0;                                         // A and P no longer hold the last step's values
        for (int r0 = 0; r0 < rows; r0 += B) {
            const int n = std::min(B, rows - r0);
            upload_tc(X + (size_t)r0 * V, n);
            forward(n);
            posterior(n, nullptr);
            if (hidden) columns(n, nullptr, nullptr, nullptr, RngKey{}, Sh.p, nullptr, nullptr, nullptr);
            BM_CUDA(cudaMemcpyAsync(out + (size_t)r0 * w, hidden ? Sh.p : P.p, (size_t)n * w * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
        }
    }

    // copies one of the last hybrid_step's buffers to the host, [rows, width] without padding: device to host only, no launch
    void debug_last_step(const std::string& n, void* host, size_t bytes) {
        BM_REQUIRE(last_rows > 0, "no training step since the engine was created or last predicted");
        const int rows = last_rows;
        auto copy = [&](const void* src, int width, size_t ld, size_t elem) {
            BM_REQUIRE(bytes == (size_t)rows * width * elem, "size mismatch for '" + n + "'");
            BM_CUDA(cudaMemcpy2DAsync(host, (size_t)width * elem, src, ld * elem, (size_t)width * elem, rows, cudaMemcpyDeviceToHost,
                                      ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
        };
        const bool chain = n == "h0" || n == "x_k" || n == "y_k" || n == "h_k" || n == "aH";
        if (chain) BM_REQUIRE(last_gen, "'" + n + "' is written only by a step whose chain ran (alpha > 0 or an unlabelled row)");
        if (n == "A") copy(A.p, H, H, sizeof(float));
        else if (n == "P") copy(P.p, C, C, sizeof(float));
        else if (n == "y0") copy(y0.p, 1, 1, sizeof(int));
        else if (n == "G") copy(Gb.p, H, ldn[1], sizeof(bf16_t));
        else if (n == "h0") {
            BM_REQUIRE(last_k == 1, "'h0' survives only a step with n_gibbs_steps = 1 (later sweeps overwrite it)");
            copy(h_b[0].p, H, ldn[1], sizeof(bf16_t));
        }
        else if (n == "x_k") copy(v_b.p, V, ldn[0], sizeof(bf16_t));
        else if (n == "y_k") copy(h_b[1].p, C, ldn[2], sizeof(bf16_t));
        else if (n == "h_k") copy(last_hk, H, ldn[1], sizeof(bf16_t));
        else if (n == "aH") copy(aHb.p, H, ldn[1], sizeof(bf16_t));
        else throw Error(BM_EINVAL, "unknown step buffer '" + n + "'");
    }
};

}  // namespace bm

using namespace bm;

extern "C" {

int bm_crbm_create(bm_ctx* hctx, const bm_crbm_cfg* cfg, bm_crbm** out) {
    BM_API_BEGIN
    Ctx* ctx = reinterpret_cast<Ctx*>(hctx);
    BM_REQUIRE(ctx && cfg && out, "null argument");
    ClassRbmTC::check_cfg(ctx, *cfg);
    BM_CUDA(cudaSetDevice(ctx->device));
    CrbmShape s;
    *out = reinterpret_cast<bm_crbm*>(new ClassRbmTC(ctx, *cfg, s));
    BM_API_END
}
void bm_crbm_destroy(bm_crbm* h) {
    if (!h) return;
    ClassRbmTC* m = reinterpret_cast<ClassRbmTC*>(h);
    cudaSetDevice(m->ctx->device);
    cudaStreamSynchronize(m->ctx->stream);
    delete m;
}
#define CRBM(h) (reinterpret_cast<ClassRbmTC*>(h))
#define CRBM_ENTER(h) BM_REQUIRE((h) != nullptr, "null crbm handle"); BM_CUDA(cudaSetDevice(CRBM(h)->ctx->device));

int bm_crbm_set_param(bm_crbm* h, const char* name, const void* host, size_t bytes) {
    BM_API_BEGIN CRBM_ENTER(h) BM_REQUIRE(name && host, "null argument"); CRBM(h)->set_param(name, host, bytes); BM_API_END
}
int bm_crbm_get_param(bm_crbm* h, const char* name, void* host, size_t bytes) {
    BM_API_BEGIN CRBM_ENTER(h) BM_REQUIRE(name && host, "null argument"); CRBM(h)->get_param(name, host, bytes); BM_API_END
}
int bm_crbm_init_weights(bm_crbm* h, double stddev, uint64_t op_seed_w, uint64_t op_seed_u) {
    BM_API_BEGIN CRBM_ENTER(h) CRBM(h)->init_weights(stddev, op_seed_w, op_seed_u); BM_API_END
}
int bm_crbm_train_step(bm_crbm* h, const void* X, const int32_t* labels, int32_t rows, double lr, double momentum, int32_t k,
                       uint64_t seed, uint32_t tick, int32_t want_metrics, double* out2) {
    BM_API_BEGIN CRBM_ENTER(h) BM_REQUIRE(X && labels, "null argument");
    CRBM(h)->hybrid_step(X, labels, rows, lr, momentum, k, seed, tick, want_metrics, out2);
    BM_API_END
}
int bm_crbm_debug_last_step(bm_crbm* h, const char* name, void* host, size_t bytes) {
    BM_API_BEGIN CRBM_ENTER(h) BM_REQUIRE(name && host, "null argument"); CRBM(h)->debug_last_step(name, host, bytes); BM_API_END
}
int bm_crbm_predict_proba(bm_crbm* h, const void* X, int32_t rows, float* out) {
    BM_API_BEGIN CRBM_ENTER(h) BM_REQUIRE(X && out, "null argument"); CRBM(h)->predict(X, rows, out, false); BM_API_END
}
int bm_crbm_transform(bm_crbm* h, const void* X, int32_t rows, float* out) {
    BM_API_BEGIN CRBM_ENTER(h) BM_REQUIRE(X && out, "null argument"); CRBM(h)->predict(X, rows, out, true); BM_API_END
}

}  // extern "C"
