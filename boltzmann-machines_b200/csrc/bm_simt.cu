// CUDA-core (FMA pipe) kernels of libbm.so: the storage-precision path (float32 / float64).
//
// Role: (1) the parity anchor -- same arithmetic type as the reference's TF-1.3 graph
// (fp32, optionally fp64; base/mixin.py:14-25), checked element-wise against the CPU oracle;
// (2) everything that is not GEMM-shaped (statistics, parameter updates, metrics, input
// preparation, multinomial sampling) for both compute modes.  The tensor-core path for the
// GEMM-shaped work lives in bm_tc.cu.
//
// Reference ops covered (paths relative to /root/reference/boltzmann_machines/):
//   layer_op        tf.matmul + multiplier + bias + activation + sampling
//                   (rbm/base_rbm.py:329-365, layers.py:47-51,84-89, dbm.py:391-425,662-684)
//   layer_op(a_trans) dW_positive / dW_negative (base_rbm.py:447-448, dbm.py:558-568)
//   colsum / bias_update / weight_update   base_rbm.py:451-474
//   prepare_input   rbm/rbm.py:101-107 (sigma division), base_rbm.py:417-418 (dropout)
//   pll_corrupt, fe_visible, rowdot, sqdiff_mean, sumsq   base_rbm.py:482-517, rbm/rbm.py:17-22,109-116
//   softmax_rows / multinomial_rows   layers.py:65-70
//   tf_normal_fill  base_rbm.py:277-279
#include "bm_internal.h"
#include <math.h>

namespace bm {

// ----------------------------------------------------------------------------------------
// math helpers
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ float  sigmoid_(float x)  { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ double sigmoid_(double x) { return 1.0 / (1.0 + exp(-x)); }
__device__ __forceinline__ float  softplus_(float x)  { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ double softplus_(double x) { return fmax(x, 0.0) + log1p(exp(-fabs(x))); }

// two float normals from two words, TF BoxMullerFloat (sin first)
__device__ __forceinline__ void box_muller_f(uint32_t x0, uint32_t x1, float& n0, float& n1) {
    float u1 = fmaxf(u32_to_unit_float(x0), 1.0e-7f);
    float v1 = 6.2831853071795864769f * u32_to_unit_float(x1);
    float u2 = sqrtf(-2.0f * logf(u1));
    n0 = sinf(v1) * u2;
    n1 = cosf(v1) * u2;
}

// ----------------------------------------------------------------------------------------
// layer_op: tiled FMA GEMM (64x64x16, 4x4 micro-tile) with the fused epilogue
// ----------------------------------------------------------------------------------------
constexpr int TM = 64, TN = 64, TK = 16;

template <typename T>
__device__ __forceinline__ void load_tiles(const T* __restrict__ A, int lda, int a_trans,
                                           const T* __restrict__ B, int ldb, int b_trans,
                                           int M, int N, int K, int m0, int n0, int k0,
                                           T (*As)[TM + 1], T (*Bs)[TN + 1], int tid) {
    if (!a_trans) {        // A[m, k]
        int m = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int gm = m0 + m, gk = k0 + kq + i;
            As[kq + i][m] = (gm < M && gk < K) ? A[(size_t)gm * lda + gk] : T(0);
        }
    } else {               // A[k, m]
        int k = tid >> 4, mq = (tid & 15) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int gm = m0 + mq + i, gk = k0 + k;
            As[k][mq + i] = (gm < M && gk < K) ? A[(size_t)gk * lda + gm] : T(0);
        }
    }
    if (!b_trans) {        // B[k, n]
        int k = tid >> 4, nq = (tid & 15) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int gn = n0 + nq + i, gk = k0 + k;
            Bs[k][nq + i] = (gn < N && gk < K) ? B[(size_t)gk * ldb + gn] : T(0);
        }
    } else {               // B[n, k]
        int n = tid >> 2, kq = (tid & 3) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int gn = n0 + n, gk = k0 + kq + i;
            Bs[kq + i][n] = (gn < N && gk < K) ? B[(size_t)gn * ldb + gk] : T(0);
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) layer_op_kernel(LayerOp<T> op) {
    __shared__ T As[TK][TM + 1];
    __shared__ T Bs[TK][TN + 1];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;

    T acc1[4][4], acc2[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc1[i][j] = T(0); acc2[i][j] = T(0); }

    for (int pair = 0; pair < 2; ++pair) {
        const T* A = pair ? op.A2 : op.A1;
        const T* B = pair ? op.B2 : op.B1;
        const int K = pair ? op.K2 : op.K1;
        const int lda = pair ? op.lda2 : op.lda1, ldb = pair ? op.ldb2 : op.ldb1;
        const int bt = pair ? op.b2_trans : op.b1_trans;
        if (K <= 0 || A == nullptr) continue;
        for (int k0 = 0; k0 < K; k0 += TK) {
            load_tiles<T>(A, lda, op.a_trans, B, ldb, bt, op.M, op.N, K, m0, n0, k0, As, Bs, tid);
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < TK; ++kk) {
                T a[4], b[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
                for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
                if (pair == 0) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) acc1[i][j] = fma(a[i], b[j], acc1[i][j]);
                } else {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) acc2[i][j] = fma(a[i], b[j], acc2[i][j]);
                }
            }
            __syncthreads();
        }
    }

    // ---- fused epilogue ---------------------------------------------------------------
    const int nb = n0 + tx * 4;                 // first of this thread's 4 aligned columns
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= op.M) continue;
        U4 w{0, 0, 0, 0};
        if (op.sample != SMP_NONE && nb < op.N) w = site_block(op.rng, (uint32_t)m, (uint32_t)(nb >> 2));
        const uint32_t words[4] = {w.x, w.y, w.z, w.w};
        float g[4] = {0.f, 0.f, 0.f, 0.f};
        if (op.sample == SMP_GAUSSIAN) {
            box_muller_f(w.x, w.y, g[0], g[1]);
            box_muller_f(w.z, w.w, g[2], g[3]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = nb + j;
            if (n >= op.N) continue;
            T c = op.s1 * acc1[i][j] + op.s2 * acc2[i][j];
            T pre = op.acc_scale * c;
            if (op.sigma) pre = pre * op.sigma[n];
            if (op.bias) pre = pre + op.bias_scale * op.bias[n];
            T mean = pre;
            if (op.act == ACT_SIGMOID) mean = sigmoid_(pre);
            else if (op.act == ACT_SOFTPLUS) mean = softplus_(pre);
            if (op.means) op.means[(size_t)m * op.ldm + n] = mean;
            if (op.states) {
                T s = mean;
                if (op.sample == SMP_BERNOULLI) {
                    // Bernoulli(probs).sample() == (u < p), layers.py:50-51
                    s = (T(u32_to_unit_float(words[j])) < mean) ? T(1) : T(0);
                } else if (op.sample == SMP_GAUSSIAN) {
                    T sd = op.noise_sigma ? op.noise_sigma[n] : T(1);
                    s = mean + sd * T(g[j]);
                }
                op.states[(size_t)m * op.lds + n] = s;
            }
        }
    }
}

template <typename T>
void launch_layer_op(Ctx* ctx, const LayerOp<T>& op) {
    if (op.M <= 0 || op.N <= 0) return;
    dim3 grid((op.N + TN - 1) / TN, (op.M + TM - 1) / TM);
    layer_op_kernel<T><<<grid, 256, 0, ctx->stream>>>(op);
    count_launch(ctx);
}
template void launch_layer_op<float>(Ctx*, const LayerOp<float>&);
template void launch_layer_op<double>(Ctx*, const LayerOp<double>&);

// ----------------------------------------------------------------------------------------
// column sums (fixed summation order -> deterministic)
// ----------------------------------------------------------------------------------------
template <typename T>
__global__ void colsum_kernel(const T* __restrict__ P, int ldp, const T* __restrict__ Q, int ldq,
                              int rows, int cols, T s1, T s2, T* __restrict__ out) {
    // block = 32 columns x 8 row-lanes; each row-lane strides over rows, then a fixed-order combine
    __shared__ double part[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    double a = 0.0;
    if (c < cols) {
        for (int r = threadIdx.y; r < rows; r += 8) {
            double v = (double)s1 * (double)P[(size_t)r * ldp + c];
            if (Q) v += (double)s2 * (double)Q[(size_t)r * ldq + c];
            a += v;
        }
    }
    part[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += part[i][threadIdx.x];
        out[c] = (T)s;
    }
}

template <typename T>
void launch_colsum(Ctx* ctx, const T* P, int ldp, const T* Q, int ldq, int rows, int cols,
                   T s1, T s2, T* out) {
    if (cols <= 0) return;
    colsum_kernel<T><<<(cols + 31) / 32, dim3(32, 8), 0, ctx->stream>>>(P, ldp, Q, ldq, rows, cols, s1, s2, out);
    count_launch(ctx);
}
template void launch_colsum<float>(Ctx*, const float*, int, const float*, int, int, int, float, float, float*);
template void launch_colsum<double>(Ctx*, const double*, int, const double*, int, int, int, double, double, double*);

// ----------------------------------------------------------------------------------------
// row reductions for the free energies
// ----------------------------------------------------------------------------------------
template <typename T>
__global__ void rowdot_kernel(const T* __restrict__ P, int ldp, const T* __restrict__ w,
                              int rows, int cols, T* __restrict__ out) {
    const int r = blockIdx.x * blockDim.y + threadIdx.y;
    if (r >= rows) return;
    double a = 0.0;
    for (int c = threadIdx.x; c < cols; c += 32) {
        double v = (double)P[(size_t)r * ldp + c];
        if (w) v *= (double)w[c];
        a += v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) out[r] = (T)a;
}
template <typename T>
void launch_rowdot(Ctx* ctx, const T* P, int ldp, const T* w, int rows, int cols, T* out) {
    if (rows <= 0) return;
    rowdot_kernel<T><<<(rows + 7) / 8, dim3(32, 8), 0, ctx->stream>>>(P, ldp, w, rows, cols, out);
    count_launch(ctx);
}
template void launch_rowdot<float>(Ctx*, const float*, int, const float*, int, int, float*);
template void launch_rowdot<double>(Ctx*, const double*, int, const double*, int, int, double*);

template <typename T>
__global__ void fe_visible_kernel(const T* __restrict__ X, int ldx, const T* __restrict__ vb,
                                  const T* __restrict__ sigma, int kind, int rows, int cols,
                                  T* __restrict__ out) {
    const int r = blockIdx.x * blockDim.y + threadIdx.y;
    if (r >= rows) return;
    double a = 0.0;
    for (int c = threadIdx.x; c < cols; c += 32) {
        T x = X[(size_t)r * ldx + c];
        if (kind == BM_UNIT_GAUSSIAN) {       // rbm/rbm.py:111-113
            T d = x - vb[c] / sigma[c];
            a += 0.5 * (double)(d * d);
        } else {                              // rbm/rbm.py:19, 54
            a -= (double)(x * vb[c]);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) out[r] = (T)a;
}
template <typename T>
void launch_fe_visible(Ctx* ctx, const T* X, int ldx, const T* vb, const T* sigma, int kind,
                       int rows, int cols, T* out) {
    if (rows <= 0) return;
    fe_visible_kernel<T><<<(rows + 7) / 8, dim3(32, 8), 0, ctx->stream>>>(X, ldx, vb, sigma, kind, rows, cols, out);
    count_launch(ctx);
}
template void launch_fe_visible<float>(Ctx*, const float*, int, const float*, const float*, int, int, int, float*);
template void launch_fe_visible<double>(Ctx*, const double*, int, const double*, const double*, int, int, int, double*);

// single-block deterministic reductions to one double
template <typename T>
__global__ void mean_combine_kernel(const T* __restrict__ a, const T* __restrict__ b, double b_sign,
                                    int n, double* __restrict__ out) {
    __shared__ double sh[1024];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        double v = (double)a[i];
        if (b) v += b_sign * (double)b[i];
        s += v;
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = sh[0] / (double)n;
}
template <typename T>
void launch_mean_combine(Ctx* ctx, const T* a, const T* b, double b_sign, int n, double* out) {
    mean_combine_kernel<T><<<1, 1024, 0, ctx->stream>>>(a, b, b_sign, n, out);
    count_launch(ctx);
}
template void launch_mean_combine<float>(Ctx*, const float*, const float*, double, int, double*);
template void launch_mean_combine<double>(Ctx*, const double*, const double*, double, int, double*);

template <typename T>
__global__ void sqdiff_partial_kernel(const T* __restrict__ P, int ldp, const T* __restrict__ Q, int ldq,
                                      int rows, int cols, double* __restrict__ partial) {
    __shared__ double sh[256];
    double s = 0.0;
    const size_t total = (size_t)rows * cols;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        double d = (double)P[(size_t)r * ldp + c];
        if (Q) d -= (double)Q[(size_t)r * ldq + c];
        s += d * d;
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}
__global__ void finish_sum_kernel(const double* __restrict__ partial, int n, double denom, double* __restrict__ out) {
    __shared__ double sh[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s += partial[i];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = sh[0] / denom;
}
static double* g_partials(Ctx* ctx) {
    // per context: the partial sums are written and read on ctx->stream, and two contexts on one device run their
    // reductions on two streams that are not ordered against each other
    if (!ctx->reduce_scratch) BM_CUDA(cudaMalloc(&ctx->reduce_scratch, 1024 * sizeof(double)));
    return ctx->reduce_scratch;
}
template <typename T>
void launch_sqdiff_mean(Ctx* ctx, const T* P, int ldp, const T* Q, int ldq, int rows, int cols,
                        double denom, double* out) {
    double* part = g_partials(ctx);
    const int blocks = 592;
    sqdiff_partial_kernel<T><<<blocks, 256, 0, ctx->stream>>>(P, ldp, Q, ldq, rows, cols, part);
    count_launch(ctx);
    finish_sum_kernel<<<1, 256, 0, ctx->stream>>>(part, blocks, denom, out);
    count_launch(ctx);
}
template void launch_sqdiff_mean<float>(Ctx*, const float*, int, const float*, int, int, int, double, double*);
template void launch_sqdiff_mean<double>(Ctx*, const double*, int, const double*, int, int, int, double, double*);

template <typename T>
void launch_sumsq(Ctx* ctx, const T* W, size_t n, double* out) {
    // sum of squares of a dense array = sqdiff with Q = null on a [1, n] view split into rows
    const int cols = 1024;
    const int rows = (int)(n / cols);
    double* part = g_partials(ctx);
    const int blocks = 592;
    if (rows > 0) {
        sqdiff_partial_kernel<T><<<blocks, 256, 0, ctx->stream>>>(W, cols, nullptr, 0, rows, cols, part);
    } else {
        BM_CUDA(cudaMemsetAsync(part, 0, blocks * sizeof(double), ctx->stream));
    }
    count_launch(ctx);
    const int tail = (int)(n - (size_t)rows * cols);
    if (tail > 0) {
        sqdiff_partial_kernel<T><<<1, 256, 0, ctx->stream>>>(W + (size_t)rows * cols, tail, nullptr, 0, 1, tail, part + blocks);
        count_launch(ctx);
    }
    finish_sum_kernel<<<1, 256, 0, ctx->stream>>>(part, blocks + (tail > 0 ? 1 : 0), 1.0, out);
    count_launch(ctx);
}
template void launch_sumsq<float>(Ctx*, const float*, size_t, double*);
template void launch_sumsq<double>(Ctx*, const double*, size_t, double*);

// ----------------------------------------------------------------------------------------
// input preparation and PLL corruption
// ----------------------------------------------------------------------------------------
template <typename T>
__global__ void prepare_input_kernel(const T* __restrict__ X, int ldx, T* __restrict__ Xp, int ldxp,
                                     int rows, int cols, const T* __restrict__ sigma, T keep,
                                     int do_dropout, RngKey rng) {
    const int cb = blockIdx.x * blockDim.x + threadIdx.x;       // column block of 4
    const int r = blockIdx.y;
    if (cb * 4 >= cols || r >= rows) return;
    U4 w{0, 0, 0, 0};
    if (do_dropout) w = site_block(rng, (uint32_t)r, (uint32_t)cb);
    const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int c = cb * 4 + j;
        if (c >= cols) break;
        T x = X[(size_t)r * ldx + c];
        if (sigma) x = x / sigma[c];
        if (do_dropout) {
            // tf.nn.dropout: x / keep * floor(keep + u)
            float m = floorf((float)keep + u32_to_unit_float(words[j]));
            x = x / keep * T(m);
        }
        Xp[(size_t)r * ldxp + c] = x;
    }
}
template <typename T>
void launch_prepare_input(Ctx* ctx, const T* X, int ldx, T* Xp, int ldxp, int rows, int cols,
                          const T* sigma, double keep, RngKey rng) {
    const int cbs = (cols + 3) / 4;
    for (int r0 = 0; r0 < rows; r0 += 32768) {            // grid.y (the row) is limited to 65535: tall batches go in slabs
        const int n = rows - r0 < 32768 ? rows - r0 : 32768;
        RngKey slab = rng;
        slab.row0 += (uint32_t)r0;                         // the draw of a row depends on its index in the batch, not in the slab
        dim3 grid((cbs + 127) / 128, n);
        prepare_input_kernel<T><<<grid, 128, 0, ctx->stream>>>(X + (size_t)r0 * ldx, ldx, Xp + (size_t)r0 * ldxp, ldxp, n, cols, sigma,
                                                               (T)(keep < 0 ? 1.0 : keep), keep >= 0 ? 1 : 0, slab);
        count_launch(ctx);
    }
}
template void launch_prepare_input<float>(Ctx*, const float*, int, float*, int, int, int, const float*, double, RngKey);
template void launch_prepare_input<double>(Ctx*, const double*, int, double*, int, int, int, const double*, double, RngKey);

template <typename T>
__global__ void pll_corrupt_kernel(const T* __restrict__ X, int ldx, T* __restrict__ Xc, int ldxc,
                                   int rows, int cols, RngKey rng) {
    const int r = blockIdx.x;
    if (r >= rows) return;
    const uint32_t idx = site_block(rng, (uint32_t)r, 0).x % (uint32_t)cols;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) {
        T x = X[(size_t)r * ldx + c];
        Xc[(size_t)r * ldxc + c] = ((uint32_t)c == idx) ? T(1) - x : x;
    }
}
template <typename T>
void launch_pll_corrupt(Ctx* ctx, const T* X, int ldx, T* Xc, int ldxc, int rows, int cols, RngKey rng) {
    if (rows <= 0) return;
    pll_corrupt_kernel<T><<<rows, 128, 0, ctx->stream>>>(X, ldx, Xc, ldxc, rows, cols, rng);
    count_launch(ctx);
}
template void launch_pll_corrupt<float>(Ctx*, const float*, int, float*, int, int, int, RngKey);
template void launch_pll_corrupt<double>(Ctx*, const double*, int, double*, int, int, int, RngKey);

// ----------------------------------------------------------------------------------------
// parameter updates
// ----------------------------------------------------------------------------------------
template <typename T>
__global__ void bias_update_kernel(BiasUpdate<T> u) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < u.H) {
        // base_rbm.py:457-461
        T q = u.damp * u.q_means[i] + (T(1) - u.damp) * u.qsum[i];
        u.q_means[i] = q;
        T pen = u.cost * (q - u.target);
        u.pen[i] = pen;
        T g = u.dhb_raw[i] / u.n_div - pen;   // :453
        T d = u.lr * (u.mom * u.dhb[i] + g);     // :473-474
        u.dhb[i] = d;
        u.hb[i] += d;
    }
    if (i < u.V) {
        T d = u.lr * (u.mom * u.dvb[i] + u.dvb_raw[i] / u.n_div);   // :451, :470-471
        u.dvb[i] = d;
        u.vb[i] += d;
    }
}
template <typename T>
void launch_bias_update(Ctx* ctx, const BiasUpdate<T>& u) {
    const int n = u.V > u.H ? u.V : u.H;
    bias_update_kernel<T><<<(n + 255) / 256, 256, 0, ctx->stream>>>(u);
    count_launch(ctx);
}
template void launch_bias_update<float>(Ctx*, const BiasUpdate<float>&);
template void launch_bias_update<double>(Ctx*, const BiasUpdate<double>&);

template <typename T>
__global__ void weight_update_kernel(const T* __restrict__ G, int ldg, T g_div, T* __restrict__ W, T* __restrict__ dW,
                                     int V, int H, const T* __restrict__ pen, T l2, T lr, T mom,
                                     __nv_bfloat16* __restrict__ Wb, int ldwb) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    const int v = blockIdx.y;
    if (h >= H || v >= V) return;
    const size_t i = (size_t)v * H + h;
    const T w = W[i];
    T g = G[(size_t)v * ldg + h] / g_div - l2 * w;      // base_rbm.py:449
    g = g - pen[h];                             // :462
    const T d = lr * (mom * dW[i] + g);         // :467
    dW[i] = d;
    const T wn = w + d;                         // :468
    W[i] = wn;
    if (Wb) Wb[(size_t)v * ldwb + h] = __float2bfloat16_rn((float)wn);
}
template <typename T>
void launch_weight_update(Ctx* ctx, const T* G, int ldg, T g_div, T* W, T* dW, int V, int H,
                          const T* pen, T l2, T lr, T mom, __nv_bfloat16* Wb, int ldwb) {
    // (the visible index travels in grid.y, limit 65535: models with more input units go in slabs of rows)
    for (int r0 = 0; r0 < V; r0 += 32768) {
        const int n = V - r0 < 32768 ? V - r0 : 32768;
        dim3 grid((H + 255) / 256, n);
        weight_update_kernel<T><<<grid, 256, 0, ctx->stream>>>(G + (size_t)r0 * ldg, ldg, g_div, W + (size_t)r0 * H, dW + (size_t)r0 * H, n, H,
                                                               pen, l2, lr, mom, Wb ? Wb + (size_t)r0 * ldwb : nullptr, ldwb);
        count_launch(ctx);
    }
}
template void launch_weight_update<float>(Ctx*, const float*, int, float, float*, float*, int, int, const float*, float, float, float, __nv_bfloat16*, int);
template void launch_weight_update<double>(Ctx*, const double*, int, double, double*, double*, int, int, const double*, double, double, double, __nv_bfloat16*, int);

// ----------------------------------------------------------------------------------------
// multinomial units (layers.py:54-70)
// ----------------------------------------------------------------------------------------
template <typename T>
__global__ void softmax_rows_kernel(T* __restrict__ X, int ldx, int rows, int cols, T scale) {
    // one block per row; numerically as the oracle: subtract the row max, exp, normalise
    __shared__ double sh[256];
    const int r = blockIdx.x;
    T* x = X + (size_t)r * ldx;
    double mx = -1e300;
    for (int c = threadIdx.x; c < cols; c += 256) mx = fmax(mx, (double)x[c]);
    sh[threadIdx.x] = mx;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + o]);
        __syncthreads();
    }
    const T m = (T)sh[0];
    __syncthreads();
    double s = 0.0;
    for (int c = threadIdx.x; c < cols; c += 256) {
        T e = (T)exp((double)(x[c] - m));
        if (sizeof(T) == 4) e = (T)expf((float)(x[c] - m));
        x[c] = e;
        s += (double)e;
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    const T tot = (T)sh[0];
    for (int c = threadIdx.x; c < cols; c += 256) x[c] = scale * x[c] / tot;
}
template <typename T>
void launch_softmax_rows(Ctx* ctx, T* X, int ldx, int rows, int cols, T scale) {
    if (rows <= 0) return;
    softmax_rows_kernel<T><<<rows, 256, 0, ctx->stream>>>(X, ldx, rows, cols, scale);
    count_launch(ctx);
}
template void launch_softmax_rows<float>(Ctx*, float*, int, int, int, float);
template void launch_softmax_rows<double>(Ctx*, double*, int, int, int, double);

template <typename T>
__global__ void multinomial_rows_kernel(const T* __restrict__ means, int ldm, int rows, int cols,
                                        int n_draws, T* __restrict__ counts, int ldc, RngKey rng) {
    // one block per row.  CDF in double, accumulated sequentially like np.cumsum, of the float32
    // probabilities p = means / sum(means); draw d takes the first j with cdf[j] > u_d.
    extern __shared__ unsigned char smem_raw[];
    double* cdf = reinterpret_cast<double*>(smem_raw);
    int* cnt = reinterpret_cast<int*>(cdf + cols);
    __shared__ double tot_sh;
    const int r = blockIdx.x;
    const T* mrow = means + (size_t)r * ldm;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) cnt[c] = 0;
    if (threadIdx.x == 0) {
        // row sum in the storage type, in index order (numpy pairwise differs by rounding only;
        // the probabilities are then rounded to float32 exactly as the oracle does)
        double tot = 0.0;
        for (int c = 0; c < cols; ++c) tot += (double)mrow[c];
        tot_sh = tot;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double run = 0.0;
        for (int c = 0; c < cols; ++c) {
            float p = (float)((double)mrow[c] / tot_sh);
            run += (double)p;
            cdf[c] = run;
        }
        const double last = cdf[cols - 1];
        for (int c = 0; c < cols; ++c) cdf[c] = cdf[c] / last;
    }
    __syncthreads();
    for (int d = threadIdx.x; d < n_draws; d += blockDim.x) {
        U4 w = site_block(rng, (uint32_t)r, (uint32_t)(d >> 2));
        const uint32_t words[4] = {w.x, w.y, w.z, w.w};
        const double u = (double)u32_to_unit_float(words[d & 3]);
        int lo = 0, hi = cols;            // first index with cdf > u
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            if (cdf[mid] > u) hi = mid; else lo = mid + 1;
        }
        if (lo > cols - 1) lo = cols - 1;
        atomicAdd(&cnt[lo], 1);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < cols; c += blockDim.x) counts[(size_t)r * ldc + c] = (T)cnt[c];
}
template <typename T>
void launch_multinomial_rows(Ctx* ctx, const T* means, int ldm, int rows, int cols, int n_draws,
                             T* counts, int ldc, RngKey rng) {
    if (rows <= 0) return;
    const size_t smem = (size_t)cols * (sizeof(double) + sizeof(int));
    if (smem > 48 * 1024)
        BM_CUDA(cudaFuncSetAttribute(multinomial_rows_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    multinomial_rows_kernel<T><<<rows, 128, smem, ctx->stream>>>(means, ldm, rows, cols, n_draws, counts, ldc, rng);
    count_launch(ctx);
}
template void launch_multinomial_rows<float>(Ctx*, const float*, int, int, int, int, float*, int, RngKey);
template void launch_multinomial_rows<double>(Ctx*, const double*, int, int, int, int, double*, int, RngKey);

// ----------------------------------------------------------------------------------------
// weight initialiser with tf.random_normal's stream
// ----------------------------------------------------------------------------------------
__global__ void tf_normal_fill_f32(float* __restrict__ W, size_t n, float stddev, uint32_t k0, uint32_t k1,
                                   uint32_t s2lo, uint32_t s2hi) {
    const size_t blk = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (blk * 4 >= n) return;
    U4 w = philox4x32_10((uint32_t)blk, (uint32_t)(blk >> 32), s2lo, s2hi, k0, k1);
    float g[4];
    box_muller_f(w.x, w.y, g[0], g[1]);
    box_muller_f(w.z, w.w, g[2], g[3]);
    for (int j = 0; j < 4 && blk * 4 + j < n; ++j) W[blk * 4 + j] = g[j] * stddev;
}
__global__ void tf_normal_fill_f64(double* __restrict__ W, size_t n, double stddev, uint32_t k0, uint32_t k1,
                                   uint32_t s2lo, uint32_t s2hi) {
    const size_t blk = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (blk * 2 >= n) return;
    U4 w = philox4x32_10((uint32_t)blk, (uint32_t)(blk >> 32), s2lo, s2hi, k0, k1);
    double u1 = fmax(u64_to_unit_double(w.x, w.y), 1.0e-7);
    double v1 = 6.283185307179586476925286766559 * u64_to_unit_double(w.z, w.w);
    double u2 = sqrt(-2.0 * log(u1));
    double g0 = sin(v1) * u2, g1 = cos(v1) * u2;
    W[blk * 2] = g0 * stddev;
    if (blk * 2 + 1 < n) W[blk * 2 + 1] = g1 * stddev;
}
template <>
void launch_tf_normal_fill<float>(Ctx* ctx, float* W, size_t n, double stddev, uint64_t op_seed) {
    const size_t nb = (n + 3) / 4;
    // tf.get_seed(op_seed) with no graph-level seed: (87654321, op_seed)
    tf_normal_fill_f32<<<(unsigned)((nb + 255) / 256), 256, 0, ctx->stream>>>(
        W, n, (float)stddev, 87654321u, 0u, (uint32_t)op_seed, (uint32_t)(op_seed >> 32));
    count_launch(ctx);
}
template <>
void launch_tf_normal_fill<double>(Ctx* ctx, double* W, size_t n, double stddev, uint64_t op_seed) {
    const size_t nb = (n + 1) / 2;
    tf_normal_fill_f64<<<(unsigned)((nb + 255) / 256), 256, 0, ctx->stream>>>(
        W, n, stddev, 87654321u, 0u, (uint32_t)op_seed, (uint32_t)(op_seed >> 32));
    count_launch(ctx);
}

template <typename T>
__global__ void fill_kernel(T* p, size_t n, T v) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
template <typename T>
void launch_fill(Ctx* ctx, T* p, size_t n, T v) {
    if (!n) return;
    fill_kernel<T><<<(unsigned)((n + 255) / 256 > 1184 ? 1184 : (n + 255) / 256), 256, 0, ctx->stream>>>(p, n, v);
    count_launch(ctx);
}
template void launch_fill<float>(Ctx*, float*, size_t, float);
template void launch_fill<double>(Ctx*, double*, size_t, double);

}  // namespace bm
