// Small CUDA-core kernels that operate on the bf16 activations of the tensor-core path:
// conversions, the three column statistics of a CD step (base_rbm.py:451-457) and the split-K
// reduction of the dW partials.
#include "bm_tc.h"

namespace bm {

// ------------------------------------------------------------------------------------------
// small helpers on bf16 activations
// ------------------------------------------------------------------------------------------
__global__ void f32_to_bf16_kernel(const float* __restrict__ src, int lds, __nv_bfloat16* __restrict__ dst, int ldd, int rows, int cols) {
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
    const int r = blockIdx.y;
    if (c >= cols) return;
    const float a = src[(size_t)r * lds + c];
    // (columns >= cols of the destination are never written: batch buffers keep constant columns there)
    if (c + 1 < cols)
        *reinterpret_cast<__nv_bfloat162*>(dst + (size_t)r * ldd + c) = __floats2bfloat162_rn(a, src[(size_t)r * lds + c + 1]);
    else
        dst[(size_t)r * ldd + c] = __float2bfloat16_rn(a);
}
// grid.y carries the row index and is limited to 65535: taller matrices (a resident dataset) go in slabs
constexpr int ROW_SLAB = 32768;
void launch_f32_to_bf16(Ctx* ctx, const float* src, int lds, __nv_bfloat16* dst, int ldd, int rows, int cols) {
    for (int r0 = 0; r0 < rows; r0 += ROW_SLAB) {
        const int n = rows - r0 < ROW_SLAB ? rows - r0 : ROW_SLAB;
        dim3 grid(((cols + 1) / 2 + 127) / 128, n);
        f32_to_bf16_kernel<<<grid, 128, 0, ctx->stream>>>(src + (size_t)r0 * lds, lds, dst + (size_t)r0 * ldd, ldd, n, cols);
        count_launch(ctx);
    }
}

__global__ void bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ src, int lds, float* __restrict__ dst, int ldd, int rows, int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    if (c < cols) dst[(size_t)r * ldd + c] = __bfloat162float(src[(size_t)r * lds + c]);
}
void launch_bf16_to_f32(Ctx* ctx, const __nv_bfloat16* src, int lds, float* dst, int ldd, int rows, int cols) {
    for (int r0 = 0; r0 < rows; r0 += ROW_SLAB) {
        const int n = rows - r0 < ROW_SLAB ? rows - r0 : ROW_SLAB;
        dim3 grid((cols + 255) / 256, n);
        bf16_to_f32_kernel<<<grid, 256, 0, ctx->stream>>>(src + (size_t)r0 * lds, lds, dst + (size_t)r0 * ldd, ldd, n, cols);
        count_launch(ctx);
    }
}

// ---- byte-valued host datasets (bm_rbm_train_epoch_u8): u8 -> bf16 / fp32 / fp64, exact for 0..255 ----
__global__ void u8_to_bf16_kernel(const uint8_t* __restrict__ src, int lds, __nv_bfloat16* __restrict__ dst, int ldd, int rows, int cols) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;            // group of 8 columns
    const int r = blockIdx.y;
    const int c = g * 8;
    if (c >= cols) return;
    const uint8_t* s = src + (size_t)r * lds + c;
    __nv_bfloat16* d = dst + (size_t)r * ldd + c;
    if (c + 8 <= cols && ((lds & 7) == 0)) {                          // 8-byte aligned source group, 16-byte aligned destination
        const uint2 b = *reinterpret_cast<const uint2*>(s);
        const uint32_t w[2] = {b.x, b.y};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t word = w[i >> 1] >> ((i & 1) * 16);
            __nv_bfloat162 h2 = __floats2bfloat162_rn((float)(word & 0xFFu), (float)((word >> 8) & 0xFFu));
            o[i] = *reinterpret_cast<uint32_t*>(&h2);
        }
        *reinterpret_cast<uint4*>(d) = make_uint4(o[0], o[1], o[2], o[3]);
    } else {
        for (int e = 0; e < 8 && c + e < cols; ++e) d[e] = __float2bfloat16_rn((float)s[e]);
    }
}
void launch_u8_to_bf16(Ctx* ctx, const uint8_t* src, int lds, __nv_bfloat16* dst, int ldd, int rows, int cols, cudaStream_t stream) {
    if (!stream) stream = ctx->stream;
    for (int r0 = 0; r0 < rows; r0 += ROW_SLAB) {
        const int n = rows - r0 < ROW_SLAB ? rows - r0 : ROW_SLAB;
        dim3 grid(((cols + 7) / 8 + 127) / 128, n);
        u8_to_bf16_kernel<<<grid, 128, 0, stream>>>(src + (size_t)r0 * lds, lds, dst + (size_t)r0 * ldd, ldd, n, cols);
        count_launch(ctx);
    }
}
template <typename T>
__global__ void u8_to_real_kernel(const uint8_t* __restrict__ src, T* __restrict__ dst, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = (T)src[i];
}
template <typename T>
void launch_u8_to_real(Ctx* ctx, const uint8_t* src, T* dst, size_t n) {
    if (!n) return;
    const size_t blocks = (n + 255) / 256;
    u8_to_real_kernel<T><<<(unsigned)(blocks < 1184 ? blocks : 1184), 256, 0, ctx->stream>>>(src, dst, n);
    count_launch(ctx);
}
template void launch_u8_to_real<float>(Ctx*, const uint8_t*, float*, size_t);
template void launch_u8_to_real<double>(Ctx*, const uint8_t*, double*, size_t);

// ---- MSRE on the bf16 activations (base_rbm.py:486-488): mean((X - v_means)^2), accumulated in fp64 ----
constexpr int SQ_BLOCKS = 592;
// one launch: every block leaves its partial sum, the block that arrives last adds them up in a fixed order (thread t takes
// partials t, t+256, ...; then the block's shared-memory tree), so the value does not depend on which block that is
__global__ void sqdiff_bf16_kernel(const __nv_bfloat16* __restrict__ P, int ldp, const __nv_bfloat16* __restrict__ Q, int ldq,
                                   int rows, int cols, double* __restrict__ partial, unsigned int* __restrict__ arrived,
                                   double denom, double* __restrict__ out) {
    __shared__ double sh[256];
    __shared__ bool last;
    double s = 0.0;
    const int gpr = (cols + 7) / 8;                                   // 8-column groups per row
    const size_t total = (size_t)rows * gpr;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / gpr), c = (int)(i % gpr) * 8;
        const __nv_bfloat16* p = P + (size_t)r * ldp + c;
        const __nv_bfloat16* q = Q + (size_t)r * ldq + c;
        float acc = 0.f;
        if (c + 8 <= cols) {                                          // leading dimensions are multiples of 8
            const uint4 a = *reinterpret_cast<const uint4*>(p), b = *reinterpret_cast<const uint4*>(q);
            const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&a);
            const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&b);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 fa = __bfloat1622float2(ha[k]), fb = __bfloat1622float2(hb[k]);
                const float d0 = fa.x - fb.x, d1 = fa.y - fb.y;
                acc = fmaf(d0, d0, acc); acc = fmaf(d1, d1, acc);
            }
        } else {
            for (int e = 0; c + e < cols; ++e) { const float d = __bfloat162float(p[e]) - __bfloat162float(q[e]); acc = fmaf(d, d, acc); }
        }
        s += (double)acc;
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = sh[0];
        __threadfence();                                              // the partial is visible before the arrival is
        last = atomicAdd(arrived, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    s = 0.0;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += 256) s += __ldcg(partial + i);
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) { *out = sh[0] / denom; *arrived = 0u; }   // (next launch on this stream starts from zero)
}
void launch_sqdiff_mean_bf16(Ctx* ctx, const __nv_bfloat16* P, int ldp, const __nv_bfloat16* Q, int ldq, int rows, int cols,
                             double denom, double* out) {
    if (!ctx->sqdiff_scratch) {
        BM_CUDA(cudaMalloc(&ctx->sqdiff_scratch, (SQ_BLOCKS + 1) * sizeof(double)));
        BM_CUDA(cudaMemsetAsync(ctx->sqdiff_scratch, 0, (SQ_BLOCKS + 1) * sizeof(double), ctx->stream));
    }
    sqdiff_bf16_kernel<<<SQ_BLOCKS, 256, 0, ctx->stream>>>(P, ldp, Q, ldq, rows, cols, ctx->sqdiff_scratch,
                                                          reinterpret_cast<unsigned int*>(ctx->sqdiff_scratch + SQ_BLOCKS), denom, out);
    count_launch(ctx);
}

// ---- column statistics of bf16 activations: up to 3 jobs (dvb, dhb, q) in one pair of launches ----
struct ColsumJobs {
    const __nv_bfloat16* P[3]; int ldp[3];
    const __nv_bfloat16* Q[3]; int ldq[3];
    float s1[3], s2[3];
    float* out[3];
    int cols[3];
    int rows, n;
};
constexpr int CS_RSPLIT = 64;

__device__ __forceinline__ void acc8(float (&a)[8], const uint4& p, float s) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&p);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); a[2 * i] = fmaf(s, f.x, a[2 * i]); a[2 * i + 1] = fmaf(s, f.y, a[2 * i + 1]); }
}
__global__ void colsum_bf16_partial_kernel(ColsumJobs j, float* __restrict__ partial, int max_cols) {
    // block: 32 x 8 threads; 256 columns (8 per thread, one 16-byte load per row) x one row slab;
    // fixed combine order (deterministic)
    __shared__ float part[8][32][9];
    const int job = blockIdx.z;
    const int cols = j.cols[job];
    const int c = (blockIdx.x * 32 + threadIdx.x) * 8;
    const int slab = (j.rows + CS_RSPLIT - 1) / CS_RSPLIT;
    const int r0 = blockIdx.y * slab, r1 = min(j.rows, r0 + slab);
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c < cols) {
        const __nv_bfloat16* P = j.P[job]; const __nv_bfloat16* Q = j.Q[job];
        const float s1 = j.s1[job], s2 = j.s2[job];
        if (c + 8 <= cols) {                       // leading dimensions are multiples of 8: 16-byte aligned
            for (int r = r0 + threadIdx.y; r < r1; r += 8) {
                const uint4 p = *reinterpret_cast<const uint4*>(P + (size_t)r * j.ldp[job] + c);
                acc8(a, p, s1);
                if (Q) { const uint4 q = *reinterpret_cast<const uint4*>(Q + (size_t)r * j.ldq[job] + c); acc8(a, q, s2); }
            }
        } else {
            for (int r = r0 + threadIdx.y; r < r1; r += 8)
                for (int e = 0; e < cols - c; ++e) {
                    a[e] = fmaf(s1, __bfloat162float(P[(size_t)r * j.ldp[job] + c + e]), a[e]);
                    if (Q) a[e] = fmaf(s2, __bfloat162float(Q[(size_t)r * j.ldq[job] + c + e]), a[e]);
                }
        }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) part[threadIdx.y][threadIdx.x][e] = a[e];
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        float* dst = partial + ((size_t)job * CS_RSPLIT + blockIdx.y) * max_cols + c;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) s += part[i][threadIdx.x][e];
            if (c + e < cols) dst[e] = s;
        }
    }
}
__global__ void colsum_bf16_finish_kernel(ColsumJobs j, const float* __restrict__ partial, int max_cols) {
    const int job = blockIdx.y;
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= j.cols[job]) return;
    float s = 0.f;
#pragma unroll 8
    for (int i = 0; i < CS_RSPLIT; ++i) s += partial[((size_t)job * CS_RSPLIT + i) * max_cols + c];
    j.out[job][c] = s;
}
static float* colsum_scratch(Ctx* ctx, size_t floats) {
    if (ctx->colsum_scratch_floats < floats) {
        if (ctx->colsum_scratch) { BM_CUDA(cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->colsum_scratch); ctx->colsum_scratch = nullptr; }
        BM_CUDA(cudaMalloc(&ctx->colsum_scratch, floats * sizeof(float)));
        ctx->colsum_scratch_floats = floats;
    }
    return ctx->colsum_scratch;
}
static void run_colsum_jobs(Ctx* ctx, const ColsumJobs& j) {
    int max_cols = 0;
    for (int i = 0; i < j.n; ++i) max_cols = j.cols[i] > max_cols ? j.cols[i] : max_cols;
    if (max_cols <= 0 || j.rows <= 0) return;
    max_cols = (max_cols + 7) & ~7;
    float* scratch = colsum_scratch(ctx, (size_t)3 * CS_RSPLIT * max_cols);
    colsum_bf16_partial_kernel<<<dim3((max_cols + 255) / 256, CS_RSPLIT, j.n), dim3(32, 8), 0, ctx->stream>>>(j, scratch, max_cols);
    count_launch(ctx);
    colsum_bf16_finish_kernel<<<dim3((max_cols + 255) / 256, j.n), 256, 0, ctx->stream>>>(j, scratch, max_cols);
    count_launch(ctx);
}
void launch_colsum_bf16(Ctx* ctx, const __nv_bfloat16* P, int ldp, const __nv_bfloat16* Q, int ldq,
                        int rows, int cols, float s1, float s2, float* out) {
    ColsumJobs j{};
    j.P[0] = P; j.ldp[0] = ldp; j.Q[0] = Q; j.ldq[0] = ldq; j.s1[0] = s1; j.s2[0] = s2; j.out[0] = out; j.cols[0] = cols;
    j.rows = rows; j.n = 1;
    run_colsum_jobs(ctx, j);
}
// up to 3 plain column sums over the same number of rows in one pair of launches
void launch_colsums_bf16(Ctx* ctx, int n, const __nv_bfloat16* const* P, const int* ldp, const int* cols, float* const* out, int rows) {
    BM_REQUIRE(n >= 1 && n <= 3, "1..3 column sums per call");
    ColsumJobs j{};
    for (int i = 0; i < n; ++i) { j.P[i] = P[i]; j.ldp[i] = ldp[i]; j.Q[i] = nullptr; j.ldq[i] = 0; j.s1[i] = 1.f; j.s2[i] = 0.f; j.out[i] = out[i]; j.cols[i] = cols[i]; }
    j.rows = rows; j.n = n;
    run_colsum_jobs(ctx, j);
}
void launch_cd_statistics_bf16(Ctx* ctx, const __nv_bfloat16* X, int ldx, const __nv_bfloat16* v, int ldv,
                               const __nv_bfloat16* h0, const __nv_bfloat16* hk, int ldh, int rows, int V, int H,
                               float* dvb_sum, float* dhb_sum, float* q_sum) {
    ColsumJobs j{};
    j.P[0] = X;  j.ldp[0] = ldx; j.Q[0] = v;  j.ldq[0] = ldv; j.s1[0] = 1.f; j.s2[0] = -1.f; j.out[0] = dvb_sum; j.cols[0] = V;   // base_rbm.py:451
    j.P[1] = h0; j.ldp[1] = ldh; j.Q[1] = hk; j.ldq[1] = ldh; j.s1[1] = 1.f; j.s2[1] = -1.f; j.out[1] = dhb_sum; j.cols[1] = H;   // :453
    j.P[2] = hk; j.ldp[2] = ldh; j.Q[2] = nullptr; j.ldq[2] = 0; j.s1[2] = 1.f; j.s2[2] = 0.f; j.out[2] = q_sum; j.cols[2] = H;   // :457
    j.rows = rows; j.n = 3;
    run_colsum_jobs(ctx, j);
}

__global__ void reduce_partials_kernel(const float* __restrict__ partial, size_t stride, int splits, float* __restrict__ G, size_t n) {
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    // 16-byte loads need every slice and G on a 16-byte boundary (callers pad the stride; checked here all the same)
    const bool vec = (stride & 3) == 0 && ((reinterpret_cast<uintptr_t>(partial) | reinterpret_cast<uintptr_t>(G)) & 15) == 0;
    if (vec && i + 4 <= n) {
        float4 a = *reinterpret_cast<const float4*>(partial + i);
        for (int s = 1; s < splits; ++s) {
            const float4 b = *reinterpret_cast<const float4*>(partial + s * stride + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        *reinterpret_cast<float4*>(G + i) = a;
    } else {
        for (size_t j = i; j < n && j < i + 4; ++j) {
            float a = partial[j];
            for (int s = 1; s < splits; ++s) a += partial[s * stride + j];
            G[j] = a;
        }
    }
}
void launch_reduce_partials(Ctx* ctx, const float* partial, size_t stride, int splits, float* G, size_t n) {
    const size_t threads = (n + 3) / 4;
    reduce_partials_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, ctx->stream>>>(partial, stride, splits, G, n);
    count_launch(ctx);
}

// Momentum update of W fused with the split-K reduction of the dW partials (single-GPU path: no
// all-reduce needs the reduced gradient in memory) and with the refresh of the bf16 shadow the
// tensor-core GEMMs read.  base_rbm.py:447-449, 462, 467-468.  V*H must be a multiple of 4 (checked).
__global__ void weight_update_splitk_kernel(const float* __restrict__ partial, size_t stride, int splits, float g_div,
                                            float* __restrict__ W, float* __restrict__ dW, int H, size_t n,
                                            const float* __restrict__ pen, float l2, float lr, float mom,
                                            __nv_bfloat16* __restrict__ Wb, int ldwb) {
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    float4 g = *reinterpret_cast<const float4*>(partial + i);
    for (int s = 1; s < splits; ++s) {
        const float4 b = *reinterpret_cast<const float4*>(partial + s * stride + i);
        g.x += b.x; g.y += b.y; g.z += b.z; g.w += b.w;
    }
    const int h = (int)(i % (size_t)H);          // H % 4 == 0: the four elements share a row
    const size_t v = i / (size_t)H;
    const float4 w = *reinterpret_cast<const float4*>(W + i);
    const float4 d0 = *reinterpret_cast<const float4*>(dW + i);
    const float4 p = *reinterpret_cast<const float4*>(pen + h);
    float4 d, wn;
    d.x = lr * (mom * d0.x + (g.x / g_div - l2 * w.x - p.x)); wn.x = w.x + d.x;
    d.y = lr * (mom * d0.y + (g.y / g_div - l2 * w.y - p.y)); wn.y = w.y + d.y;
    d.z = lr * (mom * d0.z + (g.z / g_div - l2 * w.z - p.z)); wn.z = w.z + d.z;
    d.w = lr * (mom * d0.w + (g.w / g_div - l2 * w.w - p.w)); wn.w = w.w + d.w;
    *reinterpret_cast<float4*>(dW + i) = d;
    *reinterpret_cast<float4*>(W + i) = wn;
    __nv_bfloat162 lo = __floats2bfloat162_rn(wn.x, wn.y), hi = __floats2bfloat162_rn(wn.z, wn.w);
    uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(Wb + v * (size_t)ldwb + h) = pk;
}
void launch_weight_update_splitk(Ctx* ctx, const float* partial, size_t stride, int splits, float g_div, float* W, float* dW,
                                 int V, int H, const float* pen, float l2, float lr, float mom, __nv_bfloat16* Wb, int ldwb) {
    BM_REQUIRE(H % 4 == 0 && ldwb % 4 == 0 && (stride & 3) == 0, "fused weight update needs n_hidden % 4 == 0 and 16-byte aligned slices");
    const size_t n = (size_t)V * H;
    const size_t threads = n / 4;
    weight_update_splitk_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, ctx->stream>>>(partial, stride, splits, g_div, W, dW, H, n,
                                                                                           pen, l2, lr, mom, Wb, ldwb);
    count_launch(ctx);
}


// ---- one launch for the whole update of a CD step (see CdTail in bm_tc.h) -----------------------------------------------
// block `blk` of the update of one model: blocks [0, w_blocks) update W, the rest the biases
template <int VEC>
__device__ __forceinline__ void cd_tail_block(const CdTail& t, unsigned w_blocks, unsigned blk) {
    const int V = t.V, H = t.H;
    if (blk < w_blocks) {
        // ---- weights: VEC consecutive hidden units of one visible unit per thread ----
        const size_t n = (size_t)V * H;
        const size_t i = ((size_t)blk * blockDim.x + threadIdx.x) * VEC;
        if (i >= n) return;
        const int h = (int)(i % (size_t)H);
        const size_t v = i / (size_t)H;
        float g[VEC], pen[VEC], w[VEC], d0[VEC];
        if constexpr (VEC == 4) {
            float4 a = *reinterpret_cast<const float4*>(t.part + i);
            for (int s = 1; s < t.splits; ++s) {
                const float4 b = *reinterpret_cast<const float4*>(t.part + (size_t)s * t.stride + i);
                a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
            }
            g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w;
            const float4 w4 = *reinterpret_cast<const float4*>(t.W + i), d4 = *reinterpret_cast<const float4*>(t.dW + i);
            w[0] = w4.x; w[1] = w4.y; w[2] = w4.z; w[3] = w4.w; d0[0] = d4.x; d0[1] = d4.y; d0[2] = d4.z; d0[3] = d4.w;
        } else {
            float a = t.part[i];
            for (int s = 1; s < t.splits; ++s) a += t.part[(size_t)s * t.stride + i];
            g[0] = a; w[0] = t.W[i]; d0[0] = t.dW[i];
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) pen[j] = 0.f;
        if (t.cost != 0.f) {                                     // base_rbm.py:457-461
            const size_t qrow = (size_t)(t.srow + 1) * H + h;
#pragma unroll
            for (int j = 0; j < VEC; ++j) {
                float qs = 0.f;
                for (int s = 0; s < t.splits; ++s) qs += t.part[(size_t)s * t.stride + qrow + j];
                const float q = t.damp * t.q_old[h + j] + (1.0f - t.damp) * (-qs);
                pen[j] = t.cost * (q - t.target);
            }
        }
        float d[VEC], wn[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            d[j] = t.lr * (t.mom * d0[j] + (g[j] / t.n_div - t.l2 * w[j] - pen[j]));     // :449, :462, :467
            wn[j] = w[j] + d[j];                                                           // :468
        }
        if constexpr (VEC == 4) {
            *reinterpret_cast<float4*>(t.dW + i) = make_float4(d[0], d[1], d[2], d[3]);
            *reinterpret_cast<float4*>(t.W + i) = make_float4(wn[0], wn[1], wn[2], wn[3]);
            __nv_bfloat162 lo = __floats2bfloat162_rn(wn[0], wn[1]), hi = __floats2bfloat162_rn(wn[2], wn[3]);
            uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(t.Wb + v * (size_t)t.ldwb + h) = pk;
        } else {
            t.dW[i] = d[0]; t.W[i] = wn[0];
            t.Wb[v * (size_t)t.ldwb + h] = __float2bfloat16_rn(wn[0]);
        }
        return;
    }
    // ---- biases, sparsity statistics ----
    const int i = (int)(blk - w_blocks) * blockDim.x + threadIdx.x;
    if (i < H) {
        float ds = 0.f, qs = 0.f;
        for (int s = 0; s < t.splits; ++s) {
            ds += t.part[(size_t)s * t.stride + (size_t)t.srow * H + i];
            qs += t.part[(size_t)s * t.stride + (size_t)(t.srow + 1) * H + i];
        }
        const float q = t.damp * t.q_old[i] + (1.0f - t.damp) * (-qs);                     // :457-459
        t.q_new[i] = q;
        const float pen = t.cost * (q - t.target);
        t.pen[i] = pen;
        const float g = ds / t.n_div - pen;                                                // :453, :461
        const float d = t.lr * (t.mom * t.dhb[i] + g);                                     // :473-474
        t.dhb[i] = d;
        t.hb[i] += d;
    }
    if (i < V) {
        float vs = 0.f;
        for (int s = 0; s < t.vsplits; ++s) vs += t.vpart[(size_t)s * t.vstride + i];
        const float d = t.lr * (t.mom * t.dvb[i] + vs / t.n_div);                          // :451, :470-471
        t.dvb[i] = d;
        t.vb[i] += d;
    }
}
template <int VEC>
__global__ void __launch_bounds__(256) cd_tail_kernel(const CdTail t, unsigned w_blocks) { cd_tail_block<VEC>(t, w_blocks, blockIdx.x); }
// training groups: model m takes blocks [m * per_model, (m + 1) * per_model)
template <int VEC>
__global__ void __launch_bounds__(256) cd_tail_group_kernel(const CdTail* __restrict__ tails, unsigned per_model, unsigned w_blocks) {
    cd_tail_block<VEC>(tails[blockIdx.x / per_model], w_blocks, blockIdx.x % per_model);
}
static bool cd_tail_vec(const CdTail& t) {
    return t.H % 4 == 0 && t.ldwb % 4 == 0 && (t.stride & 3) == 0 && (reinterpret_cast<uintptr_t>(t.part) & 15) == 0;
}
static void cd_tail_blocks(const CdTail& t, bool vec, unsigned* w_blocks, unsigned* b_blocks) {
    const size_t items = ((size_t)t.V * t.H) / (vec ? 4 : 1);
    *w_blocks = (unsigned)((items + 255) / 256);
    const int nb = t.V > t.H ? t.V : t.H;
    *b_blocks = (unsigned)((nb + 255) / 256);
}
void launch_cd_tail(Ctx* ctx, const CdTail& t) {
    const bool vec = cd_tail_vec(t);
    unsigned w_blocks, b_blocks;
    cd_tail_blocks(t, vec, &w_blocks, &b_blocks);
    if (vec) cd_tail_kernel<4><<<w_blocks + b_blocks, 256, 0, ctx->stream>>>(t, w_blocks);
    else cd_tail_kernel<1><<<w_blocks + b_blocks, 256, 0, ctx->stream>>>(t, w_blocks);
    count_launch(ctx);
}
void launch_cd_tail_group(Ctx* ctx, const CdTail* dev_tails, const CdTail& first, int n) {
    const bool vec = cd_tail_vec(first);
    unsigned w_blocks, b_blocks;
    cd_tail_blocks(first, vec, &w_blocks, &b_blocks);
    const unsigned per = w_blocks + b_blocks;
    if (vec) cd_tail_group_kernel<4><<<per * (unsigned)n, 256, 0, ctx->stream>>>(dev_tails, per, w_blocks);
    else cd_tail_group_kernel<1><<<per * (unsigned)n, 256, 0, ctx->stream>>>(dev_tails, per, w_blocks);
    count_launch(ctx);
}

__global__ void set_column_pair_kernel(__nv_bfloat16* __restrict__ buf, int ld, size_t rows, int col0, float a, float b) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    buf[r * (size_t)ld + col0] = __float2bfloat16_rn(a);
    buf[r * (size_t)ld + col0 + 1] = __float2bfloat16_rn(b);
}
void launch_set_column_pair(Ctx* ctx, __nv_bfloat16* buf, int ld, size_t rows, int col0, float a, float b) {
    if (rows == 0) return;
    set_column_pair_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, ctx->stream>>>(buf, ld, rows, col0, a, b);
    count_launch(ctx);
}
__global__ void fill_bf16_kernel(__nv_bfloat16* __restrict__ buf, size_t n, float v) {
    const __nv_bfloat16 x = __float2bfloat16_rn(v);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) buf[i] = x;
}
void launch_fill_bf16(Ctx* ctx, __nv_bfloat16* buf, size_t n, float v) {
    if (n == 0) return;
    const size_t blocks = (n + 255) / 256;
    fill_bf16_kernel<<<(unsigned)(blocks < 1184 ? blocks : 1184), 256, 0, ctx->stream>>>(buf, n, v);
    count_launch(ctx);
}

}  // namespace bm
