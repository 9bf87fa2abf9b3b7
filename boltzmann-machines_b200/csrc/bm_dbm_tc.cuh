// Tensor-core DBM engine (BM_COMPUTE_BF16, float32 models): included by bm_dbm.cu after Dbm<T>.
//
// Same state, same update kernels and same control flow as Dbm<float> (the reference's dbm.py, see the
// header of bm_dbm.cu); every GEMM -- the layer-wise Gibbs step with its two-sided input
// H_{i-1} W_i + H_{i+1} W_{i+1}^T (dbm.py:385-427) as ONE two-pair tensor-core op, the mean-field sweeps
// (:429-478), the particle sweeps (:480-509), the gradients pos^T mu - neg^T h (:558-568, split over the
// batch rows), the pre-activations of the AIS ladder (:650-736) -- runs on the fused tensor-core layer op
// of bm_tc.cu (bf16 operands, fp32 accumulation in registers, bias + beta scaling + sigmoid + Philox draw in
// the epilogue).  Variables stay fp32 as in the reference; activations (variational parameters, particles,
// AIS states) are kept as bf16 operands, binary samples being exact in bf16.  AIS pre-activations leave the
// kernel in fp32 and the importance weights are accumulated in fp64 from differences
//   softplus(b z) - softplus(a z) = log1p(sigmoid(a z) * expm1((b - a) z)),
// which is exact to fp32 rounding of a SMALL quantity (no cancellation between two O(1) softplus values).
//
// STATUS: the default engine of float32 DBMs with Bernoulli hidden layers (bm_dbm_cfg.compute = BM_COMPUTE_BF16, which the
// Python mirror passes unless compute='fp32' or BM_DBM_COMPUTE / BM_COMPUTE = fp32 asks for the storage-precision CUDA-core
// engine).  Multinomial hidden layers run here too (dbm_multinomial_rows_kernel after an fp32 pre-activation op); the Python
// mirror sends such models here only on an explicit compute='bf16' or BM_DBM_COMPUTE=bf16.  Models it does not support
// (DbmTC::supports) run on the CUDA-core engine.
#pragma once
#include <map>
#include <memory>
#include <utility>
#include <tuple>

namespace bm {

typedef __nv_bfloat16 bf16_t;

static inline int dbm_round_up(int x, int m) { return (x + m - 1) / m * m; }

// Convergence tests of a speculated chunk of mean-field sweeps: `hist` holds slots 0..n_tests of one layer's variational
// parameters ([slot][rows_cap, ld]); flags[j] = max(flags[j], max |slot j+1 - slot j|) over the [rows, cols] window.
__global__ void mf_chunk_diffs_kernel(const bf16_t* __restrict__ hist, size_t slot_stride, int ld, int rows, int cols,
                                      unsigned int* __restrict__ flags) {
    const int j = blockIdx.y;
    const bf16_t* a = hist + (size_t)(j + 1) * slot_stride;
    const bf16_t* b = hist + (size_t)j * slot_stride;
    float m = 0.f;
    const size_t total = (size_t)rows * cols;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        m = fmaxf(m, fabsf(__bfloat162float(a[(size_t)r * ld + c]) - __bfloat162float(b[(size_t)r * ld + c])));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(flags + j, __float_as_uint(m));
}

// The conditional of a multinomial layer from its fp32 pre-activations x + b (layers.py:65-70), one row per 256-thread block:
//   means = scale * softmax(row)                                     softmax_rows_kernel<float> (bm_simt.cu)
//   n_draws > 0: the counts of n_draws categorical draws of the row   multinomial_rows_kernel<float> on those means
// and the result leaves as the bf16 GEMM operand `out` (ldo) and, when out_f32 is given, in fp32 as well (ldf): the layer's
// persistent particles, whose counts stay exact integers above 256 where the bf16 operand rounds them.
// Bit-identical to the two kernels in sequence: the max and the double sum of the exponentials are reduced in their order (256
// strided partials, then the same tree), and one thread accumulates the row sum and the CDF sequentially, like theirs.
// Dynamic shared memory: the row (fp32), and for draws its CDF (fp64, 8-byte aligned) and the counts (int).
__global__ void __launch_bounds__(256) dbm_multinomial_rows_kernel(const float* __restrict__ pre, int ldp, int cols, float scale,
                                                                    int n_draws, bf16_t* __restrict__ out, int ldo,
                                                                    float* __restrict__ out_f32, int ldf, RngKey rng) {
    extern __shared__ __align__(16) unsigned char mult_smem[];
    float* x = reinterpret_cast<float*>(mult_smem);
    double* cdf = reinterpret_cast<double*>(mult_smem + ((size_t)cols * sizeof(float) + 7) / 8 * 8);
    int* cnt = reinterpret_cast<int*>(cdf + cols);
    __shared__ double sh[256];
    const int r = blockIdx.x, tid = threadIdx.x;
    const float* row = pre + (size_t)r * ldp;
    double mx = -1e300;
    for (int c = tid; c < cols; c += 256) { const float v = row[c]; x[c] = v; mx = fmax(mx, (double)v); }
    sh[tid] = mx;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (tid < o) sh[tid] = fmax(sh[tid], sh[tid + o]);
        __syncthreads();
    }
    const float m = (float)sh[0];
    __syncthreads();
    double s = 0.0;
    for (int c = tid; c < cols; c += 256) { const float e = expf(x[c] - m); x[c] = e; s += (double)e; }
    sh[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (tid < o) sh[tid] += sh[tid + o];
        __syncthreads();
    }
    const float tot = (float)sh[0];
    for (int c = tid; c < cols; c += 256) x[c] = scale * x[c] / tot;
    if (n_draws <= 0) {
        for (int c = tid; c < cols; c += 256) {
            out[(size_t)r * ldo + c] = __float2bfloat16_rn(x[c]);
            if (out_f32) out_f32[(size_t)r * ldf + c] = x[c];
        }
        return;
    }
    for (int c = tid; c < cols; c += 256) cnt[c] = 0;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int c = 0; c < cols; ++c) t += (double)x[c];
        double run = 0.0;
        for (int c = 0; c < cols; ++c) { run += (double)(float)((double)x[c] / t); cdf[c] = run; }
    }
    __syncthreads();
    const double last = cdf[cols - 1];
    __syncthreads();
    for (int c = tid; c < cols; c += 256) cdf[c] = cdf[c] / last;
    __syncthreads();
    for (int d = tid; d < n_draws; d += 256) {
        const U4 w = site_block(rng, (uint32_t)r, (uint32_t)(d >> 2));
        const uint32_t words[4] = {w.x, w.y, w.z, w.w};
        const double u = (double)u32_to_unit_float(words[d & 3]);
        int lo = 0, hi = cols;                                    // first index with cdf > u
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cdf[mid] > u) hi = mid; else lo = mid + 1;
        }
        atomicAdd(&cnt[lo < cols ? lo : cols - 1], 1);
    }
    __syncthreads();
    for (int c = tid; c < cols; c += 256) {
        const float k = (float)cnt[c];
        out[(size_t)r * ldo + c] = __float2bfloat16_rn(k);
        if (out_f32) out_f32[(size_t)r * ldf + c] = k;
    }
}
// The label clamp of a classification DBM (DESIGN.md §5.7): rows r < rows whose label t = labels[r] is >= 0 get the one-hot
// e_t in columns [0, cols) of `n_slots` bf16 buffers [rows, ld] spaced `slot_stride` apart (slot = blockIdx.y); rows labelled -1
// are left as they are.  One warp per row.
__global__ void cdbm_clamp_labels_kernel(const int* __restrict__ labels, int rows, int cols, bf16_t* __restrict__ out, int ld,
                                         size_t slot_stride) {
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= rows) return;
    const int t = labels[r];
    if (t < 0) return;
    bf16_t* row = out + (size_t)blockIdx.y * slot_stride + (size_t)r * ld;
    for (int c = lane; c < cols; c += 32) row[c] = __float2bfloat16_rn(c == t ? 1.f : 0.f);
}
void launch_cdbm_clamp_labels(Ctx* ctx, const int* labels, int rows, int cols, bf16_t* out, int ld, int n_slots = 1,
                              size_t slot_stride = 0) {
    if (rows <= 0 || n_slots <= 0) return;
    cdbm_clamp_labels_kernel<<<dim3((rows + 7) / 8, n_slots), 256, 0, ctx->stream>>>(labels, rows, cols, out, ld, slot_stride);
    count_launch(ctx);
}

static inline size_t dbm_multinomial_smem(int cols, bool draws) {
    return ((size_t)cols * sizeof(float) + 7) / 8 * 8 + (draws ? (size_t)cols * (sizeof(double) + sizeof(int)) : 0);
}
void launch_dbm_multinomial_rows(Ctx* ctx, const float* pre, int ldp, int rows, int cols, float scale, int n_draws,
                                 bf16_t* out, int ldo, float* out_f32, int ldf, RngKey rng) {
    if (rows <= 0) return;
    const size_t smem = dbm_multinomial_smem(cols, n_draws > 0);
    if (smem > 48 * 1024)
        BM_CUDA(cudaFuncSetAttribute(dbm_multinomial_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dbm_multinomial_rows_kernel<<<rows, 256, smem, ctx->stream>>>(pre, ldp, cols, scale, n_draws, out, ldo, out_f32, ldf, rng);
    count_launch(ctx);
}

// dst[c, r] = bf16(src[r, c]): the transposed bf16 shadow of a weight matrix (src [rows, cols] dense fp32, dst leading dimension ldd)
__global__ void transpose_f32_to_bf16_kernel(const float* __restrict__ src, int rows, int cols, bf16_t* __restrict__ dst, int ldd) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < rows && c < cols) ? src[(size_t)r * cols + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;              // dst row = source column
        if (c < cols && r < rows) dst[(size_t)c * ldd + r] = __float2bfloat16_rn(tile[threadIdx.x][i]);
    }
}

// G = (sum of `sp` positive slices) / n_div - (sum of `sn` negative slices) / m_div      (dbm.py:558-568)
__global__ void dbm_grad_combine_kernel(const float* __restrict__ pos, int sp, const float* __restrict__ neg, int sn,
                                        size_t stride, float inv_n, float inv_m, float* __restrict__ G, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int s = 0; s < sp; ++s) a += pos[(size_t)s * stride + i];
        for (int s = 0; s < sn; ++s) b += neg[(size_t)s * stride + i];
        G[i] = a * inv_n - b * inv_m;
    }
}

// ---- centering (DESIGN.md §5.8) ---------------------------------------------------------------------------------------------
// Unit layers j = 0..L (0 = visible): offsets o_j, data side d_j (X, mu_{j-1}) and particle side p_j (v, h_{j-1}).  Every fp32
// operation below is written out with _rn intrinsics so that nothing is contracted and the host restatements follow it exactly.
struct CenterArgs {
    int n_layers;                   // L + 1
    int n[9];
    const float* dsum[9];           // column sums of d_j over the rows present
    const float* psum[9];           // column sums of p_j over the particles
    float* o[9];                    // the offsets of this step (written on a model's first step)
    float* o_next[9];               // the offsets after this step: (1 - rate) o + rate mean_rows(d)
    float* s[9];                    // s_j = dsum / N - psum / M
    float rows, inv_n, inv_m, keep, rate;
    int init;                       // a model's first step: o_j <- mean_rows(d_j) first
};
__global__ void dbm_center_stats_kernel(CenterArgs a) {
    const int j = blockIdx.y, u = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= a.n_layers || u >= a.n[j]) return;
    const float d = a.dsum[j][u], mean = __fdiv_rn(d, a.rows);
    float o = a.o[j][u];
    if (a.init) { o = mean; a.o[j][u] = o; }
    a.s[j][u] = __fsub_rn(__fmul_rn(d, a.inv_n), __fmul_rn(a.psum[j][u], a.inv_m));
    a.o_next[j][u] = __fadd_rn(__fmul_rn(a.keep, o), __fmul_rn(a.rate, mean));
}

// The centered gradient of W_i (H = n_{i+1} columns) from the split-K slices of the plain one:
//   G^c = (pos / N - neg / M) - o_i s_{i+1}' - s_i o_{i+1}' + corr o_i o_{i+1}',   corr = rows / N - 1
// the literal restatement of sum (d_i - o_i)(d_{i+1} - o_{i+1})' / N - sum (p_i - o_i)(p_{i+1} - o_{i+1})' / M.  The first term
// is dbm_grad_combine_kernel's expression, so zero offsets give its result bit for bit.
__global__ void dbm_centered_grad_combine_kernel(const float* __restrict__ pos, int sp, const float* __restrict__ neg, int sn,
                                                 size_t stride, float inv_n, float inv_m, int H,
                                                 const float* __restrict__ o_in, const float* __restrict__ s_in,
                                                 const float* __restrict__ o_out, const float* __restrict__ s_out, float corr,
                                                 float* __restrict__ G, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float a = 0.f, b = 0.f;
        for (int s = 0; s < sp; ++s) a += pos[(size_t)s * stride + i];
        for (int s = 0; s < sn; ++s) b += neg[(size_t)s * stride + i];
        const size_t r = i / (size_t)H, c = i % (size_t)H;
        float g = a * inv_n - b * inv_m;
        g = __fsub_rn(g, __fmul_rn(o_in[r], s_out[c]));
        g = __fsub_rn(g, __fmul_rn(s_in[r], o_out[c]));
        g = __fadd_rn(g, __fmul_rn(corr, __fmul_rn(o_in[r], o_out[c])));
        G[i] = g;
    }
}

// The coupling of unit layer j to the offsets of its neighbours, c_j = W_{j-1}' o_{j-1} + W_j o_{j+1} (missing terms dropped),
// in fp32.  mode 0: cpl_j <- c_j.  mode 1: b_j <- b_j - (c_j - cpl_j), which keeps a_j = b_j + c_j when W has changed.
// Block (32, 8) per 32 units of layer blockIdx.y.  The column term: thread (x, y) sums rows y, y + 8, ... of column x with
// fma, then the 8 partials add in order; the row term: warp y takes units y, y + 8, y + 16, y + 24, lane l sums k = l, l + 32,
// ... with fma, then the xor tree; c = colterm + rowterm.
struct CouplingArgs {
    int n_layers;                   // L + 1
    int n[9];
    const float* W[8];              // W_i [n_i, n_{i+1}]
    const float* o[9];
    float* cpl[9];
    float* b[9];                    // vb, hb, hb_1, ...
    int mode;
};
__global__ void __launch_bounds__(256) dbm_coupling_kernel(CouplingArgs a) {
    __shared__ float colp[8][33];
    __shared__ float rowp[32];
    const int j = blockIdx.y, tx = threadIdx.x, ty = threadIdx.y;
    const int n = a.n[j], u0 = blockIdx.x * 32;
    if (u0 >= n) return;                                     // uniform over the block
    float cp = 0.f;
    if (j > 0 && u0 + tx < n) {
        const float* W = a.W[j - 1];
        const float* o = a.o[j - 1];
        for (int r = ty; r < a.n[j - 1]; r += 8) cp = __fmaf_rn(W[(size_t)r * n + u0 + tx], o[r], cp);
    }
    colp[ty][tx] = cp;
    for (int q = ty; q < 32; q += 8) {
        float s = 0.f;
        if (j + 1 < a.n_layers && u0 + q < n) {
            const int m = a.n[j + 1];
            const float* W = a.W[j] + (size_t)(u0 + q) * m;
            const float* o = a.o[j + 1];
            for (int k = tx; k < m; k += 32) s = __fmaf_rn(W[k], o[k], s);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, off));
        if (tx == 0) rowp[q] = s;
    }
    __syncthreads();
    if (ty == 0 && u0 + tx < n) {
        float c = 0.f;
#pragma unroll
        for (int y = 0; y < 8; ++y) c = __fadd_rn(c, colp[y][tx]);
        c = __fadd_rn(c, rowp[tx]);
        const int u = u0 + tx;
        if (a.mode == 0) a.cpl[j][u] = c;
        else a.b[j][u] = __fsub_rn(a.b[j][u], __fsub_rn(c, a.cpl[j][u]));
    }
}

// AIS unit update from fp32 pre-activations: out = sample ? (u < sigmoid(beta * pre)) : sigmoid(beta * pre), bf16.
// pre == nullptr: pre-activation 0 (the uniform base-rate draw x_0 ~ Ber(1/2), dbm.py:700-702).
// ldo % 4 == 0 (buffers are padded to 64 columns): the four columns of a Philox block leave as one 8-byte store.
__global__ void ais_unit_bf16_kernel(const float* __restrict__ pre, int ldp, float beta, bf16_t* __restrict__ out, int ldo,
                                     int rows, int cols, int sample, RngKey rng) {
    const int cb = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    if (cb * 4 >= cols || r >= rows) return;
    U4 w{0, 0, 0, 0};
    if (sample) w = site_block(rng, (uint32_t)r, (uint32_t)cb);
    const uint32_t words[4] = {w.x, w.y, w.z, w.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int c = cb * 4 + j;
        const float z = (pre && c < cols) ? beta * pre[(size_t)r * ldp + c] : 0.f;
        const float p = 1.0f / (1.0f + expf(-z));
        o[j] = (c < cols) ? (sample ? ((u32_to_unit_float(words[j]) < p) ? 1.0f : 0.0f) : p) : 0.f;
    }
    const __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], o[3]);
    uint2 pk;
    pk.x = *reinterpret_cast<const uint32_t*>(&lo); pk.y = *reinterpret_cast<const uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(out + (size_t)r * ldo + cb * 4) = pk;       // columns >= cols land in the padding
}

// v's operand of the clamped AIS ladder (DESIGN.md §5.4g): chain i of a slice is chain c0 + i of the call, which reads row
// (c0 + i) / n_runs of X [rows, V] (float32, device).  out [n, ldo] bf16 with the padding columns zero; binary rows are exact.
__global__ void ais_clamp_rows_kernel(const float* __restrict__ X, int V, long long c0, int n_runs, bf16_t* __restrict__ out,
                                      int ldo, int n) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y;
    if (c >= ldo || i >= n) return;
    const float* x = X + (size_t)((c0 + i) / n_runs) * V;
    out[(size_t)i * ldo + c] = __float2bfloat16_rn(c < V ? x[c] : 0.f);
}

// softplus(b z) - softplus(a z), b >= a >= 0, without cancellation
__device__ __forceinline__ float softplus_diff(float a, float b, float z) {
    const float s = 1.0f / (1.0f + expf(-a * z));          // sigmoid(a z)
    return log1pf(s * expm1f((b - a) * z));
}

// logw[r] += log p*_b(x_r) - log p*_a(x_r),  log p*_beta(x) = beta x.c1 + sum softplus(beta pa) + sum softplus(beta pb)
// (dbm.py:650-668); one warp per chain, fp64 accumulation
__global__ void ais_accum2_bf16_kernel(double* __restrict__ logw, float a, float b, const bf16_t* __restrict__ x, int ldx, int H0,
                                       const float* __restrict__ hb0, const float* __restrict__ pa, int V,
                                       const float* __restrict__ pb, int H1, int rows) {
    const int r = blockIdx.x * blockDim.y + threadIdx.y;
    if (r >= rows) return;
    double acc = 0.0;
    float lin = 0.f;
    for (int j = threadIdx.x; j < H0; j += 32) lin += __bfloat162float(x[(size_t)r * ldx + j]) * hb0[j];
    acc += ((double)b - (double)a) * (double)lin;
    float part = 0.f;
    int n = 0;
    for (int j = threadIdx.x; j < V; j += 32) {
        part += softplus_diff(a, b, pa[(size_t)r * V + j]);
        if (++n == 8) { acc += (double)part; part = 0.f; n = 0; }
    }
    for (int j = threadIdx.x; j < H1; j += 32) {
        part += softplus_diff(a, b, pb[(size_t)r * H1 + j]);
        if (++n == 8) { acc += (double)part; part = 0.f; n = 0; }
    }
    acc += (double)part;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) logw[r] += acc;
}

// One pass over the shared pre-activations of a temperature step: the importance-weight increment of ais_accum2_bf16_kernel
// AND the first unit updates of the next transition (v ~ sigmoid(beta_next pa), h2 ~ sigmoid(beta_next pb), exactly the
// expressions of ais_unit_bf16_kernel) -- pa / pb are read once instead of three times.  One warp per chain; a lane owns
// whole Philox blocks (4 consecutive columns).  emit == 0: weights only (the last increment of the ladder).
__device__ __forceinline__ float ais_fused_row(const float* __restrict__ pre, int n, float a, float b, float beta_next, int emit,
                                               int sample, bf16_t* __restrict__ out, const RngKey& rng, int r, int lane) {
    float part = 0.f;
    for (int cb = lane; cb * 4 < n; cb += 32) {
        float z[4], o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) z[j] = (cb * 4 + j < n) ? pre[cb * 4 + j] : 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) if (cb * 4 + j < n) part += softplus_diff(a, b, z[j]);
        if (emit) {
            U4 w{0, 0, 0, 0};
            if (sample) w = site_block(rng, (uint32_t)r, (uint32_t)cb);
            const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float zz = (cb * 4 + j < n) ? beta_next * z[j] : 0.f;
                const float p = 1.0f / (1.0f + expf(-zz));
                o[j] = (cb * 4 + j < n) ? (sample ? ((u32_to_unit_float(words[j]) < p) ? 1.0f : 0.0f) : p) : 0.f;
            }
            const __nv_bfloat162 lo = __floats2bfloat162_rn(o[0], o[1]), hi = __floats2bfloat162_rn(o[2], o[3]);
            uint2 pk;
            pk.x = *reinterpret_cast<const uint32_t*>(&lo); pk.y = *reinterpret_cast<const uint32_t*>(&hi);
            *reinterpret_cast<uint2*>(out + cb * 4) = pk;
        }
    }
    return part;
}
__global__ void ais_fused_step_kernel(double* __restrict__ logw, float a, float b, float beta_next, int emit,
                                      const bf16_t* __restrict__ x, int ldx, int H0, const float* __restrict__ hb0,
                                      const float* __restrict__ pa, int V, bf16_t* __restrict__ va, int ldv, int sample_v, RngKey rng_v,
                                      const float* __restrict__ pb, int H1, bf16_t* __restrict__ hc, int ldh, int sample_h2, RngKey rng_h2,
                                      int rows) {
    const int r = blockIdx.x * blockDim.y + threadIdx.y;
    if (r >= rows) return;
    const int lane = threadIdx.x;
    float lin = 0.f;
    for (int j = lane; j < H0; j += 32) lin += __bfloat162float(x[(size_t)r * ldx + j]) * hb0[j];
    double acc = ((double)b - (double)a) * (double)lin;
    acc += (double)ais_fused_row(pa + (size_t)r * V, V, a, b, beta_next, emit, sample_v, va + (size_t)r * ldv, rng_v, r, lane);
    acc += (double)ais_fused_row(pb + (size_t)r * H1, H1, a, b, beta_next, emit, sample_h2, hc + (size_t)r * ldh, rng_h2, r, lane);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) logw[r] += acc;
}

// The terms of hidden layer i in the variational bound of a DBM of any depth (dbm.py:743-757 for L layers), in float64 per
// row: out[r] (+)= t.mu + mu.c + H(clip(mu, 1e-7, 1 - 1e-7)) with t = mu_{i-1} W_i (X W_0 for i = 0); the launch of layer 0
// also sets out[r] = X.b_v first.  One warp per row, one launch per layer.
__global__ void dbm_bound_layer_rows_kernel(const float* __restrict__ X, int V, const float* __restrict__ vb,
                                            const float* __restrict__ mu, const float* __restrict__ t, const float* __restrict__ hb,
                                            int H, int first, int rows, double* __restrict__ out) {
    const int r = blockIdx.x * blockDim.y + threadIdx.y;
    if (r >= rows) return;
    double a = 0.0;
    for (int j = threadIdx.x; j < H; j += 32) {
        const double m = (double)mu[(size_t)r * H + j];
        a += (double)t[(size_t)r * H + j] * m + m * (double)hb[j];
        const double s = (double)fminf(fmaxf((float)m, 1e-7f), 1.0f - 1e-7f);
        a += -s * log(s) - (1.0 - s) * log(1.0 - s);
    }
    if (first)
        for (int j = threadIdx.x; j < V; j += 32) a += (double)X[(size_t)r * V + j] * (double)vb[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) out[r] = first ? a : out[r] + a;
}

// ---- parallel tempering: the swap round ------------------------------------------------------------
// Slot m of the ladder holds rows [m M, (m+1) M) of every bf16 particle buffer x[0] = v, x[1 + i] = h_i.  P[i] [T M, H_i] holds
// the raw products h_{i-1} W_i + c_i of the same states (one fp32 tensor-core op per layer), so that
//   -E(x) = v.b + sum_i h_i . (h_{i-1} W_i + c_i).
struct PtSwapArgs {
    int L, T, M, V;
    int H[8];
    int ld[9];
    bf16_t* x[9];
    const float* P[8];
    const float* vb;
    const double* betas;            // [T] device
    int parity;                     // pairs (m, m+1) with m % 2 == parity are proposed
    RngKey rng;                     // seed, tick, row0 of the swap draws (site and t are set per pair)
    unsigned long long* accepted;   // [T - 1], cumulative
};
// One 256-thread block per particle p: the T energies of its slots (one warp per slot; per lane a strided sum in double, then
// the xor tree), the decision of every proposed pair (u from Philox (SITE_DBM_PT, t = m) at column 0 of row row0 + p; accept
// when log u < (beta_m - beta_{m+1}) (E_m - E_{m+1})), then the exchange of the accepted pairs' rows in every particle buffer.
// The proposed pairs are disjoint, so the exchanges never touch one row twice.  Dynamic shared memory: T doubles + T ints.
__global__ void __launch_bounds__(256) dbm_pt_swap_kernel(PtSwapArgs a) {
    extern __shared__ double pt_smem[];
    double* E = pt_smem;
    int* acc = reinterpret_cast<int*>(pt_smem + a.T);
    const int p = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int m = warp; m < a.T; m += 8) {
        const size_t row = (size_t)m * a.M + p;
        double s = 0.0;
        for (int j = lane; j < a.V; j += 32) s += (double)__bfloat162float(a.x[0][row * a.ld[0] + j]) * (double)a.vb[j];
        for (int i = 0; i < a.L; ++i)
            for (int j = lane; j < a.H[i]; j += 32)
                s += (double)__bfloat162float(a.x[i + 1][row * a.ld[i + 1] + j]) * (double)a.P[i][row * a.H[i] + j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) E[m] = -s;
    }
    __syncthreads();
    for (int m = threadIdx.x; m + 1 < a.T; m += blockDim.x) {
        int ok = 0;
        if ((m & 1) == a.parity) {
            RngKey k = a.rng;
            k.c2 = (SITE_DBM_PT & 0xFFu) | (((uint32_t)m & 0xFFFFFFu) << 8);
            const double u = (double)u32_to_unit_float(site_block(k, (uint32_t)p, 0).x);
            ok = log(u) < (a.betas[m] - a.betas[m + 1]) * (E[m] - E[m + 1]);
            if (ok) atomicAdd(a.accepted + m, 1ull);
        }
        acc[m] = ok;
    }
    __syncthreads();
    for (int m = 0; m + 1 < a.T; ++m) {
        if (!acc[m]) continue;
        for (int l = 0; l <= a.L; ++l) {
            const int n = l == 0 ? a.V : a.H[l - 1];
            bf16_t* r0 = a.x[l] + ((size_t)m * a.M + p) * a.ld[l];
            bf16_t* r1 = a.x[l] + ((size_t)(m + 1) * a.M + p) * a.ld[l];
            for (int j = threadIdx.x; j < n; j += blockDim.x) { const bf16_t t = r0[j]; r0[j] = r1[j]; r1[j] = t; }
        }
    }
}

// ---------------------------------------------------------------------------------------------
struct DbmTC : Dbm<float> {
    std::vector<int> ldn;                        // leading dimension of a bf16 activation of layer idx (0 = visible)
    std::vector<DevBuf<bf16_t>> Wb;              // bf16 shadows of W_i: [size(i), ldn[i+1]]
    // The layer-wise conditional adds y W_{i+1}^T to x W_i in one accumulator.  A second, TRANSPOSED shadow of W_{i+1}
    // ([H_{i+1}, ld(H_i)], i >= 1) lets both operand pairs read their B operand MN-major -- the layout combination the RBM
    // program runs.
    std::vector<DevBuf<bf16_t>> WbT;
    DevBuf<bf16_t> Xb, recon_b, v_b, v2_b, v3_b;
    std::vector<DevBuf<bf16_t>> mu_b, h_b, h2_b, h3_b;
    std::vector<DevBuf<float>> Gp;               // split-K slices of the gradient GEMMs
    // The fp32 copy h[i] of a multinomial layer's particles is never widened from bf16: it holds what set_param /
    // init_particles put there, then what the row kernel writes on every committed sweep (exact counts, where the bf16
    // operand rounds above 256).  Only the other layers' copies are widened from bf16 on demand.
    bool particles_f32_stale = false;            // the bf16 particles are newer than the fp32 copies get_param reads
    DevBuf<float> pre_f32;                       // fp32 pre-activations of a multinomial layer's conditional [max(B, M), H]

    // A multinomial conditional needs whole rows: its op writes fp32 pre-activations (ACT_LINEAR) and one row kernel turns
    // them into means / counts.  A chain of ops is therefore cut after every such op: the ops between two cuts run as one
    // program launch, the row kernel between two launches, all in stream order.  Without multinomial layers a chain is one
    // program, exactly as the ops were listed.
    // cut: the launch ends after this op even without a row kernel (tempered chains longer than one program)
    // clamp: after the row kernel, the rows of `out` labelled >= 0 in this device array are set to their one-hot label
    // vmask: then the visible clamp of a fill chain (DESIGN.md §5.9): vout <- vx wherever vmask ([rows, V] bytes) is set
    struct RowStep { int layer = -1; bf16_t* out = nullptr; float* out_f32 = nullptr; int rows = 0; bool sample = false; uint32_t site = 0, t = 0; bool cut = false;
                     const int* clamp = nullptr; const uint8_t* vmask = nullptr; const bf16_t* vx = nullptr; bf16_t* vout = nullptr; };
    struct TcChain { std::vector<std::unique_ptr<TcProgram>> progs; std::vector<RowStep> after; };
    // mean-field as persistent dataflow programs of up to MF_CHUNK speculated sweeps per launch: slot history + programs
    static constexpr int MF_CHUNK = 5;
    int mf_chunk = 0;                            // MF_CHUNK, clamped by max_mf and by TC_PROGRAM_OPS, at least 1
    std::vector<DevBuf<bf16_t>> hist;            // per layer: (mf_chunk + 2) slots of [B, ldn[i+1]]
    DevBuf<unsigned int> mf_flags;
    std::map<std::tuple<int, int, int>, TcChain> mf_progs;                   // keyed by (rows, sweeps in the chunk, mf_clamp)
    // The label layer of a classification DBM (ClassDbmTC, DESIGN.md §5.7) is the top layer L - 1.  Its E-step values of rows
    // labelled t >= 0 (mf_labels, device) are the one-hot e_t in every history slot:
    //   CLAMP_NONE  every value is free: the plain engine, op for op
    //   CLAMP_ROWS  a mixed batch: the top layer's row kernel is followed by the clamp of the labelled rows
    //   CLAMP_ALL   every row labelled: the top layer's ops are not run; the ops below it read the one-hot slots
    enum { CLAMP_NONE = 0, CLAMP_ROWS = 1, CLAMP_ALL = 2 };
    int mf_clamp = CLAMP_NONE;
    const int* mf_labels = nullptr;
    bool top_is_label = false;                   // the top layer's bias takes the plain momentum update, no sparsity term
    // committed particle sweeps as ONE persistent program: keyed by (sweeps, sampled, t0)
    std::map<std::tuple<int, int, int>, TcChain> pcd_progs;
    // parallel tempering (bm_dbm_cfg.n_temps): T slots of M chains in rows [m M, (m+1) M) of the bf16 particle buffers; the
    // fp32 copies v / h[i] (get_param "v", "h...") hold slot 0.  T == 1: the engine without tempering, op for op.
    int T = 1;
    std::vector<double> betas{1.0};
    DevBuf<double> pt_betas;
    DevBuf<unsigned long long> pt_accepted;      // [T - 1] swaps accepted since create
    std::vector<long long> pt_proposed;          // [T - 1] swaps proposed since create (known on the host)
    std::vector<DevBuf<float>> pt_pre;           // per layer [T M, H_i]: h_{i-1} W_i + c_i of the current particles
    std::map<std::tuple<int, int, int>, TcChain> pt_progs;   // committed tempered sweeps: keyed by (sweeps, sampled, t0)
    // centering (bm_dbm_cfg.centering, DESIGN.md §5.8): per unit layer j = 0..L the offsets off[oc][j] (a step's moved offsets
    // go to off[1 - oc], which then becomes current), s_j of the step and the coupling c_j before the update.  Off: none of it
    // exists and the step is the plain one, launch for launch.
    bool centering = false;
    float offset_rate = 0.f;
    bool offsets_set = false;                    // "offsets_set": the first step sets the offsets to the data means
    int oc = 0;
    std::vector<DevBuf<float>> off[2], cen_s, cpl;

    // float32; Bernoulli or Gaussian visibles; Bernoulli and multinomial hidden layers in any order (the DBM's multinomial
    // particles are refused on a sharded context by init_particles)
    static bool supports(const bm_dbm_cfg& f) {
        if (f.dtype != BM_DTYPE_F32) return false;
        if (!(f.v_kind == BM_UNIT_BERNOULLI || f.v_kind == BM_UNIT_GAUSSIAN)) return false;
        for (int i = 0; i < f.n_layers; ++i)
            if (f.h_kinds[i] != BM_UNIT_BERNOULLI && f.h_kinds[i] != BM_UNIT_MULTINOMIAL) return false;
        return f.n_layers <= TC_PROGRAM_OPS;     // one mean-field sweep (L ops) fits in one program
    }
    bool multinomial(int i) const { return h_kinds[i] == BM_UNIT_MULTINOMIAL; }
    // exact log Z / log p*(v) (bm_dbm_exact.cuh): 2^exact_chunk_bits states per launch of the enumeration (bounds g and the
    // rows' pairs); bm_dbm_debug_exact_chunk lowers it so that small models span several launches
    static constexpr int EXACT_CHUNK_BITS = 22;
    int exact_chunk_bits = EXACT_CHUNK_BITS;
    void exact(const void* X, int rows, double* log_p_star, double* log_Z) override;

    DbmTC(Ctx* c, const bm_dbm_cfg& f) : Dbm<float>(c, f) {
        if (f.n_temps >= 1) {                    // validated by bm_dbm_create (check_pt_cfg)
            T = f.n_temps;
            betas.assign(f.betas, f.betas + T);
        }
        const size_t TM = (size_t)T * M;
        ldn.push_back(dbm_round_up(V, 64));
        for (int i = 0; i < L; ++i) ldn.push_back(dbm_round_up(Hs[i], 64));
        Wb.resize(L); WbT.resize(L); mu_b.resize(L); h_b.resize(L); h2_b.resize(L); h3_b.resize(L); Gp.resize(L);
        Xb.ensure((size_t)B * ldn[0]); recon_b.ensure((size_t)B * ldn[0]);
        v_b.ensure(TM * ldn[0]); v2_b.ensure(TM * ldn[0]);
        for (DevBuf<bf16_t>* b : {&Xb, &recon_b, &v_b, &v2_b}) b->zero(ctx->stream);
        if (T > 1) {
            pt_betas.ensure(T);
            BM_CUDA(cudaMemcpyAsync(pt_betas.p, betas.data(), (size_t)T * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
            pt_accepted.ensure(T - 1); pt_accepted.zero(ctx->stream);
            pt_proposed.assign(T - 1, 0);
            pt_pre.resize(L);
            for (int i = 0; i < L; ++i) pt_pre[i].ensure(TM * Hs[i]);
        }
        for (int i = 0; i < L; ++i) {
            Wb[i].ensure((size_t)size_of(i, V, Hs) * ldn[i + 1]);
            mu_b[i].ensure((size_t)B * ldn[i + 1]);
            h_b[i].ensure(TM * ldn[i + 1]); h2_b[i].ensure(TM * ldn[i + 1]);
            for (DevBuf<bf16_t>* b : {&Wb[i], &mu_b[i], &h_b[i], &h2_b[i]}) b->zero(ctx->stream);
        }
        for (int i = 1; i < L; ++i) { WbT[i].ensure((size_t)Hs[i] * ldn[i]); WbT[i].zero(ctx->stream); }
        mf_chunk = std::max(1, std::min(std::min(MF_CHUNK, max_mf), TC_PROGRAM_OPS / L));
        hist.resize(L);
        for (int i = 0; i < L; ++i) { hist[i].ensure((size_t)(mf_chunk + 2) * B * ldn[i + 1]); hist[i].zero(ctx->stream); }
        mf_flags.ensure(mf_chunk);
        int hmax = 0;
        for (int i = 0; i < L; ++i) if (multinomial(i)) hmax = std::max(hmax, Hs[i]);
        if (hmax) pre_f32.ensure((size_t)std::max(B, M) * hmax);
        if (f.centering) {                       // validated by bm_dbm_create (check_centering_cfg)
            centering = true;
            offset_rate = (float)f.offset_rate;
            for (auto* v : {&off[0], &off[1], &cen_s, &cpl}) v->resize(L + 1);
            for (int j = 0; j <= L; ++j)
                for (DevBuf<float>* b : {&off[0][j], &off[1][j], &cen_s[j], &cpl[j]}) { b->ensure(size_of(j, V, Hs)); b->zero(ctx->stream); }
        }
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    static TcMat mat(const bf16_t* p, int rows, int cols, int ld) { TcMat m; m.ptr = p; m.rows = rows; m.cols = cols; m.ld = ld; return m; }

    // ---- fp32 <-> bf16 coherence ---------------------------------------------------------------------------
    void refresh_shadow(int i) {
        const int in = size_of(i, V, Hs);
        launch_f32_to_bf16(ctx, W[i].p, Hs[i], Wb[i].p, ldn[i + 1], in, Hs[i]);
        if (i >= 1) {
            transpose_f32_to_bf16_kernel<<<dim3((Hs[i] + 31) / 32, (in + 31) / 32), dim3(32, 8), 0, ctx->stream>>>(W[i].p, in, Hs[i], WbT[i].p, ldn[i]);
            count_launch(ctx);
        }
    }
    // second operand pair of a conditional: y W_{i+1}^T with y = `above` [rows, H_{i+1}]
    void above_pair(TcGemm& g, int i, const bf16_t* above, int rows) {
        const int H = Hs[i], Hn = Hs[i + 1];
        g.n_pairs = 2;
        g.A[1] = mat(above, rows, Hn, ldn[i + 2]); g.K[1] = Hn;
        g.B[1] = mat(WbT[i + 1].p, Hn, H, ldn[i + 1]); g.b_t[1] = true;                              // W_{i+1}^T stored [K, N]
    }
    void narrow_state() {          // fp32 variables (as set by the caller / initialised) -> bf16 operands
        launch_f32_to_bf16(ctx, v.p, V, v_b.p, ldn[0], M, V);
        for (int i = 0; i < L; ++i) {
            launch_f32_to_bf16(ctx, h[i].p, Hs[i], h_b[i].p, ldn[i + 1], M, Hs[i]);
            launch_f32_to_bf16(ctx, mu[i].p, Hs[i], mu_b[i].p, ldn[i + 1], B, Hs[i]);
            refresh_shadow(i);
        }
        // the bf16 operands are what the engine computes with: get_param reports them (widened), not the unrounded input
        widen_mu(B);
        particles_f32_stale = true;
    }
    void widen_particles() {
        if (!particles_f32_stale) return;
        launch_bf16_to_f32(ctx, v_b.p, ldn[0], v.p, V, M, V);
        for (int i = 0; i < L; ++i)
            if (!multinomial(i)) launch_bf16_to_f32(ctx, h_b[i].p, ldn[i + 1], h[i].p, Hs[i], M, Hs[i]);
        particles_f32_stale = false;
    }
    void widen_mu(int rows) { for (int i = 0; i < L; ++i) launch_bf16_to_f32(ctx, mu_b[i].p, ldn[i + 1], mu[i].p, Hs[i], rows, Hs[i]); }

    // "v_pt" -> 0, "h_pt" -> 1, "h_pt_<i>" -> i + 1: the tempered slots 1..T-1 of a particle layer ([T-1, M, n] on the host)
    int pt_layer(const std::string& name) const {
        if (T <= 1) return -1;
        if (name == "v_pt") return 0;
        if (name == "h_pt") return 1;
        for (int i = 1; i < L; ++i) if (name == "h_pt" + sfx(i)) return i + 1;
        return -1;
    }
    void pt_param(int idx, void* host, const void* in, size_t bytes) {
        const int n = size_of(idx, V, Hs);
        const int rows = (T - 1) * M;
        BM_REQUIRE(bytes == (size_t)rows * n * sizeof(float), "size mismatch for a tempered particle layer");
        bf16_t* slots = (idx == 0 ? v_b.p : h_b[idx - 1].p) + (size_t)M * ldn[idx];
        DevBuf<float> tmp;
        tmp.ensure((size_t)rows * n);
        if (in) {
            BM_CUDA(cudaMemcpyAsync(tmp.p, in, bytes, cudaMemcpyHostToDevice, ctx->stream));
            launch_f32_to_bf16(ctx, tmp.p, n, slots, ldn[idx], rows, n);
        } else {
            launch_bf16_to_f32(ctx, slots, ldn[idx], tmp.p, n, rows, n);
            BM_CUDA(cudaMemcpyAsync(host, tmp.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        }
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    // centering's variables: "v_offset" [V], "h_offset", "h_offset_<i>" [H_i] and "offsets_set" [1] (0 or 1).  false: not one.
    bool offset_param(const std::string& name, void* host, const void* in, size_t bytes) {
        if (!centering) return false;
        if (name == "offsets_set") {
            BM_REQUIRE(bytes == sizeof(float), "size mismatch for 'offsets_set'");
            float f = offsets_set ? 1.f : 0.f;
            if (in) { memcpy(&f, in, sizeof(f)); offsets_set = f != 0.f; } else memcpy(host, &f, sizeof(f));
            return true;
        }
        int j = name == "v_offset" ? 0 : -1;
        for (int i = 0; i < L && j < 0; ++i) if (name == "h_offset" + sfx(i)) j = i + 1;
        if (j < 0) return false;
        BM_REQUIRE(bytes == (size_t)size_of(j, V, Hs) * sizeof(float), "size mismatch for '" + name + "'");
        if (in) BM_CUDA(cudaMemcpyAsync(off[oc][j].p, in, bytes, cudaMemcpyHostToDevice, ctx->stream));
        else BM_CUDA(cudaMemcpyAsync(host, off[oc][j].p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        return true;
    }
    void set_param(const char* name, const void* host, size_t bytes) override {
        if (offset_param(name, nullptr, host, bytes)) return;
        const int pt = pt_layer(name);
        if (pt >= 0) { pt_param(pt, nullptr, host, bytes); return; }
        widen_particles();                         // the fp32 copies become the truth for one moment
        Dbm<float>::set_param(name, host, bytes);
        narrow_state();
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void get_param(const char* name, void* host, size_t bytes) override {
        if (offset_param(name, host, nullptr, bytes)) return;
        const int pt = pt_layer(name);
        if (pt >= 0) { pt_param(pt, host, nullptr, bytes); return; }
        widen_particles();
        Dbm<float>::get_param(name, host, bytes);
    }
    void init_particles(uint64_t seed) override {
        widen_particles();
        Dbm<float>::init_particles(seed);
        narrow_state();
        // tempered slots: the layers' initialisers at rows row0 + M .. row0 + T M - 1 (all layers Bernoulli: U[0, 1))
        if (T > 1) {
            const int rows = (T - 1) * M;
            DevBuf<float> tmp;
            for (int idx = 0; idx <= L; ++idx) {
                const int n = size_of(idx, V, Hs);
                tmp.ensure((size_t)rows * n);
                for (int r0 = 0; r0 < rows; r0 += 32768) {
                    const int r = std::min(32768, rows - r0);
                    particle_init_kernel<float><<<dim3(((n + 3) / 4 + 127) / 128, r), 128, 0, ctx->stream>>>(
                        tmp.p + (size_t)r0 * n, r, n, BM_UNIT_BERNOULLI, nullptr,
                        make_rng(seed, SITE_PARTICLE_INIT, idx, 0, particle_row0() + (uint32_t)M + (uint32_t)r0));
                    count_launch(ctx);
                }
                launch_f32_to_bf16(ctx, tmp.p, n, (idx == 0 ? v_b.p : h_b[idx - 1].p) + (size_t)M * ldn[idx], ldn[idx], rows, n);
                BM_CUDA(cudaStreamSynchronize(ctx->stream));          // tmp is reused by the next layer
            }
        }
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void pt_counts(int64_t* accepted, int64_t* proposed) override {
        BM_REQUIRE(T > 1, "this DBM has no tempered chains (bm_dbm_cfg.n_temps >= 2)");
        std::vector<unsigned long long> a(T - 1);
        BM_CUDA(cudaMemcpyAsync(a.data(), pt_accepted.p, (size_t)(T - 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        for (int m = 0; m + 1 < T; ++m) { accepted[m] = (int64_t)a[m]; proposed[m] = pt_proposed[m]; }
    }

    // ---- one fused conditional on the tensor cores -----------------------------------------------------------
    // act(acc_scale * (below W_i [+ above W_{i+1}^T]) + bias_scale * b_i): means XOR sampled states (bf16).  A multinomial
    // layer's op leaves x + b in pre_f32 and the row kernel writes `out` (and, given out_f32, the fp32 particles)
    void hidden_tc(int i, const bf16_t* below, const bf16_t* above, bf16_t* out, bool sample, int rows,
                   float acc_scale, float bias_scale, RngKey rng, float* out_f32 = nullptr) {
        launch_tc_gemm(ctx, hidden_gemm(i, below, above, out, sample, rows, acc_scale, bias_scale, rng));
        if (multinomial(i)) multinomial_rows(i, rows, out, out_f32, sample, rng);
    }
    void multinomial_rows(int i, int rows, bf16_t* out, float* out_f32, bool sample, RngKey rng) {
        const int n = (int)h_n_samples[i];
        launch_dbm_multinomial_rows(ctx, pre_f32.p, Hs[i], rows, Hs[i], (float)h_n_samples[i], sample ? n : 0, out, ldn[i + 1],
                                    out_f32, Hs[i], rng);
    }
    TcGemm hidden_gemm(int i, const bf16_t* below, const bf16_t* above, bf16_t* out, bool sample, int rows,
                       float acc_scale, float bias_scale, RngKey rng) {
        const int in = size_of(i, V, Hs), H = Hs[i];
        TcGemm g;
        g.M = rows; g.N = H;
        g.A[0] = mat(below, rows, in, ldn[i]); g.K[0] = in;
        g.B[0] = mat(Wb[i].p, in, H, ldn[i + 1]); g.b_t[0] = true;           // x W_i: W_i stored [K, N]
        if (above) above_pair(g, i, above, rows);
        g.acc_scale = acc_scale; g.bias_scale = bias_scale; g.bias = hb[i].p;
        if (multinomial(i)) { g.act = ACT_LINEAR; g.out_f32 = pre_f32.p; g.ld_f32 = H; return g; }     // layers.py:65-66
        g.act = ACT_SIGMOID; g.rng = rng;
        if (sample) { g.sample = SMP_BERNOULLI; g.out_state_bf = out; g.ld_state_bf = ldn[i + 1]; }
        else { g.out_mean_bf = out; g.ld_mean_bf = ldn[i + 1]; }
        return g;
    }
    void visible_tc(const bf16_t* h0, bf16_t* out, bool sample, int rows, RngKey rng) { launch_tc_gemm(ctx, visible_gemm(h0, out, sample, rows, rng)); }
    TcGemm visible_gemm(const bf16_t* h0, bf16_t* out, bool sample, int rows, RngKey rng) {
        TcGemm g;
        g.M = rows; g.N = V;
        g.A[0] = mat(h0, rows, Hs[0], ldn[1]); g.K[0] = Hs[0];
        g.B[0] = mat(Wb[0].p, V, Hs[0], ldn[1]); g.b_t[0] = false;            // h W_0^T: W_0 stored [N, K]
        g.bias = vb.p; g.rng = rng;
        if (v_kind == BM_UNIT_BERNOULLI) {
            g.act = ACT_SIGMOID;
            if (sample) g.sample = SMP_BERNOULLI;
        } else {                                                               // layers.py:84-89
            g.act = ACT_LINEAR; g.sigma = sigma.p;
            if (sample) { g.sample = SMP_GAUSSIAN; g.noise_sigma = sigma.p; }
        }
        if (sample) { g.out_state_bf = out; g.ld_state_bf = ldn[0]; }
        else { g.out_mean_bf = out; g.ld_mean_bf = ldn[0]; }
        return g;
    }
    // raw fp32 product A W_i (+ bias): the bound's t-terms and the AIS pre-activations
    void linear_tc(const bf16_t* A, int lda, int rows, int K, const bf16_t* Wsh, int w_rows, int w_cols, int ldw, bool b_t,
                   int N, const float* bias, float* out) {
        TcGemm g;
        g.M = rows; g.N = N;
        g.A[0] = mat(A, rows, K, lda); g.K[0] = K;
        g.B[0] = mat(Wsh, w_rows, w_cols, ldw); g.b_t[0] = b_t;
        g.bias = bias; g.act = ACT_LINEAR;
        g.out_f32 = out; g.ld_f32 = N;
        launch_tc_gemm(ctx, g);
    }

    // dbm.py:385-427 on bf16 operands.  Hn[i] receive the new hidden values (states when sampled, else means)
    void gibbs_tc(const bf16_t* vin, const std::vector<const bf16_t*>& Hin, const std::vector<bf16_t*>& Hn, bf16_t* v_new,
                  bool update_v, bool sample, int rows, uint64_t seed, uint32_t tstep, uint32_t tick, bool commit) {
        for (int i = 0; i < L; ++i) {
            const bf16_t* below = i == 0 ? vin : Hn[i - 1];
            const bf16_t* above = (i + 1 < L) ? Hin[i + 1] : nullptr;
            hidden_tc(i, below, above, Hn[i], sample && sample_h[i], rows, 1.f, 1.f, make_rng(seed, SITE_DBM_H + i, tstep, tick, particle_row0()),
                      commit ? h[i].p : nullptr);
        }
        if (update_v) visible_tc(Hn[0], v_new, sample && sample_vis, rows, make_rng(seed, SITE_DBM_V, tstep, tick, particle_row0()));
    }

    const float* upload_tc(const void* Xh, int rows) {
        const float* X = upload(Xh, rows);
        launch_f32_to_bf16(ctx, X, V, Xb.p, ldn[0], rows, V);
        return X;
    }

    // `ops` with dependencies as indices into it; row[k].layer >= 0: a row kernel follows op k.  A dependency on an op of an
    // earlier launch is dropped: the kernel boundary orders it.
    static void cut_chain(TcChain& chain, const std::vector<TcGemm>& ops, const std::vector<RowStep>& row) {
        size_t lo = 0;
        for (size_t k = 0; k < ops.size(); ++k) {
            if (row[k].layer < 0 && !row[k].cut && k + 1 < ops.size()) continue;
            std::unique_ptr<TcProgram> p(new TcProgram());
            for (size_t j = lo; j <= k; ++j) {
                TcGemm g = ops[j];
                int n = 0;
                for (int d = 0; d < g.n_deps; ++d)
                    if (g.dep[d] >= (int)lo) { g.dep[n] = g.dep[d] - (int)lo; g.dep_all[n] = g.dep_all[d]; ++n; }
                for (int d = n; d < g.n_deps; ++d) { g.dep[d] = -1; g.dep_all[d] = false; }
                g.n_deps = n;
                p->ops.push_back(g);
            }
            chain.progs.push_back(std::move(p));
            chain.after.push_back(row[k]);
            lo = k + 1;
        }
    }
    // the programs get `rng` (seed / tick / row0 shared by their ops); a sampling row kernel draws from (seed, site, t, tick)
    // at the same first row
    void run_chain(TcChain& chain, RngKey rng, uint64_t seed, uint32_t tick) {
        for (size_t k = 0; k < chain.progs.size(); ++k) {
            launch_tc_program(ctx, *chain.progs[k], rng, 0);
            const RowStep& st = chain.after[k];
            if (st.layer >= 0)
                multinomial_rows(st.layer, st.rows, st.out, st.out_f32, st.sample,
                                 st.sample ? make_rng(seed, st.site, st.t, tick, rng.row0) : RngKey{});
            if (st.clamp) launch_cdbm_clamp_labels(ctx, st.clamp, st.rows, Hs[st.layer], st.out, ldn[st.layer + 1]);
            if (st.vmask) launch_dbm_fill_clamp<bf16_t>(ctx, st.vmask, st.vx, ldn[0], st.vout, ldn[0], st.rows, V);
        }
    }

    // ---- E-step (dbm.py:429-478) ------------------------------------------------------------------------------
    // The E-step as persistent dataflow programs: `mf_chunk` sweeps (mf_chunk x L two-pair ops) per launch, every op
    // waiting per 256-row block on the ops it reads (layer i-1 of the same sweep, layer i+1 of the previous one) --
    // no kernel boundary and no host round trip between dependent sweeps.  The sweeps of a chunk are SPECULATED: every
    // sweep writes its own history slot, one kernel evaluates the chunk's convergence tests (dbm.py:449-452) afterwards
    // and the host picks the first sweep index that passed, so the result and n_mf_updates are those of the
    // sweep-by-sweep loop.  Slots: 0 = S_{a-1}, 1 = S_a, 2.. = S_{a+1}...; test t of the chunk compares slots t+1 and t.
    bf16_t* slot(int i, int s) { return hist[i].p + (size_t)s * B * ldn[i + 1]; }
    int mean_field_tc(int rows) {
        const int top = L - 1;
        const bool skip_top = mf_clamp == CLAMP_ALL;                         // the label layer's ops are not run
        if (mf_clamp != CLAMP_NONE) {        // labelled rows: e_t in the previous value and in every history slot
            launch_cdbm_clamp_labels(ctx, mf_labels, rows, Hs[top], mu_b[top].p, ldn[top + 1]);
            launch_cdbm_clamp_labels(ctx, mf_labels, rows, Hs[top], hist[top].p, ldn[top + 1], mf_chunk + 2, (size_t)B * ldn[top + 1]);
        }
        for (int i = 0; i < L; ++i) {                                        // approximate-inference pass -> slot 0
            const bf16_t* below = i == 0 ? Xb.p : slot(i - 1, 0);
            const float sc = (i == 0 || i < L - 1) ? 2.f : 1.f;
            if (!(skip_top && i == top)) hidden_tc(i, below, nullptr, slot(i, 0), false, rows, sc, 1.f, RngKey{});
            if (mf_clamp == CLAMP_ROWS && i == top) launch_cdbm_clamp_labels(ctx, mf_labels, rows, Hs[top], slot(top, 0), ldn[top + 1]);
            BM_CUDA(cudaMemcpyAsync(slot(i, 1), mu_b[i].p, (size_t)rows * ldn[i + 1] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        }
        int a = 0, result_slot = 1;
        bool done = false;
        while (!done && a < max_mf) {
            const int c = std::min(mf_chunk, max_mf - a);
            TcChain& chain = mf_progs[std::make_tuple(rows, c, mf_clamp)];
            if (chain.progs.empty()) {
                std::vector<TcGemm> ops;
                std::vector<RowStep> row;
                std::vector<int> prev(L, -1), cur(L, -1);                    // op indices of each layer in the last / this sweep
                for (int s = 1; s <= c; ++s) {                               // sweep s: slot s -> slot s + 1
                    for (int i = 0; i < L; ++i) {
                        if (skip_top && i == top) continue;
                        const bf16_t* below = i == 0 ? Xb.p : slot(i - 1, s + 1);
                        const bf16_t* above = (i + 1 < L) ? slot(i + 1, s) : nullptr;
                        TcGemm g = hidden_gemm(i, below, above, slot(i, s + 1), false, rows, 1.f, 1.f, RngKey{});
                        if (i > 0) { g.dep[g.n_deps] = cur[i - 1]; g.dep_all[g.n_deps] = false; ++g.n_deps; }                // layer i-1, this sweep
                        if (above && prev[i + 1] >= 0) { g.dep[g.n_deps] = prev[i + 1]; g.dep_all[g.n_deps] = false; ++g.n_deps; } // layer i+1, previous sweep
                        g.lane = LANE_CHAIN;
                        cur[i] = (int)ops.size();
                        ops.push_back(g);
                        RowStep st;
                        if (multinomial(i)) { st.layer = i; st.out = slot(i, s + 1); st.rows = rows; }
                        if (mf_clamp == CLAMP_ROWS && i == top) st.clamp = mf_labels;
                        row.push_back(st);
                    }
                    prev = cur;
                }
                cut_chain(chain, ops, row);
            }
            run_chain(chain, RngKey{}, 0, 0);
            BM_CUDA(cudaMemsetAsync(mf_flags.p, 0, (size_t)c * sizeof(unsigned int), ctx->stream));
            for (int i = 0; i < L; ++i) {
                if (skip_top && i == top) continue;                          // every slot holds the same one-hot rows
                mf_chunk_diffs_kernel<<<dim3((unsigned)(ctx->sm_count / 2), c), 256, 0, ctx->stream>>>(hist[i].p, (size_t)B * ldn[i + 1], ldn[i + 1], rows, Hs[i], mf_flags.p);
                count_launch(ctx);
            }
            allreduce_max_u32(ctx, mf_flags.p, (size_t)c);       // sharded rows: the same sweep index on every rank
            unsigned int bits[MF_CHUNK];
            BM_CUDA(cudaMemcpyAsync(bits, mf_flags.p, (size_t)c * sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
            int t = 0;
            for (; t < c; ++t) { float diff; memcpy(&diff, &bits[t], sizeof(diff)); if (!(diff > (float)mf_tol)) break; }   // :451-452
            if (t < c) { done = true; result_slot = t + 1; a += t; }
            else {
                a += c;
                result_slot = c + 1;
                if (a < max_mf)                                              // next chunk starts from S_{a-1}, S_a in slots 0, 1
                    for (int i = 0; i < L; ++i) {
                        const size_t bytes = (size_t)rows * ldn[i + 1] * sizeof(bf16_t);
                        BM_CUDA(cudaMemcpyAsync(slot(i, 0), slot(i, c), bytes, cudaMemcpyDeviceToDevice, ctx->stream));
                        BM_CUDA(cudaMemcpyAsync(slot(i, 1), slot(i, c + 1), bytes, cudaMemcpyDeviceToDevice, ctx->stream));
                    }
                if (a < max_mf) result_slot = 1;
            }
        }
        for (int i = 0; i < L; ++i)
            BM_CUDA(cudaMemcpyAsync(mu_b[i].p, slot(i, result_slot), (size_t)rows * ldn[i + 1] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        widen_mu(rows);                        // get_param('mu'), transform and the bound read the fp32 variables
        return a;
    }

    // ---- PCD particle update (dbm.py:480-509) -----------------------------------------------------------------
    // k committed sweeps of the persistent chains as one dataflow program: per sweep L hidden ops and the visible op,
    // each waiting per 256-row block on the ops it reads (for a single hidden layer this is the RBM chain of bm_rbm_tc.cu:
    // PCD-k on an RBM is the reference's DBM with one layer).  Ping-pong buffers: a buffer is overwritten two sweeps
    // after it was written, and every reader of the old value precedes the writer in the dependency chain.
    void particles_program(int n_steps, bool sample, uint64_t seed, uint32_t tick, int t0) {
        TcChain& chain = pcd_progs[std::make_tuple(n_steps, sample ? 1 : 0, t0)];
        std::vector<bf16_t*> cur(L), nxt(L);
        for (int i = 0; i < L; ++i) { cur[i] = h_b[i].p; nxt[i] = h2_b[i].p; }
        bf16_t* vc = v_b.p; bf16_t* vn = v2_b.p;
        const bool build = chain.progs.empty();
        std::vector<TcGemm> ops;
        std::vector<RowStep> row;
        int last_vis = -1;
        std::vector<int> last_h(L, -1), this_h(L, -1);
        for (int s = 0; s < n_steps; ++s) {
            if (build) {
                const uint32_t tstep = (uint32_t)(t0 + s + 1);
                for (int i = 0; i < L; ++i) {
                    const bf16_t* below = i == 0 ? vc : nxt[i - 1];
                    const bf16_t* above = (i + 1 < L) ? cur[i + 1] : nullptr;
                    TcGemm g = hidden_gemm(i, below, above, nxt[i], sample && sample_h[i], M, 1.f, 1.f, make_rng(0, SITE_DBM_H + i, tstep, 0, 0));
                    const int below_op = i == 0 ? last_vis : this_h[i - 1];
                    if (below_op >= 0) { g.dep[g.n_deps] = below_op; g.dep_all[g.n_deps] = false; ++g.n_deps; }
                    if (above && last_h[i + 1] >= 0) { g.dep[g.n_deps] = last_h[i + 1]; g.dep_all[g.n_deps] = false; ++g.n_deps; }
                    g.lane = LANE_CHAIN;
                    this_h[i] = (int)ops.size();
                    ops.push_back(g);
                    RowStep st;
                    if (multinomial(i)) {      // committed sweeps: the row kernel also writes the fp32 particles
                        st.layer = i; st.out = nxt[i]; st.out_f32 = h[i].p; st.rows = M; st.sample = sample && sample_h[i];
                        st.site = SITE_DBM_H + i; st.t = tstep;
                    }
                    row.push_back(st);
                }
                TcGemm gv = visible_gemm(nxt[0], vn, sample && sample_vis, M, make_rng(0, SITE_DBM_V, tstep, 0, 0));
                gv.dep[0] = this_h[0]; gv.dep_all[0] = false; gv.n_deps = 1;
                gv.lane = LANE_CHAIN;
                last_vis = (int)ops.size();
                ops.push_back(gv);
                row.push_back(RowStep());
                last_h = this_h;
            }
            std::swap(cur, nxt); std::swap(vc, vn);
        }
        if (build) cut_chain(chain, ops, row);
        run_chain(chain, make_rng(seed, 0, 0, tick, particle_row0()), seed, tick);
        for (int i = 0; i < L; ++i)
            if (cur[i] != h_b[i].p)
                BM_CUDA(cudaMemcpyAsync(h_b[i].p, cur[i], (size_t)M * ldn[i + 1] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        if (vc != v_b.p) BM_CUDA(cudaMemcpyAsync(v_b.p, vc, (size_t)M * ldn[0] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        particles_f32_stale = true;
    }

    // ---- parallel tempering (DESIGN.md §5.4) -------------------------------------------------------------------------
    // k committed sweeps of all T slots: per sweep and slot the ops of particles_program with acc_scale = bias_scale = beta_m,
    // reading and writing the slot's rows and drawing at rows row0 + m M + p (TcGemm::row_off).  Dependencies stay inside a
    // slot, and slot m runs on CTA pairs of its own (as the members of a training group), so the slots' ops run side by side.
    // Ops are listed sweep by sweep, layer by layer, slot by slot.  A chain longer than one program is cut between sweeps; a
    // single sweep of more than TC_PROGRAM_OPS ops (many slots) is cut every TC_PROGRAM_OPS ops, the kernel boundary then
    // ordering whatever depends across the cut.  Sweep s draws at t = t0 + s + 1.
    void particles_program_pt(int n_steps, bool sample, uint64_t seed, uint32_t tick, int t0) {
        TcChain& chain = pt_progs[std::make_tuple(n_steps, sample ? 1 : 0, t0)];
        std::vector<bf16_t*> cur(L), nxt(L);
        for (int i = 0; i < L; ++i) { cur[i] = h_b[i].p; nxt[i] = h2_b[i].p; }
        bf16_t* vc = v_b.p; bf16_t* vn = v2_b.p;
        if (chain.progs.empty()) {
            auto rows_of = [&](bf16_t* base, int idx, int m) { return base + (size_t)m * M * ldn[idx]; };
            const int total_pairs = ctx->sm_count / 2;
            int per = 0;                                               // CTA pairs of a slot: its largest op's units, at most 1/T of the grid
            std::vector<TcGemm> ops;
            std::vector<RowStep> row;
            std::vector<int> last_vis(T, -1);
            std::vector<std::vector<int>> last_h(T, std::vector<int>(L, -1)), this_h = last_h;
            const int sweep_ops = T * (L + 1);
            const int sweeps_per_launch = std::max(1, TC_PROGRAM_OPS / sweep_ops);
            for (int s = 0; s < n_steps; ++s) {
                const uint32_t tstep = (uint32_t)(t0 + s + 1);
                for (int i = 0; i <= L; ++i)
                    for (int m = 0; m < T; ++m) {
                        const float b = (float)betas[m];
                        TcGemm g;
                        if (i < L) {
                            const bf16_t* below = i == 0 ? rows_of(vc, 0, m) : rows_of(nxt[i - 1], i, m);
                            const bf16_t* above = (i + 1 < L) ? rows_of(cur[i + 1], i + 2, m) : nullptr;
                            g = hidden_gemm(i, below, above, rows_of(nxt[i], i + 1, m), sample && sample_h[i], M, b, b,
                                            make_rng(0, SITE_DBM_H + i, tstep, 0, 0));
                            const int below_op = i == 0 ? last_vis[m] : this_h[m][i - 1];
                            if (below_op >= 0) { g.dep[g.n_deps] = below_op; g.dep_all[g.n_deps] = false; ++g.n_deps; }
                            if (above && last_h[m][i + 1] >= 0) { g.dep[g.n_deps] = last_h[m][i + 1]; g.dep_all[g.n_deps] = false; ++g.n_deps; }
                            this_h[m][i] = (int)ops.size();
                        } else {
                            g = visible_gemm(rows_of(nxt[0], 1, m), rows_of(vn, 0, m), sample && sample_vis, M, make_rng(0, SITE_DBM_V, tstep, 0, 0));
                            g.acc_scale = b; g.bias_scale = b;
                            g.dep[0] = this_h[m][0]; g.dep_all[0] = false; g.n_deps = 1;
                            last_vis[m] = (int)ops.size();
                        }
                        g.row_off = (uint32_t)m * (uint32_t)M;
                        g.lane = LANE_CHAIN;
                        g.pair_begin = m;                                      // the slot, until the pair ranges are known
                        if (s == 0) per = std::max(per, tc_plan_units(ctx, g));
                        ops.push_back(g);
                        RowStep st;
                        if (sweep_ops <= TC_PROGRAM_OPS)                       // a launch ends with a whole sweep
                            st.cut = (i == L && m == T - 1 && (s + 1) % sweeps_per_launch == 0);
                        else                                                   // or with TC_PROGRAM_OPS ops of a long sweep
                            st.cut = (ops.size() % TC_PROGRAM_OPS == 0) || (i == L && m == T - 1);
                        row.push_back(st);
                    }
                for (int m = 0; m < T; ++m) last_h[m] = this_h[m];
                std::swap(cur, nxt); std::swap(vc, vn);
            }
            per = std::max(1, std::min(total_pairs / T, per));
            for (TcGemm& g : ops) { g.pair_begin = (g.pair_begin * per) % (total_pairs - per + 1); g.pair_count = per; }
            cut_chain(chain, ops, row);
        } else if (n_steps % 2) {
            std::swap(cur, nxt); std::swap(vc, vn);
        }
        run_chain(chain, make_rng(seed, 0, 0, tick, particle_row0()), seed, tick);
        const size_t TM = (size_t)T * M;
        for (int i = 0; i < L; ++i)
            if (cur[i] != h_b[i].p)
                BM_CUDA(cudaMemcpyAsync(h_b[i].p, cur[i], TM * ldn[i + 1] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        if (vc != v_b.p) BM_CUDA(cudaMemcpyAsync(v_b.p, vc, TM * ldn[0] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        particles_f32_stale = true;
    }
    // One swap round over the committed particles: the energies' products (one raw fp32 op per weight matrix over all T M rows),
    // then dbm_pt_swap_kernel.  The proposed pairs alternate with the call's tick: (m, m+1) with m = tick (mod 2).
    void pt_swap_round(uint64_t seed, uint32_t tick) {
        const int TM = T * M;
        PtSwapArgs a;
        memset(&a, 0, sizeof(a));
        a.L = L; a.T = T; a.M = M; a.V = V;
        a.x[0] = v_b.p; a.ld[0] = ldn[0];
        for (int i = 0; i < L; ++i) {
            const int in = size_of(i, V, Hs);
            linear_tc(i == 0 ? v_b.p : h_b[i - 1].p, ldn[i], TM, in, Wb[i].p, in, Hs[i], ldn[i + 1], true, Hs[i], hb[i].p, pt_pre[i].p);
            a.H[i] = Hs[i]; a.x[i + 1] = h_b[i].p; a.ld[i + 1] = ldn[i + 1]; a.P[i] = pt_pre[i].p;
        }
        a.vb = vb.p; a.betas = pt_betas.p;
        a.parity = (int)(tick & 1u);
        a.rng = make_rng(seed, SITE_DBM_PT, 0, tick, particle_row0());
        a.accepted = pt_accepted.p;
        dbm_pt_swap_kernel<<<M, 256, (size_t)T * (sizeof(double) + sizeof(int)), ctx->stream>>>(a);
        count_launch(ctx);
        for (int m = a.parity; m + 1 < T; m += 2) pt_proposed[m] += M;
        particles_f32_stale = true;
    }

    // committed sweeps that fit in one program run as that program; uncommitted runs (the second half of sample_v) and
    // longer chains take one launch per op.  With tempering, a committed update runs every slot (cut into launches between
    // sweeps when it is long) and ends with a swap round; an uncommitted run only needs slot 0, whose output it is.
    void particles_tc(int n_steps, bool sample, uint64_t seed, uint32_t tick, int t0, bool commit, bf16_t** v_final) {
        sv_k = 0;                                     // h2_b / v2_b are about to be overwritten
        if (commit && T > 1) {
            if (n_steps >= 1) particles_program_pt(n_steps, sample, seed, tick, t0);
            pt_swap_round(seed, tick);
            if (v_final) *v_final = v_b.p;
            return;
        }
        if (commit && n_steps >= 1 && n_steps * (L + 1) <= TC_PROGRAM_OPS) {
            particles_program(n_steps, sample, seed, tick, t0);
            if (v_final) *v_final = v_b.p;
            return;
        }
        std::vector<bf16_t*> cur(L), nxt(L), spare(L);
        for (int i = 0; i < L; ++i) { cur[i] = h_b[i].p; nxt[i] = h2_b[i].p; spare[i] = nullptr; }
        bf16_t* vc = v_b.p; bf16_t* vn = v2_b.p; bf16_t* vspare = nullptr;
        if (!commit) {      // an uncommitted run must never write the persistent particles: ping-pong on scratch
            v3_b.ensure((size_t)M * ldn[0]); vspare = v3_b.p;
            for (int i = 0; i < L; ++i) { h3_b[i].ensure((size_t)M * ldn[i + 1]); spare[i] = h3_b[i].p; }
        }
        for (int s = 0; s < n_steps; ++s) {
            std::vector<const bf16_t*> Hin(cur.begin(), cur.end());
            gibbs_tc(vc, Hin, nxt, vn, true, sample, M, seed, (uint32_t)(t0 + s + 1), tick, commit);
            if (!commit && s == 0) { cur = nxt; nxt = spare; vc = vn; vn = vspare; }
            else { std::swap(cur, nxt); std::swap(vc, vn); }
        }
        if (commit) {
            for (int i = 0; i < L; ++i)
                if (cur[i] != h_b[i].p)
                    BM_CUDA(cudaMemcpyAsync(h_b[i].p, cur[i], (size_t)M * ldn[i + 1] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
            if (vc != v_b.p) BM_CUDA(cudaMemcpyAsync(v_b.p, vc, (size_t)M * ldn[0] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
            if (n_steps > 0) particles_f32_stale = true;
            if (v_final) *v_final = v_b.p;
        } else if (v_final) *v_final = vc;
    }

    void reconstruction_tc(int rows) {                                        // :626-628; fp32 copy in `recon`
        visible_tc(mu_b[0].p, recon_b.p, false, rows, RngKey{});
        launch_bf16_to_f32(ctx, recon_b.p, ldn[0], recon.p, V, rows, V);
    }
    double msre_tc(const float* X, int rows) {
        reconstruction_tc(rows);
        launch_sqdiff_mean<float>(ctx, X, V, recon.p, V, rows, V, (double)rows * V, scal.p);
        double hval = 0.0;
        BM_CUDA(cudaMemcpyAsync(&hval, scal.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        return allreduce_mean(hval);
    }

    // G_i = pos^T mu_i / N - neg^T h_i / M (dbm.py:558-568): two split-K tensor-core GEMMs over the rows
    void gradient_tc(int i, const bf16_t* pos, int pos_rows, const bf16_t* neg, float n_div, float m_div) {
        const int in = size_of(i, V, Hs), H = Hs[i];
        const int total_pairs = ctx->sm_count / 2;
        const int pair_tiles = ((in + 255) / 256) * ((H + 255) / 256);
        auto splits_for = [&](int rows) { return std::max(1, std::min(total_pairs / std::max(pair_tiles, 1), (rows + 63) / 64)); };
        const int sp = splits_for(pos_rows), sn = splits_for(M);
        const size_t stride = (size_t)in * H;
        Gp[i].ensure((size_t)(sp + sn) * stride);
        auto half = [&](const bf16_t* a, const bf16_t* b, int rows, int splits, float* out) {
            TcGemm g;
            g.M = in; g.N = H;
            g.A[0] = mat(a, rows, in, ldn[i]); g.a_t[0] = true;               // stored [K = rows, M = in]
            g.B[0] = mat(b, rows, H, ldn[i + 1]); g.b_t[0] = true;            // stored [K = rows, N = H]
            g.K[0] = rows;
            g.splits = splits; g.split_stride = stride;
            g.out_f32 = out; g.ld_f32 = H;
            launch_tc_gemm(ctx, g);
        };
        half(pos, mu_b[i].p, pos_rows, sp, Gp[i].p);
        half(neg, h_b[i].p, M, sn, Gp[i].p + (size_t)sp * stride);
        if (centering)
            dbm_centered_grad_combine_kernel<<<592, 256, 0, ctx->stream>>>(
                Gp[i].p, sp, Gp[i].p + (size_t)sp * stride, sn, stride, 1.0f / n_div, 1.0f / m_div, H, off[oc][i].p, cen_s[i].p,
                off[oc][i + 1].p, cen_s[i + 1].p, (float)((double)pos_rows / (double)n_div - 1.0), G[i].p, stride);
        else
            dbm_grad_combine_kernel<<<592, 256, 0, ctx->stream>>>(Gp[i].p, sp, Gp[i].p + (size_t)sp * stride, sn, stride,
                                                                  1.0f / n_div, 1.0f / m_div, G[i].p, stride);
        count_launch(ctx);
    }

    // centering: s_j and (first step) the offsets from the step's column sums, the moved offsets into off[1 - oc]
    void center_stats(int rows, float N, float Mp) {
        CenterArgs a;
        memset(&a, 0, sizeof(a));
        a.n_layers = L + 1;
        int nmax = 0;
        for (int j = 0; j <= L; ++j) {
            a.n[j] = size_of(j, V, Hs); nmax = std::max(nmax, a.n[j]);
            a.dsum[j] = j == 0 ? xsum.p : musum[j - 1].p;
            a.psum[j] = j == 0 ? vsum.p : hsum[j - 1].p;
            a.o[j] = off[oc][j].p; a.o_next[j] = off[1 - oc][j].p; a.s[j] = cen_s[j].p;
        }
        a.rows = (float)rows; a.inv_n = 1.0f / N; a.inv_m = 1.0f / Mp;
        a.keep = (float)(1.0 - (double)offset_rate); a.rate = offset_rate;
        a.init = offsets_set ? 0 : 1;
        dbm_center_stats_kernel<<<dim3((nmax + 255) / 256, L + 1), 256, 0, ctx->stream>>>(a);
        count_launch(ctx);
        offsets_set = true;
    }
    // centering: mode 0 stores c_j of the current W and offsets; mode 1 takes the change of c_j out of b_j
    void coupling(int mode) {
        CouplingArgs a;
        memset(&a, 0, sizeof(a));
        a.n_layers = L + 1;
        int nmax = 0;
        for (int j = 0; j <= L; ++j) {
            a.n[j] = size_of(j, V, Hs); nmax = std::max(nmax, a.n[j]);
            if (j < L) a.W[j] = W[j].p;
            a.o[j] = off[oc][j].p; a.cpl[j] = cpl[j].p; a.b[j] = j == 0 ? vb.p : hb[j - 1].p;
        }
        a.mode = mode;
        dbm_coupling_kernel<<<dim3((nmax + 31) / 32, L + 1), dim3(32, 8), 0, ctx->stream>>>(a);
        count_launch(ctx);
    }

    void train_step(const void* Xh, int rows, double lr, double mom, int k, uint64_t seed, uint32_t tick, int want, double* out) override {
        BM_REQUIRE(rows >= 1, "empty batch");
        const float* X = upload_tc(Xh, rows);
        const int n_mf = mean_field_tc(rows);
        particles_tc(k, true, seed, tick, 0, true, nullptr);
        if (want) { BM_REQUIRE(out, "metrics requested without a buffer"); out[0] = msre_tc(X, rows); out[1] = (double)n_mf; }
        const int nr = nranks();                               // data parallelism: see the header of bm_dbm.cu
        const float N = (float)((double)B * nr), Mp = (float)((double)M * nr);      // configured (global) sizes (dbm.py:254-255)
        const float rows_g = (float)((double)rows * nr);
        // column sums of mu_i (over the batch rows) and of h_i, v (over the particles), three per pair of launches; X over the rows.
        // A centered step reads them in its gradients' combine, so they go first there.
        auto column_sums = [&]() {
            std::vector<const bf16_t*> P; std::vector<int> ld, nc; std::vector<float*> out;
            auto flush = [&](int nrows) {
                for (size_t o = 0; o < P.size(); o += 3) {
                    const int n = (int)std::min<size_t>(3, P.size() - o);
                    launch_colsums_bf16(ctx, n, P.data() + o, ld.data() + o, nc.data() + o, out.data() + o, nrows);
                }
                P.clear(); ld.clear(); nc.clear(); out.clear();
            };
            for (int i = 0; i < L; ++i) { P.push_back(mu_b[i].p); ld.push_back(ldn[i + 1]); nc.push_back(Hs[i]); out.push_back(musum[i].p); }
            flush(rows);
            for (int i = 0; i < L; ++i) { P.push_back(h_b[i].p); ld.push_back(ldn[i + 1]); nc.push_back(Hs[i]); out.push_back(hsum[i].p); }
            P.push_back(v_b.p); ld.push_back(ldn[0]); nc.push_back(V); out.push_back(vsum.p);
            flush(M);
            launch_colsum<float>(ctx, X, V, (const float*)nullptr, 0, rows, V, 1.f, 0.f, xsum.p);
        };
        if (centering) {
            column_sums();
            center_stats(rows, N, Mp);
            coupling(0);
        }
        for (int i = 0; i < L; ++i) gradient_tc(i, i == 0 ? Xb.p : mu_b[i - 1].p, rows, i == 0 ? v_b.p : h_b[i - 1].p, N, Mp);
        if (!centering) column_sums();
        allreduce_step_statistics();
        dbm_vbias_kernel<float><<<(V + 255) / 256, 256, 0, ctx->stream>>>(V, xsum.p, vsum.p, rows_g, Mp, vb.p, dvb.p, (float)lr, (float)mom);
        count_launch(ctx);
        for (int i = 0; i < L; ++i) {
            const int in = size_of(i, V, Hs), H = Hs[i];
            if (top_is_label && i == L - 1) {      // yb: sum q(y) / rows - sum y / M, the plain momentum update (pen stays 0)
                dbm_vbias_kernel<float><<<(H + 255) / 256, 256, 0, ctx->stream>>>(H, musum[i].p, hsum[i].p, rows_g, Mp, hb[i].p, dhb[i].p,
                                                                                 (float)lr, (float)mom);
            } else {
                BM_REQUIRE(i < H, "the reference's sparsity update indexes element i of layer i's unit vector");
                dbm_sparsity_bias_kernel<float><<<(H + 255) / 256, 256, 0, ctx->stream>>>(
                    H, i, musum[i].p, hsum[i].p, rows_g, Mp, qm[i].p, mm[i].p, pen[i].p, hb[i].p, dhb[i].p,
                    (float)damping, (float)sp_cost[i], (float)sp_target[i], (float)lr, (float)mom);
            }
            count_launch(ctx);
            launch_weight_update<float>(ctx, G[i].p, H, 1.f, W[i].p, dW[i].p, in, H, pen[i].p, (float)l2, (float)lr, (float)mom, nullptr, 0);
            colnorm_kernel<float><<<(H + 31) / 32, dim3(32, 8), 0, ctx->stream>>>(W[i].p, in, H, norm[i].p);       // :511-513
            count_launch(ctx);
            max_norm_scale_kernel<float><<<dim3((H + 255) / 256, in < 32768 ? in : 32768), 256, 0, ctx->stream>>>(W[i].p, in, H, norm[i].p, (float)max_norm);
            count_launch(ctx);
            refresh_shadow(i);
        }
        if (centering) {          // b_j = a_j - c_j with the new W and the step's offsets; then the moved offsets
            coupling(1);
            oc = 1 - oc;
        }
    }

    void val_metrics(const void* Xh, int rows, int k, uint64_t seed, uint32_t tick, double* out) override {
        const float* X = upload_tc(Xh, rows);
        const int n_mf = mean_field_tc(rows);
        particles_tc(k, true, seed, tick, 0, true, nullptr);                  // dbm.py:523 control dependencies
        out[0] = msre_tc(X, rows); out[1] = (double)n_mf;
    }
    void transform(const void* Xh, int rows, void* out) override {
        upload_tc(Xh, rows);
        mean_field_tc(rows);
        BM_CUDA(cudaMemcpyAsync(out, mu[L - 1].p, (size_t)rows * Hs[L - 1] * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void reconstruct(const void* Xh, int rows, void* out) override {
        upload_tc(Xh, rows);
        mean_field_tc(rows);
        reconstruction_tc(rows);
        BM_CUDA(cudaMemcpyAsync(out, recon.p, (size_t)rows * V * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void log_proba(const void* Xh, int rows, double* out) override {
        if (L != 2) { log_proba_layers(Xh, rows, out); return; }
        BM_REQUIRE(!multinomial(0) && !multinomial(1), "log_proba is defined for binary hidden layers (dbm.py:946-948)");
        const float* X = upload_tc(Xh, rows);
        mean_field_tc(rows);
        linear_tc(Xb.p, ldn[0], rows, V, Wb[0].p, V, Hs[0], ldn[1], true, Hs[0], nullptr, t[0].p);              // t1 = X W_0
        linear_tc(mu_b[0].p, ldn[1], rows, Hs[0], Wb[1].p, Hs[0], Hs[1], ldn[2], true, Hs[1], nullptr, t[1].p); // t2 = mu_0 W_1
        dbm_bound_rows_kernel<float><<<(rows + 7) / 8, dim3(32, 8), 0, ctx->stream>>>(X, V, mu[0].p, Hs[0], mu[1].p, Hs[1], t[0].p, t[1].p,
                                                                                     vb.p, hb[0].p, hb[1].p, rows, rowd.p);
        count_launch(ctx);
        BM_CUDA(cudaMemcpyAsync(out, rowd.p, (size_t)rows * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    // AIS and the bound at a depth other than 2 (DESIGN.md §5.4c), and AIS from a base-rate model at any depth (§5.4d), are
    // defined for binary layers; the AIS ladder's state ops also take their linear term from sampled states, so the odd layers
    // h_1, h_3, ... must be sampled
    void depth_check(bool ais, bool base = false) const {
        const std::string what = base ? std::string("AIS from a base-rate model")
                                      : std::string(ais ? "AIS" : "log_proba") + " at " + std::to_string(L) + " hidden layers";
        bool binary = v_kind == BM_UNIT_BERNOULLI;
        for (int i = 0; i < L; ++i) binary = binary && h_kinds[i] == BM_UNIT_BERNOULLI;
        if (!binary) throw Error(BM_EUNSUPPORTED, what + " is defined for binary layers (Bernoulli visible and hidden units)");
        for (int i = 0; ais && i < L; i += 2)
            if (!sample_h[i]) throw Error(BM_EUNSUPPORTED, what + " needs sampled states in the odd layers h_1, h_3, ... (sample_h)");
    }
    // dbm.py:743-757 for L hidden layers: t_i = mu_{i-1} W_i (X W_0 for i = 0) on the tensor cores, then the row kernel
    void log_proba_layers(const void* Xh, int rows, double* out) {
        depth_check(false);
        const float* X = upload_tc(Xh, rows);
        mean_field_tc(rows);
        for (int i = 0; i < L; ++i) {
            const int in = size_of(i, V, Hs);
            linear_tc(i == 0 ? Xb.p : mu_b[i - 1].p, ldn[i], rows, in, Wb[i].p, in, Hs[i], ldn[i + 1], true, Hs[i], nullptr, t[i].p);
        }
        for (int i = 0; i < L; ++i) {
            dbm_bound_layer_rows_kernel<<<(rows + 7) / 8, dim3(32, 8), 0, ctx->stream>>>(X, V, vb.p, mu[i].p, t[i].p, hb[i].p, Hs[i],
                                                                                       i == 0 ? 1 : 0, rows, rowd.p);
            count_launch(ctx);
        }
        BM_CUDA(cudaMemcpyAsync(out, rowd.p, (size_t)rows * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void sample_v(int k, uint64_t seed, uint32_t tick, void* out) override {
        // dbm.py:641-648: k sampled sweeps (committed), k more without sampling; v <- their visible means
        particles_tc(k, true, seed, tick, 0, true, nullptr);
        bf16_t* vf = nullptr;
        particles_tc(k, false, seed, tick, k, false, &vf);
        if (vf != v_b.p) BM_CUDA(cudaMemcpyAsync(v_b.p, vf, (size_t)M * ldn[0] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        particles_f32_stale = true;
        widen_particles();
        BM_CUDA(cudaMemcpyAsync(out, v.p, (size_t)M * V * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        sv_k = k;
    }
    // as Dbm<T>::sample_v_debug on the bf16 ping-pong (h2_b / v2_b for odd sweeps, h3_b / v3_b for even ones; slot 0's rows),
    // as bf16 bit patterns
    void sample_v_debug(const char* name, void* host, size_t bytes) override {
        BM_REQUIRE(sv_k > 0, "sample_v_debug: no uncommitted sample_v sweep since the last particle update");
        std::string n(name);
        int t = sv_k;
        const std::string suffix = "_prev";
        if (n.size() > suffix.size() && n.compare(n.size() - suffix.size(), suffix.size(), suffix) == 0) {
            n = n.substr(0, n.size() - suffix.size()); --t;
        }
        BM_REQUIRE(t >= 1, "sample_v_debug: the sweep before the first uncommitted one is the committed particles (get_param)");
        const bool odd = (t & 1) != 0;
        const bf16_t* src = nullptr; int width = 0, ld = 0;
        if (n == "v") { src = odd ? v2_b.p : v3_b.p; width = V; ld = ldn[0]; }
        else
            for (int i = 0; i < L; ++i)
                if (n == "h" + sfx(i)) { src = odd ? h2_b[i].p : h3_b[i].p; width = Hs[i]; ld = ldn[i + 1]; }
        BM_REQUIRE(src, std::string("sample_v_debug: unknown name '") + name + "'");
        BM_REQUIRE(bytes == (size_t)M * width * sizeof(bf16_t), std::string("sample_v_debug: size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpy2DAsync(host, (size_t)width * sizeof(bf16_t), src, (size_t)ld * sizeof(bf16_t), (size_t)width * sizeof(bf16_t),
                                  M, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // ---- clamped Gibbs chains (DESIGN.md §5.9) ---------------------------------------------------------------------------
    // The chain of particles_program on scratch of its own: index t % 2 of fv_b / fh_b holds sweep t (0: the start).  A sweep is
    // L hidden ops and the visible op, cut after the visible op for the clamp (dbm_fill_clamp_kernel blends the batch's bf16
    // operand into v under the mask), so every sweep is one program launch -- plus the row kernels of multinomial layers and,
    // on a classification DBM with labelled rows, the label clamp after the label's row kernel.  The last sweep also computes
    // the visible means p(v | h_1) (one more op in its program).  Programs are cached by (rows, sweeps, label clamp).
    DevBuf<float> fX_f, fout_f;
    DevBuf<bf16_t> fXb, fmean_b, fv_b[2];
    std::vector<DevBuf<bf16_t>> fh_b[2];
    DevBuf<uint8_t> fmask_d;
    DevBuf<int> flab;
    std::map<std::tuple<int, int, int>, TcChain> fill_progs;
    void fill(const void* Xh, const uint8_t* mask, const int32_t* labels, int rows, uint32_t row0, int k, uint64_t seed,
              uint32_t tick, void* out) override {
        check_fill_args(mask, labels, rows, k, B, V, top_is_label ? Hs[L - 1] : 0);
        int labelled = 0;
        if (labels) for (int r = 0; r < rows; ++r) labelled += labels[r] >= 0;
        if (fh_b[0].empty()) {
            fX_f.ensure((size_t)B * V); fout_f.ensure((size_t)B * V); fmask_d.ensure((size_t)B * V);
            for (DevBuf<bf16_t>* b : {&fXb, &fmean_b, &fv_b[0], &fv_b[1]}) { b->ensure((size_t)B * ldn[0]); b->zero(ctx->stream); }
            for (int s = 0; s < 2; ++s) {
                fh_b[s].resize(L);
                for (int i = 0; i < L; ++i) { fh_b[s][i].ensure((size_t)B * ldn[i + 1]); fh_b[s][i].zero(ctx->stream); }
            }
            if (top_is_label) flab.ensure(B);
        }
        f_rows = 0;
        BM_CUDA(cudaMemcpyAsync(fX_f.p, Xh, (size_t)rows * V * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        BM_CUDA(cudaMemcpyAsync(fmask_d.p, mask, (size_t)rows * V, cudaMemcpyHostToDevice, ctx->stream));
        if (labelled) BM_CUDA(cudaMemcpyAsync(flab.p, labels, (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        launch_f32_to_bf16(ctx, fX_f.p, V, fXb.p, ldn[0], rows, V);
        // start: v0 = X where observed, act(0 W_0' + b) elsewhere; h0 from the E-step's approximate-inference pass (dbm.py:434-446)
        BM_CUDA(cudaMemsetAsync(fh_b[1][0].p, 0, (size_t)rows * ldn[1] * sizeof(bf16_t), ctx->stream));
        visible_tc(fh_b[1][0].p, fv_b[0].p, false, rows, RngKey{});
        launch_dbm_fill_clamp<bf16_t>(ctx, fmask_d.p, fXb.p, ldn[0], fv_b[0].p, ldn[0], rows, V);
        for (int i = 0; i < L; ++i) {
            const float sc = (i == 0 || i < L - 1) ? 2.f : 1.f;
            hidden_tc(i, i == 0 ? fv_b[0].p : fh_b[0][i - 1].p, nullptr, fh_b[0][i].p, false, rows, sc, 1.f, RngKey{});
            if (labelled && top_is_label && i == L - 1) launch_cdbm_clamp_labels(ctx, flab.p, rows, Hs[i], fh_b[0][i].p, ldn[i + 1]);
        }
        TcChain& chain = fill_progs[std::make_tuple(rows, k, labelled ? 1 : 0)];
        if (chain.progs.empty()) {
            std::vector<TcGemm> ops;
            std::vector<RowStep> row;
            for (int t = 1; t <= k; ++t) {
                const int c = (t - 1) & 1, n = t & 1;
                int prev = -1, first = -1;                       // this sweep's op of layer i - 1 / of layer 0
                for (int i = 0; i < L; ++i) {
                    const bf16_t* below = i == 0 ? fv_b[c].p : fh_b[n][i - 1].p;
                    const bf16_t* above = (i + 1 < L) ? fh_b[c][i + 1].p : nullptr;
                    TcGemm g = hidden_gemm(i, below, above, fh_b[n][i].p, sample_h[i] != 0, rows, 1.f, 1.f,
                                           make_rng(0, SITE_DBM_H + i, (uint32_t)t, 0, 0));
                    if (prev >= 0) { g.dep[g.n_deps] = prev; g.dep_all[g.n_deps] = false; ++g.n_deps; }
                    g.lane = LANE_CHAIN;
                    prev = (int)ops.size();
                    if (i == 0) first = prev;
                    ops.push_back(g);
                    RowStep st;
                    if (multinomial(i)) {
                        st.layer = i; st.out = fh_b[n][i].p; st.rows = rows; st.sample = sample_h[i] != 0;
                        st.site = SITE_DBM_H + i; st.t = (uint32_t)t;
                    }
                    if (labelled && top_is_label && i == L - 1) st.clamp = flab.p;
                    row.push_back(st);
                }
                TcGemm gv = visible_gemm(fh_b[n][0].p, fv_b[n].p, sample_vis != 0, rows, make_rng(0, SITE_DBM_V, (uint32_t)t, 0, 0));
                gv.dep[0] = first; gv.dep_all[0] = false; gv.n_deps = 1;
                gv.lane = LANE_CHAIN;
                ops.push_back(gv);
                row.push_back(RowStep());
                if (t == k) {                                    // p(v | h_1) of the last sweep
                    TcGemm gm = visible_gemm(fh_b[n][0].p, fmean_b.p, false, rows, RngKey{});
                    gm.dep[0] = first; gm.dep_all[0] = false; gm.n_deps = 1;
                    gm.lane = LANE_CHAIN;
                    ops.push_back(gm);
                    row.push_back(RowStep());
                }
                RowStep& end = row.back();                       // the visible clamp ends the sweep's launch
                end.vmask = fmask_d.p; end.vx = fXb.p; end.vout = fv_b[n].p; end.rows = rows; end.cut = true;
            }
            cut_chain(chain, ops, row);
        }
        run_chain(chain, make_rng(seed, 0, 0, tick, row0), seed, tick);
        launch_dbm_fill_out<bf16_t, float>(ctx, fmask_d.p, fX_f.p, fmean_b.p, ldn[0], fout_f.p, rows, V);
        BM_CUDA(cudaMemcpyAsync(out, fout_f.p, (size_t)rows * V * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        f_rows = rows; f_k = k;
    }
    // as Dbm<T>::fill_debug, as bf16 bit patterns; on a classification DBM the label layer is "y" / "y_prev"
    void fill_debug(const char* name, void* host, size_t bytes) override {
        BM_REQUIRE(f_rows > 0, "fill_debug: no fill has run on this DBM");
        std::string n(name);
        int which = f_k & 1;
        const std::string suffix = "_prev";
        if (n.size() > suffix.size() && n.compare(n.size() - suffix.size(), suffix.size(), suffix) == 0) {
            n = n.substr(0, n.size() - suffix.size()); which = 1 - which;
        }
        const bf16_t* src = nullptr; int width = 0, ld = 0;
        if (n == "v") { src = fv_b[which].p; width = V; ld = ldn[0]; }
        else if (n == "mean" && std::string(name) == "mean") { src = fmean_b.p; width = V; ld = ldn[0]; }
        else
            for (int i = 0; i < L; ++i) {
                const bool label = top_is_label && i == L - 1;
                if (n == (label ? std::string("y") : "h" + sfx(i))) { src = fh_b[which][i].p; width = Hs[i]; ld = ldn[i + 1]; }
            }
        BM_REQUIRE(src, std::string("fill_debug: unknown name '") + name + "'");
        BM_REQUIRE(bytes == (size_t)f_rows * width * sizeof(bf16_t), std::string("fill_debug: size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpy2DAsync(host, (size_t)width * sizeof(bf16_t), src, (size_t)ld * sizeof(bf16_t), (size_t)width * sizeof(bf16_t),
                                  f_rows, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // ---- AIS (dbm.py:650-736) -------------------------------------------------------------------------------------
    // Per temperature: 2 tensor-core GEMMs for the shared pre-activations (x W_0^T + b, x W_1 + c_2; fp32 out),
    // one pass that adds log p*_{i+1}(x) - log p*_i(x) of the same x to the chain's fp64 log-weight, two unit
    // kernels (v, h2) and ONE two-pair tensor-core op for x' = act(beta (v W_0 + h2 W_1^T) + beta c_1) with the
    // Bernoulli draw in its epilogue.
    // (sharding over ranks / calls: Dbm<float>::ais, ais_rows; run r draws from row row0 + r of the AIS sites)
    // AIS with everything but the GEMMs' operands kept out of memory: per temperature step THREE tensor-core ops whose
    // epilogues do the rest (TcPhaseLite::ais_kind) --
    //   U_v : z = x W_0^T + b   -> logw += sum softplus(beta_i z) - softplus(beta_{i-1} z);  v  ~ sigmoid(beta_{i+1} z)
    //   U_h2: z = x W_1 + c_2   -> logw += ...                                               h2 ~ sigmoid(beta_{i+1} z)
    //   T   : x' ~ sigmoid(beta_{i+1} (v W_0 + h2 W_1^T + c_1))   -> logw += (beta_{i+1} - beta_i) x'.c_1
    // -- "the same kernel with a scalar beta multiplied into the pre-activation" (north_star).  The fp32 pre-activations
    // (145 MB per step at 20 000 runs) never exist; up to 30 steps run as one persistent dataflow launch, every op waiting
    // per 256-run block on the op(s) it reads.  dbm.py:650-736; same draws (sites, ticks, rows) as the kernel-per-pass variant.
    void ais_local(int R, uint32_t row0, int n_betas, int k, uint64_t seed, const float* const* base, double* logw_out) override {
        if (L != 2 || has_base(base)) { ais_local_layers(R, row0, n_betas, k, seed, base, logw_out); return; }
        // the transition's epilogue takes the linear term from sampled states
        if (!sample_h[0]) { ais_local_passes(R, row0, n_betas, k, seed, logw_out); return; }
        const int H0 = Hs[0], H1 = Hs[1];
        const int ld0 = ldn[1], ldv = ldn[0], ld1 = ldn[2];
        DevBuf<bf16_t> x, xn, va, hc;
        x.ensure((size_t)R * ld0); xn.ensure((size_t)R * ld0); va.ensure((size_t)R * ldv); hc.ensure((size_t)R * ld1);
        for (DevBuf<bf16_t>* b : {&x, &xn, &va, &hc}) b->zero(ctx->stream);
        bf16_t* xc = x.p; bf16_t* xo = xn.p;
        {   // x_0 ~ Ber(1/2)   (:700-702)
            dim3 g(((H0 + 3) / 4 + 127) / 128, R);
            ais_unit_bf16_kernel<<<g, 128, 0, ctx->stream>>>(nullptr, 0, 0.f, xc, ld0, R, H0, 1, make_rng(seed, SITE_AIS_INIT, 0, 0, row0));
            count_launch(ctx);
        }
        // the temperatures of the transitions, accumulated in the storage dtype like the reference's loop (:710-711)
        const float delta = (float)(1.0 / n_betas);
        std::vector<float> t;
        t.push_back(delta);
        while (t.back() < 1.f - delta + 1e-5f) t.push_back(t.back() + delta);
        const int nT = (int)t.size();                                    // transition j (at t[j]) produces x_{j+1}
        auto inc_a = [&](int j) { return j == 0 ? 0.f : t[j - 1]; };       // x_{j+1} is weighted with log p_b - log p_a
        auto inc_b = [&](int j) { return j == nT - 1 ? 1.0f : t[j]; };
        std::vector<TcGemm> all;
        std::vector<int> dep0, dep1;                                      // global producer indices (-1: none)
        int last_T = -1;
        auto unit_op = [&](bool vis, const bf16_t* xs, float a, float b, bool weigh, float next, bool emit, uint32_t tick) {
            TcGemm g;
            g.M = R; g.N = vis ? V : H1;
            g.A[0] = mat(xs, R, H0, ld0); g.K[0] = H0;
            if (vis) { g.B[0] = mat(Wb[0].p, V, H0, ld0); g.b_t[0] = false; g.bias = vb.p; }           // x W_0^T: W_0 stored [N, K]
            else { g.B[0] = mat(Wb[1].p, H0, H1, ld1); g.b_t[0] = true; g.bias = hb[1].p; }             // x W_1:   W_1 stored [K, N]
            g.act = ACT_LINEAR;
            g.ais_kind = 1; g.ais_a = a; g.ais_b = b; g.ais_next = next; g.ais_logw = weigh ? logw_out : nullptr;
            g.tick_off = tick;
            if (emit) {
                const bool smp = vis ? sample_vis : (sample_h[1] != 0);
                g.sample = smp ? SMP_BERNOULLI : SMP_NONE;
                g.out_state_bf = vis ? va.p : hc.p; g.ld_state_bf = vis ? ldv : ld1;
                g.rng = make_rng(0, vis ? SITE_AIS_V : SITE_AIS_H2, 0, 0, 0);
            }
            all.push_back(g); dep0.push_back(last_T); dep1.push_back(-1);
            return (int)all.size() - 1;
        };
        for (int j = 0; j < nT; ++j) {
            for (int sw = 0; sw < k; ++sw) {
                const uint32_t tick = (uint32_t)(j * k + sw);
                const bool weigh = sw == 0 && j >= 1;                     // the increment of x_j (produced by transition j-1)
                const float a = weigh ? inc_a(j - 1) : 0.f, b = weigh ? inc_b(j - 1) : 0.f;
                const int ua = unit_op(true, xc, a, b, weigh, t[j], true, tick);
                const int ub = unit_op(false, xc, a, b, weigh, t[j], true, tick);
                TcGemm o;                                                 // x' = act(beta (v W_0 + h2 W_1^T), beta c_1)
                o.M = R; o.N = H0;
                o.A[0] = mat(va.p, R, V, ldv); o.K[0] = V; o.B[0] = mat(Wb[0].p, V, H0, ld0); o.b_t[0] = true;
                above_pair(o, 0, hc.p, R);
                o.acc_scale = t[j]; o.bias_scale = t[j]; o.bias = hb[0].p; o.act = ACT_SIGMOID;
                o.sample = SMP_BERNOULLI; o.out_state_bf = xo; o.ld_state_bf = ld0;
                o.rng = make_rng(0, SITE_AIS_H1, 0, 0, 0);
                o.tick_off = tick;
                o.ais_kind = 2;
                if (sw == k - 1) {
                    o.ais_logw = logw_out;
                    o.ais_lin = (float)(((double)inc_b(j) - (double)inc_a(j)) / ((double)t[j] * -1.4426950408889634));
                }
                all.push_back(o); dep0.push_back(ua); dep1.push_back(ub);
                last_T = (int)all.size() - 1;
                std::swap(xc, xo);
            }
        }
        unit_op(true, xc, inc_a(nT - 1), inc_b(nT - 1), true, 0.f, false, 0);      // + log p_M(x_M) - log p_{M-1}(x_M)   :728
        unit_op(false, xc, inc_a(nT - 1), inc_b(nT - 1), true, 0.f, false, 0);
        // launches of up to TC_PROGRAM_OPS ops; a dependency on an op of an earlier launch is the kernel boundary
        TcProgram prog;
        for (size_t lo = 0; lo < all.size(); lo += (size_t)TC_PROGRAM_OPS) {
            const size_t hi = std::min(all.size(), lo + (size_t)TC_PROGRAM_OPS);
            prog.ops.assign(all.begin() + lo, all.begin() + hi);
            for (size_t i = lo; i < hi; ++i) {
                TcGemm& g = prog.ops[i - lo];
                g.n_deps = 0;
                for (int d : {dep0[i], dep1[i]})
                    if (d >= (int)lo) { g.dep[g.n_deps] = d - (int)lo; g.dep_all[g.n_deps] = false; ++g.n_deps; }
                g.lane = LANE_ALL;
            }
            launch_tc_program(ctx, prog, make_rng(seed, 0, 0, 0, row0), 0);
        }
        BM_CUDA(cudaStreamSynchronize(ctx->stream));            // the workspaces above are released on return
    }

    void ais_check(int R, int n_betas, int k, const float* const* base) const override {
        const bool with_base = has_base(base);
        if (L == 2 && !with_base) { Dbm<float>::ais_check(R, n_betas, k, nullptr); return; }
        depth_check(true, with_base);
        BM_REQUIRE(R >= 1 && n_betas >= 2 && k >= 1, "bad AIS arguments");
        for (int j = 0; with_base && j <= L; ++j)
            for (int c = 0, w = j == 0 ? V : Hs[j - 1]; base[j] && c < w; ++c)
                if (!std::isfinite(base[j][c]))
                    throw Error(BM_EINVAL, "AIS base of layer " + std::to_string(j) + " (0: v) has a non-finite entry");
    }
    // The ladder at any other depth (DESIGN.md §5.4c).  Unit layer j = 0..L is v (j = 0) or h_j; the odd layers are the state
    // x, v and the even layers are summed out: log p*_beta(x) = beta sum_{odd j} c_j.x_j + sum_{even j} sum softplus(beta z_j),
    // z_j = c_j + x_{j-1} W_{j-1} + x_{j+1} W_j^T.  Per sweep, one ais_kind 1 op per summed-out layer (z_j from its one or two
    // state neighbours: the weight increment, then the layer's draw at the transition's beta) and one ais_kind 2 op per state
    // layer (the draw from its one or two summed-out neighbours, plus the linear term): L + 1 ops.  The state layers ping-pong;
    // every op waits per 256-run block on the last writers of its neighbours, which orders every read of a buffer before the
    // next write to it.  Draws: v at SITE_AIS_V; hidden layer i = j - 1 at SITE_AIS_H1 (i even) or SITE_AIS_H2 (i odd) with
    // t = i / 2, its initial state at SITE_AIS_INIT with the same t -- at L = 2 the ladder and the sites of ais_local.
    // With a base-rate model (DESIGN.md §5.4d; base: NULL or L + 1 nullable host vectors a_j) the path runs from
    // p_A ∝ exp(sum_j a_j.x_j): every op reads u_j = z_j - a_j, i.e. the bias b_j - a_j, and adds a_j after the beta scaling in
    // its epilogue (TcGemm::ais_base); the initial states are drawn from sigmoid(a_j).
    // With v clamped (DESIGN.md §5.4g; clamp: the bf16 rows of v [R, ldn[0]], no base) the roles move up one layer: v is a
    // constant operand, the odd layers are summed out and the even layers h_2, h_4, ... are the state.  Every layer drawn is
    // sampled, whatever sample_h says, and every draw is at SITE_AIS_CLAMPED: t = 2 j for the initial state of layer j, 2 j + 1
    // for its transition draws.
    void ais_local_layers(int R, uint32_t row0, int n_betas, int k, uint64_t seed, const float* const* base, double* logw_out,
                          const bf16_t* clamp = nullptr) {
        const int NL = L + 1;
        auto width = [&](int j) { return j == 0 ? V : Hs[j - 1]; };
        auto slot = [&](int j) { return (uint32_t)((j - 1) / 2); };
        std::vector<int> summed, state;                                   // the layers' roles, each in increasing j
        for (int j = clamp ? 1 : 0; j < NL; ++j) ((j % 2 == 1) == (clamp != nullptr) ? summed : state).push_back(j);
        std::vector<const float*> bias(NL), abase(NL, nullptr);
        std::vector<DevBuf<float>> a_dev(NL), d_dev(NL);
        std::vector<std::vector<float>> d_host(NL);
        for (int j = 0; j < NL; ++j) {
            bias[j] = j == 0 ? vb.p : hb[j - 1].p;
            if (!base || !base[j]) continue;
            const int w = width(j);
            d_host[j].resize(w);
            BM_CUDA(cudaMemcpyAsync(d_host[j].data(), bias[j], (size_t)w * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
            for (int c = 0; c < w; ++c) d_host[j][c] -= base[j][c];             // b_j - a_j in float32
            a_dev[j].ensure(w); d_dev[j].ensure(w);
            BM_CUDA(cudaMemcpyAsync(a_dev[j].p, base[j], (size_t)w * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
            BM_CUDA(cudaMemcpyAsync(d_dev[j].p, d_host[j].data(), (size_t)w * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
            abase[j] = a_dev[j].p; bias[j] = d_dev[j].p;
        }
        std::vector<DevBuf<bf16_t>> buf(NL), buf2(NL);
        std::vector<bf16_t*> cur(NL), nxt(NL);
        if (clamp) cur[0] = nxt[0] = const_cast<bf16_t*>(clamp);                // read only
        for (int j = clamp ? 1 : 0; j < NL; ++j) {
            buf[j].ensure((size_t)R * ldn[j]); buf[j].zero(ctx->stream);
            cur[j] = nxt[j] = buf[j].p;
        }
        for (int j : state) { buf2[j].ensure((size_t)R * ldn[j]); buf2[j].zero(ctx->stream); nxt[j] = buf2[j].p; }
        for (int j : state) {                   // x_0 ~ Ber(1/2)   (:700-702), or Ber(sigmoid(a_j)): a_j broadcast to every run
            dim3 g(((width(j) + 3) / 4 + 127) / 128, R);
            ais_unit_bf16_kernel<<<g, 128, 0, ctx->stream>>>(abase[j], 0, abase[j] ? 1.f : 0.f, cur[j], ldn[j], R, width(j), 1,
                                                             clamp ? make_rng(seed, SITE_AIS_CLAMPED, 2 * j, 0, row0)
                                                                   : make_rng(seed, SITE_AIS_INIT, slot(j), 0, row0));
            count_launch(ctx);
        }
        // the temperatures, as ais_local accumulates them
        const float delta = (float)(1.0 / n_betas);
        std::vector<float> t;
        t.push_back(delta);
        while (t.back() < 1.f - delta + 1e-5f) t.push_back(t.back() + delta);
        const int nT = (int)t.size();
        auto inc_a = [&](int j) { return j == 0 ? 0.f : t[j - 1]; };
        auto inc_b = [&](int j) { return j == nT - 1 ? 1.0f : t[j]; };
        std::vector<TcGemm> all;
        std::vector<int> dep0, dep1;                                      // global producer indices (-1: none)
        std::vector<int> last(NL, -1);                                    // the op that last wrote layer j
        // z_j from the neighbours of layer j in `x`
        auto layer_op = [&](int j, const std::vector<bf16_t*>& x) {
            TcGemm g;
            g.M = R; g.N = width(j);
            if (j == 0) {                                                 // x_1 W_0^T: W_0 stored [N, K]
                g.A[0] = mat(x[1], R, Hs[0], ldn[1]); g.K[0] = Hs[0];
                g.B[0] = mat(Wb[0].p, V, Hs[0], ldn[1]); g.b_t[0] = false;
            } else {                                                      // x_{j-1} W_{j-1} (+ x_{j+1} W_j^T)
                const int i = j - 1, in = width(j - 1);
                g.A[0] = mat(x[j - 1], R, in, ldn[j - 1]); g.K[0] = in;
                g.B[0] = mat(Wb[i].p, in, Hs[i], ldn[j]); g.b_t[0] = true;
                if (j < L) above_pair(g, i, x[j + 1], R);
            }
            g.bias = bias[j]; g.ais_base = abase[j];
            dep0.push_back(j >= 1 ? last[j - 1] : -1); dep1.push_back(j + 1 < NL ? last[j + 1] : -1);
            return g;
        };
        auto unit_op = [&](int j, float a, float b, bool weigh, float next, bool emit, uint32_t tick) {
            TcGemm g = layer_op(j, cur);
            g.act = ACT_LINEAR;
            g.ais_kind = 1; g.ais_a = a; g.ais_b = b; g.ais_next = next; g.ais_logw = weigh ? logw_out : nullptr;
            g.tick_off = tick;
            if (emit) {
                const bool smp = clamp || (j == 0 ? sample_vis != 0 : sample_h[j - 1] != 0);
                g.sample = smp ? SMP_BERNOULLI : SMP_NONE;
                g.out_state_bf = cur[j]; g.ld_state_bf = ldn[j];
                g.rng = clamp ? make_rng(0, SITE_AIS_CLAMPED, 2 * j + 1, 0, 0)
                              : j == 0 ? make_rng(0, SITE_AIS_V, 0, 0, 0) : make_rng(0, SITE_AIS_H2, slot(j), 0, 0);
                last[j] = (int)all.size();
            }
            all.push_back(g);
        };
        for (int s = 0; s < nT; ++s) {
            for (int sw = 0; sw < k; ++sw) {
                const uint32_t tick = (uint32_t)(s * k + sw);
                const bool weigh = sw == 0 && s >= 1;                    // the increment of x_s (produced by transition s-1)
                const float a = weigh ? inc_a(s - 1) : 0.f, b = weigh ? inc_b(s - 1) : 0.f;
                for (int j : summed) unit_op(j, a, b, weigh, t[s], true, tick);
                for (int j : state) {                                     // x'_j ~ sigmoid(beta (z_j - c_j) + beta c_j)
                    TcGemm o = layer_op(j, cur);
                    o.acc_scale = t[s]; o.bias_scale = t[s]; o.act = ACT_SIGMOID;
                    o.sample = SMP_BERNOULLI; o.out_state_bf = nxt[j]; o.ld_state_bf = ldn[j];
                    o.rng = clamp ? make_rng(0, SITE_AIS_CLAMPED, 2 * j + 1, 0, 0) : make_rng(0, SITE_AIS_H1, slot(j), 0, 0);
                    o.tick_off = tick;
                    o.ais_kind = 2;
                    if (sw == k - 1) {
                        o.ais_logw = logw_out;
                        o.ais_lin = (float)(((double)inc_b(s) - (double)inc_a(s)) / ((double)t[s] * -1.4426950408889634));
                    }
                    last[j] = (int)all.size();
                    all.push_back(o);
                    std::swap(cur[j], nxt[j]);                            // the other state ops read summed-out layers only
                }
            }
        }
        for (int j : summed) unit_op(j, inc_a(nT - 1), inc_b(nT - 1), true, 0.f, false, 0);               // :728
        // launches of up to TC_PROGRAM_OPS ops; a dependency on an op of an earlier launch is the kernel boundary
        TcProgram prog;
        for (size_t lo = 0; lo < all.size(); lo += (size_t)TC_PROGRAM_OPS) {
            const size_t hi = std::min(all.size(), lo + (size_t)TC_PROGRAM_OPS);
            prog.ops.assign(all.begin() + lo, all.begin() + hi);
            for (size_t i = lo; i < hi; ++i) {
                TcGemm& g = prog.ops[i - lo];
                g.n_deps = 0;
                for (int d : {dep0[i], dep1[i]})
                    if (d >= (int)lo) { g.dep[g.n_deps] = d - (int)lo; g.dep_all[g.n_deps] = false; ++g.n_deps; }
                g.lane = LANE_ALL;
            }
            launch_tc_program(ctx, prog, make_rng(seed, 0, 0, 0, row0), 0);
        }
        BM_CUDA(cudaStreamSynchronize(ctx->stream));            // the workspaces above are released on return
    }

    // ---- AIS with v clamped (DESIGN.md §5.4g) -------------------------------------------------------------------------
    // Chain c = r n_runs + k is run k of row r; it draws from Philox row (row0 + r) n_runs + k, so a row's runs depend only on
    // its index in the caller's data.  The chains run in slices of at most AIS_CLAMPED_CHAINS consecutive chains: one ladder
    // of ais_local_layers each, on v's bf16 operand built for the slice.  log_w[c] = log Z_0 + b_v.X_r + the increments, with
    // log Z_0 = (sum_i H_i) log 2 and b_v.X_r in float64 on the host from the float32 X.  At L = 1 there is nothing to
    // anneal: every run is log_proba's value, exact there (and, as log_proba does, the call writes the E-step's means).
    static constexpr int AIS_CLAMPED_CHAINS = 32768;
    void ais_clamped(const void* Xh, int rows, uint32_t row0, int n_runs, int n_betas, int k, uint64_t seed, double* log_w) override {
        bool binary = v_kind == BM_UNIT_BERNOULLI;
        for (int i = 0; i < L; ++i) binary = binary && h_kinds[i] == BM_UNIT_BERNOULLI;
        if (!binary) throw Error(BM_EUNSUPPORTED, "AIS with v clamped is defined for binary layers (Bernoulli visible and hidden units)");
        BM_REQUIRE(rows >= 1 && n_runs >= 1 && n_betas >= 2 && k >= 1, "bad AIS arguments");
        BM_REQUIRE(Xh && log_w, "ais_clamped: null argument");
        BM_REQUIRE(((uint64_t)row0 + (uint64_t)rows) * (uint64_t)n_runs < (1ull << 32),
                   "ais_clamped: (row0 + rows) * n_runs must stay below 2^32 (the chains' Philox rows)");
        const float* X = static_cast<const float*>(Xh);
        for (size_t i = 0; i < (size_t)rows * V; ++i)
            BM_REQUIRE(std::isfinite(X[i]), "ais_clamped: X has a non-finite entry");
        const long long total = (long long)rows * n_runs;
        if (L == 1) {
            std::vector<double> lp(B);
            for (int lo = 0; lo < rows; lo += B) {
                const int n = std::min(B, rows - lo);
                log_proba(X + (size_t)lo * V, n, lp.data());
                for (int r = 0; r < n; ++r) std::fill(log_w + (size_t)(lo + r) * n_runs, log_w + (size_t)(lo + r + 1) * n_runs, lp[r]);
            }
            return;
        }
        std::vector<float> b_v(V);
        BM_CUDA(cudaMemcpyAsync(b_v.data(), vb.p, (size_t)V * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        DevBuf<float> Xd;
        Xd.ensure((size_t)rows * V);
        BM_CUDA(cudaMemcpyAsync(Xd.p, X, (size_t)rows * V * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        const int cap = (int)std::min<long long>(total, AIS_CLAMPED_CHAINS);
        DevBuf<bf16_t> vop;
        DevBuf<double> lw;
        vop.ensure((size_t)cap * ldn[0]); lw.ensure(cap);
        std::vector<double> hw(cap);
        double logZ0 = 0.0;
        for (int i = 0; i < L; ++i) logZ0 += (double)Hs[i] * 0.69314718055994530942;
        for (long long c0 = 0; c0 < total; c0 += cap) {
            const int n = (int)std::min<long long>(cap, total - c0);
            ais_clamp_rows_kernel<<<dim3((ldn[0] + 127) / 128, n), 128, 0, ctx->stream>>>(Xd.p, V, c0, n_runs, vop.p, ldn[0], n);
            count_launch(ctx);
            lw.zero(ctx->stream);
            ais_local_layers(n, (uint32_t)((uint64_t)row0 * n_runs + (uint64_t)c0), n_betas, k, seed, nullptr, lw.p, vop.p);
            BM_CUDA(cudaMemcpyAsync(hw.data(), lw.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
            for (int i = 0; i < n; ++i) {
                const long long r = (c0 + i) / n_runs;
                double bvx = 0.0;
                for (int c = 0; c < V; ++c) bvx += (double)b_v[c] * (double)X[(size_t)r * V + c];
                log_w[c0 + i] = hw[i] + logZ0 + bvx;
            }
        }
    }

    // the same ladder for models whose first hidden layer is not sampled: fp32 pre-activations in memory and, per temperature,
    // one pass over them for the weight increment and the next transition's first unit updates
    void ais_local_passes(int R, uint32_t row0, int n_betas, int k, uint64_t seed, double* logw_out) {
        const int H0 = Hs[0], H1 = Hs[1];
        const int ld0 = ldn[1], ldv = ldn[0], ld1 = ldn[2];
        DevBuf<bf16_t> x, xn, va, hc;
        DevBuf<float> pa, pb;
        struct { double* p; } logw{logw_out};
        x.ensure((size_t)R * ld0); xn.ensure((size_t)R * ld0); va.ensure((size_t)R * ldv); hc.ensure((size_t)R * ld1);
        pa.ensure((size_t)R * V); pb.ensure((size_t)R * H1);
        for (DevBuf<bf16_t>* b : {&x, &xn, &va, &hc}) b->zero(ctx->stream);
        const dim3 rgrid((R + 7) / 8), rblock(32, 8);
        auto pre = [&](const bf16_t* xs) {          // pa = x W_0^T + b ; pb = x W_1 + c_2   (beta-free, shared)
            linear_tc(xs, ld0, R, H0, Wb[0].p, V, H0, ld0, false, V, vb.p, pa.p);
            linear_tc(xs, ld0, R, H0, Wb[1].p, H0, H1, ld1, true, H1, hb[1].p, pb.p);
        };
        bf16_t* xc = x.p; bf16_t* xo = xn.p;
        int it = 0;
        // `fused`: pa / pb of sweep 0 are current and the fused pass of this temperature step has already produced its va / hc
        auto transition = [&](float beta, bool fused) {
            for (int s = 0; s < k; ++s) {
                const uint32_t tick = (uint32_t)(it * k + s);
                if (!(fused && s == 0)) {
                    pre(xc);
                    dim3 gv(((V + 3) / 4 + 127) / 128, R), gh(((H1 + 3) / 4 + 127) / 128, R);
                    ais_unit_bf16_kernel<<<gv, 128, 0, ctx->stream>>>(pa.p, V, beta, va.p, ldv, R, V, sample_vis, make_rng(seed, SITE_AIS_V, 0, tick, row0));
                    ais_unit_bf16_kernel<<<gh, 128, 0, ctx->stream>>>(pb.p, H1, beta, hc.p, ld1, R, H1, sample_h[1], make_rng(seed, SITE_AIS_H2, 0, tick, row0));
                    count_launch(ctx); count_launch(ctx);
                }
                TcGemm o;                     // x' = act(beta (v W_0 + h2 W_1^T), beta c_1)
                o.M = R; o.N = H0;
                o.A[0] = mat(va.p, R, V, ldv); o.K[0] = V; o.B[0] = mat(Wb[0].p, V, H0, ld0); o.b_t[0] = true;
                above_pair(o, 0, hc.p, R);
                o.acc_scale = beta; o.bias_scale = beta; o.bias = hb[0].p; o.act = ACT_SIGMOID;
                o.rng = make_rng(seed, SITE_AIS_H1, 0, tick, row0);
                if (sample_h[0]) { o.sample = SMP_BERNOULLI; o.out_state_bf = xo; o.ld_state_bf = ld0; }
                else { o.out_mean_bf = xo; o.ld_mean_bf = ld0; }
                launch_tc_gemm(ctx, o);
                std::swap(xc, xo);
            }
            ++it;
        };
        {   // x_0 ~ Ber(1/2)   (:700-702)
            dim3 g(((H0 + 3) / 4 + 127) / 128, R);
            ais_unit_bf16_kernel<<<g, 128, 0, ctx->stream>>>(nullptr, 0, 0.f, xc, ld0, R, H0, 1, make_rng(seed, SITE_AIS_INIT, 0, 0, row0));
            count_launch(ctx);
        }
        // increment of the log-weights on the current x (pa / pb current) and, in the same pass, sweep 0's unit updates at beta_next
        auto step = [&](float prev, float beta, float beta_next) {
            const uint32_t tick = (uint32_t)(it * k);            // sweep 0 of the transition that follows
            ais_fused_step_kernel<<<rgrid, rblock, 0, ctx->stream>>>(
                logw.p, prev, beta, beta_next, 1, xc, ld0, H0, hb[0].p,
                pa.p, V, va.p, ldv, sample_vis, make_rng(seed, SITE_AIS_V, 0, tick, row0),
                pb.p, H1, hc.p, ld1, sample_h[1], make_rng(seed, SITE_AIS_H2, 0, tick, row0), R);
            count_launch(ctx);
        };
        const float delta = (float)(1.0 / n_betas);
        transition(delta, false);                               // x_1 ~ T_1(x_1 | x_0)            :705
        pre(xc);
        float beta = delta, prev = 0.f;                         // - log p_0(x_1) pairs with + log p_1(x_1) :708
        while (beta < 1.f - delta + 1e-5f) {                    // :710-711 (beta accumulates in the storage dtype)
            step(prev, beta, beta + delta);                     // + log p_i(x_i) - log p_{i-1}(x_i)  [+ v, h2 of T_{i+1}]
            transition(beta + delta, true);                     // x_{i+1} ~ T_{i+1}
            pre(xc);
            prev = beta;
            beta = beta + delta;
        }
        // + log p_M(x_M) - log p_{M-1}(x_M)   :728  (the weight-only kernel: the fused one with emit = 0 sums in another order)
        ais_accum2_bf16_kernel<<<rgrid, rblock, 0, ctx->stream>>>(logw.p, prev, 1.0f, xc, ld0, H0, hb[0].p, pa.p, V, pb.p, H1, R);
        count_launch(ctx);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));            // the workspaces above are released on return
    }
};

}  // namespace bm
