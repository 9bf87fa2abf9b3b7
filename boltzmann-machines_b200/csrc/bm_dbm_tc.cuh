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
// STATUS: the default engine of float32 DBMs (bm_dbm_cfg.compute = BM_COMPUTE_BF16, which the Python mirror passes unless
// compute='fp32' or BM_DBM_COMPUTE / BM_COMPUTE = fp32 asks for the storage-precision CUDA-core engine).  Models it does not
// support (DbmTC::supports) run on that engine.
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
    bool particles_f32_stale = false;            // the bf16 particles are newer than the fp32 copies get_param reads
    // mean-field as persistent dataflow programs of up to MF_CHUNK speculated sweeps per launch: slot history + programs
    static constexpr int MF_CHUNK = 5;
    int mf_chunk = 0;                            // MF_CHUNK, clamped by max_mf and by TC_PROGRAM_OPS, at least 1
    std::vector<DevBuf<bf16_t>> hist;            // per layer: (mf_chunk + 2) slots of [B, ldn[i+1]]
    DevBuf<unsigned int> mf_flags;
    std::map<std::pair<int, int>, std::unique_ptr<TcProgram>> mf_progs;      // keyed by (rows, sweeps in the chunk)
    // committed particle sweeps as ONE persistent program: keyed by (sweeps, sampled, t0)
    std::map<std::tuple<int, int, int>, std::unique_ptr<TcProgram>> pcd_progs;

    static bool supports(const bm_dbm_cfg& f) {
        if (f.dtype != BM_DTYPE_F32) return false;
        if (!(f.v_kind == BM_UNIT_BERNOULLI || f.v_kind == BM_UNIT_GAUSSIAN)) return false;
        for (int i = 0; i < f.n_layers; ++i) if (f.h_kinds[i] != BM_UNIT_BERNOULLI) return false;
        return f.n_layers <= TC_PROGRAM_OPS;     // one mean-field sweep (L ops) fits in one program
    }

    DbmTC(Ctx* c, const bm_dbm_cfg& f) : Dbm<float>(c, f) {
        ldn.push_back(dbm_round_up(V, 64));
        for (int i = 0; i < L; ++i) ldn.push_back(dbm_round_up(Hs[i], 64));
        Wb.resize(L); WbT.resize(L); mu_b.resize(L); h_b.resize(L); h2_b.resize(L); h3_b.resize(L); Gp.resize(L);
        Xb.ensure((size_t)B * ldn[0]); recon_b.ensure((size_t)B * ldn[0]);
        v_b.ensure((size_t)M * ldn[0]); v2_b.ensure((size_t)M * ldn[0]);
        for (DevBuf<bf16_t>* b : {&Xb, &recon_b, &v_b, &v2_b}) b->zero(ctx->stream);
        for (int i = 0; i < L; ++i) {
            Wb[i].ensure((size_t)size_of(i, V, Hs) * ldn[i + 1]);
            mu_b[i].ensure((size_t)B * ldn[i + 1]);
            h_b[i].ensure((size_t)M * ldn[i + 1]); h2_b[i].ensure((size_t)M * ldn[i + 1]);
            for (DevBuf<bf16_t>* b : {&Wb[i], &mu_b[i], &h_b[i], &h2_b[i]}) b->zero(ctx->stream);
        }
        for (int i = 1; i < L; ++i) { WbT[i].ensure((size_t)Hs[i] * ldn[i]); WbT[i].zero(ctx->stream); }
        mf_chunk = std::max(1, std::min(std::min(MF_CHUNK, max_mf), TC_PROGRAM_OPS / L));
        hist.resize(L);
        for (int i = 0; i < L; ++i) { hist[i].ensure((size_t)(mf_chunk + 2) * B * ldn[i + 1]); hist[i].zero(ctx->stream); }
        mf_flags.ensure(mf_chunk);
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
        for (int i = 0; i < L; ++i) launch_bf16_to_f32(ctx, h_b[i].p, ldn[i + 1], h[i].p, Hs[i], M, Hs[i]);
        particles_f32_stale = false;
    }
    void widen_mu(int rows) { for (int i = 0; i < L; ++i) launch_bf16_to_f32(ctx, mu_b[i].p, ldn[i + 1], mu[i].p, Hs[i], rows, Hs[i]); }

    void set_param(const char* name, const void* host, size_t bytes) override {
        widen_particles();                         // the fp32 copies become the truth for one moment
        Dbm<float>::set_param(name, host, bytes);
        narrow_state();
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void get_param(const char* name, void* host, size_t bytes) override {
        widen_particles();
        Dbm<float>::get_param(name, host, bytes);
    }
    void init_particles(uint64_t seed) override {
        widen_particles();
        Dbm<float>::init_particles(seed);
        narrow_state();
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // ---- one fused conditional on the tensor cores -----------------------------------------------------------
    // act(acc_scale * (below W_i [+ above W_{i+1}^T]) + bias_scale * b_i): means XOR sampled states (bf16)
    void hidden_tc(int i, const bf16_t* below, const bf16_t* above, bf16_t* out, bool sample, int rows,
                   float acc_scale, float bias_scale, RngKey rng) {
        launch_tc_gemm(ctx, hidden_gemm(i, below, above, out, sample, rows, acc_scale, bias_scale, rng));
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
                  bool update_v, bool sample, int rows, uint64_t seed, uint32_t tstep, uint32_t tick) {
        for (int i = 0; i < L; ++i) {
            const bf16_t* below = i == 0 ? vin : Hn[i - 1];
            const bf16_t* above = (i + 1 < L) ? Hin[i + 1] : nullptr;
            hidden_tc(i, below, above, Hn[i], sample && sample_h[i], rows, 1.f, 1.f, make_rng(seed, SITE_DBM_H + i, tstep, tick, particle_row0()));
        }
        if (update_v) visible_tc(Hn[0], v_new, sample && sample_vis, rows, make_rng(seed, SITE_DBM_V, tstep, tick, particle_row0()));
    }

    const float* upload_tc(const void* Xh, int rows) {
        const float* X = upload(Xh, rows);
        launch_f32_to_bf16(ctx, X, V, Xb.p, ldn[0], rows, V);
        return X;
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
        for (int i = 0; i < L; ++i) {                                        // approximate-inference pass -> slot 0
            const bf16_t* below = i == 0 ? Xb.p : slot(i - 1, 0);
            const float sc = (i == 0 || i < L - 1) ? 2.f : 1.f;
            hidden_tc(i, below, nullptr, slot(i, 0), false, rows, sc, 1.f, RngKey{});
            BM_CUDA(cudaMemcpyAsync(slot(i, 1), mu_b[i].p, (size_t)rows * ldn[i + 1] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        }
        int a = 0, result_slot = 1;
        bool done = false;
        while (!done && a < max_mf) {
            const int c = std::min(mf_chunk, max_mf - a);
            std::unique_ptr<TcProgram>& pslot = mf_progs[std::make_pair(rows, c)];
            if (!pslot) {
                pslot.reset(new TcProgram());
                std::vector<TcGemm>& ops = pslot->ops;
                for (int s = 1; s <= c; ++s)                                 // sweep s: slot s -> slot s + 1
                    for (int i = 0; i < L; ++i) {
                        const bf16_t* below = i == 0 ? Xb.p : slot(i - 1, s + 1);
                        const bf16_t* above = (i + 1 < L) ? slot(i + 1, s) : nullptr;
                        TcGemm g = hidden_gemm(i, below, above, slot(i, s + 1), false, rows, 1.f, 1.f, RngKey{});
                        const int self = (int)ops.size();
                        if (i > 0) { g.dep[g.n_deps] = self - 1; g.dep_all[g.n_deps] = false; ++g.n_deps; }           // layer i-1, this sweep
                        if (above && s > 1) { g.dep[g.n_deps] = self - L + 1; g.dep_all[g.n_deps] = false; ++g.n_deps; } // layer i+1, previous sweep
                        g.lane = LANE_CHAIN;
                        ops.push_back(g);
                    }
            }
            launch_tc_program(ctx, *pslot, RngKey{}, 0);
            BM_CUDA(cudaMemsetAsync(mf_flags.p, 0, (size_t)c * sizeof(unsigned int), ctx->stream));
            for (int i = 0; i < L; ++i) {
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
        std::unique_ptr<TcProgram>& pslot = pcd_progs[std::make_tuple(n_steps, sample ? 1 : 0, t0)];
        std::vector<bf16_t*> cur(L), nxt(L);
        for (int i = 0; i < L; ++i) { cur[i] = h_b[i].p; nxt[i] = h2_b[i].p; }
        bf16_t* vc = v_b.p; bf16_t* vn = v2_b.p;
        const bool build = !pslot;
        if (build) pslot.reset(new TcProgram());
        std::vector<TcGemm>& ops = pslot->ops;
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
                }
                TcGemm gv = visible_gemm(nxt[0], vn, sample && sample_vis, M, make_rng(0, SITE_DBM_V, tstep, 0, 0));
                gv.dep[0] = this_h[0]; gv.dep_all[0] = false; gv.n_deps = 1;
                gv.lane = LANE_CHAIN;
                last_vis = (int)ops.size();
                ops.push_back(gv);
                last_h = this_h;
            }
            std::swap(cur, nxt); std::swap(vc, vn);
        }
        launch_tc_program(ctx, *pslot, make_rng(seed, 0, 0, tick, particle_row0()), 0);
        for (int i = 0; i < L; ++i)
            if (cur[i] != h_b[i].p)
                BM_CUDA(cudaMemcpyAsync(h_b[i].p, cur[i], (size_t)M * ldn[i + 1] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        if (vc != v_b.p) BM_CUDA(cudaMemcpyAsync(v_b.p, vc, (size_t)M * ldn[0] * sizeof(bf16_t), cudaMemcpyDeviceToDevice, ctx->stream));
        particles_f32_stale = true;
    }

    // committed sweeps that fit in one program run as that program; uncommitted runs (the second half of sample_v) and
    // longer chains take one launch per op
    void particles_tc(int n_steps, bool sample, uint64_t seed, uint32_t tick, int t0, bool commit, bf16_t** v_final) {
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
            gibbs_tc(vc, Hin, nxt, vn, true, sample, M, seed, (uint32_t)(t0 + s + 1), tick);
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
        dbm_grad_combine_kernel<<<592, 256, 0, ctx->stream>>>(Gp[i].p, sp, Gp[i].p + (size_t)sp * stride, sn, stride,
                                                              1.0f / n_div, 1.0f / m_div, G[i].p, stride);
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
        for (int i = 0; i < L; ++i) gradient_tc(i, i == 0 ? Xb.p : mu_b[i - 1].p, rows, i == 0 ? v_b.p : h_b[i - 1].p, N, Mp);
        {   // column sums of mu_i (over the batch rows) and of h_i, v (over the particles), three per pair of launches
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
        }
        launch_colsum<float>(ctx, X, V, (const float*)nullptr, 0, rows, V, 1.f, 0.f, xsum.p);
        allreduce_step_statistics();
        dbm_vbias_kernel<float><<<(V + 255) / 256, 256, 0, ctx->stream>>>(V, xsum.p, vsum.p, rows_g, Mp, vb.p, dvb.p, (float)lr, (float)mom);
        count_launch(ctx);
        for (int i = 0; i < L; ++i) {
            const int in = size_of(i, V, Hs), H = Hs[i];
            BM_REQUIRE(i < H, "the reference's sparsity update indexes element i of layer i's unit vector");
            dbm_sparsity_bias_kernel<float><<<(H + 255) / 256, 256, 0, ctx->stream>>>(
                H, i, musum[i].p, hsum[i].p, rows_g, Mp, qm[i].p, mm[i].p, pen[i].p, hb[i].p, dhb[i].p,
                (float)damping, (float)sp_cost[i], (float)sp_target[i], (float)lr, (float)mom);
            count_launch(ctx);
            launch_weight_update<float>(ctx, G[i].p, H, 1.f, W[i].p, dW[i].p, in, H, pen[i].p, (float)l2, (float)lr, (float)mom, nullptr, 0);
            colnorm_kernel<float><<<(H + 31) / 32, dim3(32, 8), 0, ctx->stream>>>(W[i].p, in, H, norm[i].p);       // :511-513
            count_launch(ctx);
            max_norm_scale_kernel<float><<<dim3((H + 255) / 256, in < 32768 ? in : 32768), 256, 0, ctx->stream>>>(W[i].p, in, H, norm[i].p, (float)max_norm);
            count_launch(ctx);
            refresh_shadow(i);
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
        BM_REQUIRE(L == 2, "log_proba is defined for 2 hidden layers");
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
    void ais_local(int R, uint32_t row0, int n_betas, int k, uint64_t seed, double* logw_out) override {
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
