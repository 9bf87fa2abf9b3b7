// DBM engine behind bm_dbm_* (include/bm.h): device-resident weights, momentum accumulators,
// variational parameters and persistent particles of a Deep Boltzmann Machine, and what the
// reference executes inside session.run for it (paths relative to /root/reference/boltzmann_machines/):
//   layer-wise Gibbs step dbm.py:385-427 (two-operand accumulate: H_{i-1} W_i + H_{i+1} W_{i+1}^T in ONE
//   fused layer op), mean-field E-step :429-478, PCD particle update :480-509, gradients / sparsity /
//   momentum / max-norm :511-513,550-615, msre :625-633, sample_v :641-648, AIS :650-736 (the two
//   pre-activations x W_0^T + b and x W_1 + c_2 are computed once per temperature and shared by the
//   importance weight and by the transition), variational bound :738-759.
// Storage-precision (float32 / float64) CUDA-core path: the shared fused LayerOp of bm_simt.cu.
//
// Data parallelism (SURVEY 8e; not in the reference, which is single-device): on a context with a communicator every
// rank holds batch_size rows of the batch (and of mu) and n_particles persistent particles -- the global model has
// nranks times as many of each.  Rows are independent given the weights: the sampling sites are keyed by the GLOBAL
// particle index (row0 = rank * n_particles), the mean-field convergence test takes the max over all ranks, and the
// row sums that enter the update (pos^T mu - neg^T h per layer, the column sums of mu, h, X, v) are sum-allreduced
// in one buffer before every rank applies the identical update.  With one rank nothing below changes.
#include "bm_rbm.h"
#include <algorithm>
#include <cmath>
#include <vector>
#include <string>

namespace bm {

// ---------------------------------------------------------------------------------------------
// small kernels specific to the DBM
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void max_abs_diff_kernel(const T* __restrict__ a, const T* __restrict__ b, size_t n, unsigned int* __restrict__ out) {
    // max |a-b| over all elements; non-negative floats order like their bit patterns
    float m = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        m = fmaxf(m, (float)fabs((double)a[i] - (double)b[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

template <typename T>
__global__ void dbm_sparsity_bias_kernel(int H, int layer, const T* __restrict__ mu_sum, const T* __restrict__ h_sum,
                                         T n_div, T m_div, T* __restrict__ q_means, T* __restrict__ mu_means,
                                         T* __restrict__ pen, T* __restrict__ hb, T* __restrict__ dhb,
                                         T damp, T cost, T target, T lr, T mom) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= H) return;
    // dbm.py:581-586: `q_means[i]` / `mu_means[i]` take ELEMENT `layer` of the per-unit sum vectors (sic)
    const T q = damp * q_means[j] + (T(1) - damp) * h_sum[layer];
    const T mm = damp * mu_means[j] + (T(1) - damp) * mu_sum[layer];
    q_means[j] = q; mu_means[j] = mm;
    const T p = cost * (q - target) + cost * (mm - target);          // :587-588
    pen[j] = p;
    const T g = mu_sum[j] / n_div - h_sum[j] / m_div - p;            // :575, :590
    const T d = lr * (mom * dhb[j] + g);                              // :613-614
    dhb[j] = d;
    hb[j] += d;
}

template <typename T>
__global__ void dbm_vbias_kernel(int V, const T* __restrict__ x_sum, const T* __restrict__ v_sum, T n_rows, T m_div,
                                 T* __restrict__ vb, T* __restrict__ dvb, T lr, T mom) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= V) return;
    const T g = x_sum[j] / n_rows - v_sum[j] / m_div;                // :553 (reduce_mean over the rows present)
    const T d = lr * (mom * dvb[j] + g);                              // :595-596
    dvb[j] = d;
    vb[j] += d;
}

template <typename T>
__global__ void colnorm_kernel(const T* __restrict__ W, int rows, int cols, T* __restrict__ norm) {
    __shared__ double part[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    double a = 0.0;
    if (c < cols)
        for (int r = threadIdx.y; r < rows; r += 8) { const double w = (double)W[(size_t)r * cols + c]; a += w * w; }
    part[threadIdx.y][threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) s += part[i][threadIdx.x];
        norm[c] = (T)sqrt(s);
    }
}
template <typename T>
__global__ void max_norm_scale_kernel(T* __restrict__ W, int rows, int cols, const T* __restrict__ norm, T max_norm) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    const T n = norm[c];
    const T num = n < max_norm ? n : max_norm;                       // dbm.py:513: T * min(norm, c) / max(norm, 1e-8)
    const T den = n > T(1e-8) ? n : T(1e-8);
    // (rows stride over grid.y: the launch caps it at 32768 blocks, below the 65535 limit of that dimension)
    for (int r = blockIdx.y; r < rows; r += gridDim.y) W[(size_t)r * cols + c] = W[(size_t)r * cols + c] * num / den;
}

// per-row terms of the variational bound (dbm.py:743-757); t1 = X W_0, t2 = mu_0 W_1
template <typename T>
__global__ void dbm_bound_rows_kernel(const T* __restrict__ X, int V, const T* __restrict__ mu0, int H0,
                                      const T* __restrict__ mu1, int H1, const T* __restrict__ t1, const T* __restrict__ t2,
                                      const T* __restrict__ vb, const T* __restrict__ hb0, const T* __restrict__ hb1,
                                      int rows, double* __restrict__ out) {
    const int r = blockIdx.x * blockDim.y + threadIdx.y;
    if (r >= rows) return;
    double a = 0.0;
    for (int j = threadIdx.x; j < H0; j += 32) {
        const double m = (double)mu0[(size_t)r * H0 + j];
        a += (double)t1[(size_t)r * H0 + j] * m + m * (double)hb0[j];
        double s = fmin(fmax(m, 1e-7), 1.0 - 1e-7);
        if (sizeof(T) == 4) s = (double)fminf(fmaxf((float)m, 1e-7f), 1.0f - 1e-7f);
        a += -s * log(s) - (1.0 - s) * log(1.0 - s);
    }
    for (int j = threadIdx.x; j < H1; j += 32) {
        const double m = (double)mu1[(size_t)r * H1 + j];
        a += (double)t2[(size_t)r * H1 + j] * m + m * (double)hb1[j];
        double s = fmin(fmax(m, 1e-7), 1.0 - 1e-7);
        if (sizeof(T) == 4) s = (double)fminf(fmaxf((float)m, 1e-7f), 1.0f - 1e-7f);
        a += -s * log(s) - (1.0 - s) * log(1.0 - s);
    }
    for (int j = threadIdx.x; j < V; j += 32) a += (double)X[(size_t)r * V + j] * (double)vb[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) out[r] = a;
}

// AIS: logw[r] += sign * log p*_beta(x_r) = sign * (beta x.c1 + sum softplus(beta pa) + sum softplus(beta pb))
template <typename T>
__global__ void ais_accum_kernel(double* __restrict__ logw, double sign, double beta, const T* __restrict__ x, int H0,
                                 const T* __restrict__ hb0, const T* __restrict__ pa, int V, const T* __restrict__ pb, int H1, int rows) {
    const int r = blockIdx.x * blockDim.y + threadIdx.y;
    if (r >= rows) return;
    double a = 0.0;
    for (int j = threadIdx.x; j < H0; j += 32) a += beta * (double)x[(size_t)r * H0 + j] * (double)hb0[j];
    for (int j = threadIdx.x; j < V; j += 32) { const double z = beta * (double)pa[(size_t)r * V + j]; a += fmax(z, 0.0) + log1p(exp(-fabs(z))); }
    for (int j = threadIdx.x; j < H1; j += 32) { const double z = beta * (double)pb[(size_t)r * H1 + j]; a += fmax(z, 0.0) + log1p(exp(-fabs(z))); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) logw[r] += sign * a;
}

// out = sample? (u < sigmoid(beta * pre)) : sigmoid(beta * pre)      (AIS transition from shared pre-activations)
template <typename T>
__global__ void ais_unit_kernel(const T* __restrict__ pre, T beta, T* __restrict__ out, int rows, int cols, int sample, RngKey rng) {
    const int cb = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    if (cb * 4 >= cols || r >= rows) return;
    U4 w{0, 0, 0, 0};
    if (sample) w = site_block(rng, (uint32_t)r, (uint32_t)cb);
    const uint32_t words[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int c = cb * 4 + j;
        if (c >= cols) break;
        // activation(beta * x, beta * b) with x + b precomputed: sigmoid(beta*x + beta*b) (dbm.py:669)
        const T z = beta * pre[(size_t)r * cols + c];
        T p = T(1) / (T(1) + (sizeof(T) == 4 ? (T)expf(-(float)z) : (T)exp(-(double)z)));
        out[(size_t)r * cols + c] = sample ? ((T(u32_to_unit_float(words[j])) < p) ? T(1) : T(0)) : p;
    }
}

template <typename T>
__global__ void particle_init_kernel(T* __restrict__ out, int rows, int cols, int kind, const T* __restrict__ sigma, RngKey rng) {
    const int cb = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    if (cb * 4 >= cols || r >= rows) return;
    const U4 w = site_block(rng, (uint32_t)r, (uint32_t)cb);
    const uint32_t words[4] = {w.x, w.y, w.z, w.w};
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    if (kind == BM_UNIT_GAUSSIAN) {
        float u1 = fmaxf(u32_to_unit_float(w.x), 1.0e-7f), v1 = 6.2831853071795864769f * u32_to_unit_float(w.y);
        float u2 = sqrtf(-2.0f * logf(u1)); g[0] = sinf(v1) * u2; g[1] = cosf(v1) * u2;
        u1 = fmaxf(u32_to_unit_float(w.z), 1.0e-7f); v1 = 6.2831853071795864769f * u32_to_unit_float(w.w);
        u2 = sqrtf(-2.0f * logf(u1)); g[2] = sinf(v1) * u2; g[3] = cosf(v1) * u2;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int c = cb * 4 + j;
        if (c >= cols) break;
        out[(size_t)r * cols + c] = kind == BM_UNIT_GAUSSIAN ? (T)g[j] * sigma[c] : (T)u32_to_unit_float(words[j]);
    }
}
template <typename T>
__global__ void scale_all_kernel(T* p, size_t n, const double* total) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        p[i] = (T)((double)p[i] / *total);
}

// ---- clamped Gibbs chains (bm_dbm_fill, DESIGN.md §5.9) ---------------------------------------------------------------
// The visible clamp: v[r, c] <- X[r, c] wherever mask[r, c] (dense [rows, cols] bytes, 0 / 1) is set.  S is the chain's element
// type: the storage dtype on the CUDA-core engine, bf16 operands on the tensor-core one.
template <typename S>
__global__ void dbm_fill_clamp_kernel(const uint8_t* __restrict__ mask, const S* __restrict__ X, int ldx, S* __restrict__ v, int ldv,
                                      int rows, int cols) {
    const size_t n = (size_t)rows * cols;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / cols, c = i % cols;
        if (mask[i]) v[r * ldv + c] = X[r * ldx + c];
    }
}
__device__ __forceinline__ float fill_widen(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float fill_widen(float x) { return x; }
__device__ __forceinline__ double fill_widen(double x) { return x; }
// The result of a fill: out[r, c] = mask ? X[r, c] : mean[r, c] (mean: the chain's element type S, widened to the model's T).
template <typename S, typename T>
__global__ void dbm_fill_out_kernel(const uint8_t* __restrict__ mask, const T* __restrict__ X, const S* __restrict__ mean, int ldm,
                                    T* __restrict__ out, int rows, int cols) {
    const size_t n = (size_t)rows * cols;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / cols, c = i % cols;
        out[i] = mask[i] ? X[i] : (T)fill_widen(mean[r * ldm + c]);
    }
}
static inline unsigned fill_grid(int rows, int cols) {
    const size_t n = (size_t)rows * cols;
    return (unsigned)std::min<size_t>((n + 255) / 256, 4096);
}
template <typename S>
void launch_dbm_fill_clamp(Ctx* ctx, const uint8_t* mask, const S* X, int ldx, S* v, int ldv, int rows, int cols) {
    dbm_fill_clamp_kernel<S><<<fill_grid(rows, cols), 256, 0, ctx->stream>>>(mask, X, ldx, v, ldv, rows, cols);
    count_launch(ctx);
}
template <typename S, typename T>
void launch_dbm_fill_out(Ctx* ctx, const uint8_t* mask, const T* X, const S* mean, int ldm, T* out, int rows, int cols) {
    dbm_fill_out_kernel<S, T><<<fill_grid(rows, cols), 256, 0, ctx->stream>>>(mask, X, mean, ldm, out, rows, cols);
    count_launch(ctx);
}

// What bm_dbm_fill refuses before anything is launched.  C: classes of the label layer (0: none).
static void check_fill_args(const uint8_t* mask, const int32_t* labels, int rows, int k, int B, int V, int C) {
    BM_REQUIRE(rows >= 1 && rows <= B, "fill: rows must lie in 1..batch_size (" + std::to_string(rows) + " given)");
    BM_REQUIRE(k >= 1, "fill: n_gibbs_steps must be >= 1");
    const size_t n = (size_t)rows * V;
    for (size_t i = 0; i < n; ++i)
        if (mask[i] > 1)
            throw Error(BM_EINVAL, "fill: mask byte " + std::to_string(i % V) + " of row " + std::to_string(i / V) + " is " +
                                   std::to_string((int)mask[i]) + ", not 0 or 1");
    if (!labels) return;
    if (C == 0) throw Error(BM_EINVAL, "this DBM has no label layer (bm_dbm_cfg.n_classes)");
    for (int r = 0; r < rows; ++r)
        if (labels[r] < -1 || labels[r] >= C)
            throw Error(BM_EINVAL, "label " + std::to_string(labels[r]) + " of row " + std::to_string(r) + " is outside [-1, n_classes)");
}

// ---------------------------------------------------------------------------------------------
struct DbmBase {
    Ctx* ctx = nullptr;
    virtual ~DbmBase() {}
    virtual void set_param(const char* name, const void* host, size_t bytes) = 0;
    virtual void get_param(const char* name, void* host, size_t bytes) = 0;
    virtual void init_particles(uint64_t seed) = 0;
    virtual void train_step(const void* X, int rows, double lr, double mom, int k, uint64_t seed, uint32_t tick, int want, double* out) = 0;
    virtual void val_metrics(const void* X, int rows, int k, uint64_t seed, uint32_t tick, double* out) = 0;
    virtual void transform(const void* X, int rows, void* out) = 0;
    virtual void reconstruct(const void* X, int rows, void* out) = 0;
    virtual void log_proba(const void* X, int rows, double* out) = 0;
    virtual void sample_v(int k, uint64_t seed, uint32_t tick, void* out) = 0;
    // base: NULL or L + 1 nullable host vectors (v, h_1 .. h_L) of an AIS base-rate model (DESIGN.md §5.4d); all-null is NULL
    virtual void ais(int n_runs, int n_betas, int k, uint64_t seed, const float* const* base, double* out) = 0;
    virtual void ais_rows(int n_runs, int n_betas, int k, uint64_t seed, uint32_t first_run, const float* const* base, double* out) = 0;
    virtual void pt_counts(int64_t*, int64_t*) { throw Error(BM_EINVAL, "this DBM has no tempered chains (bm_dbm_cfg.n_temps)"); }
    virtual void train_step_labeled(const void*, const int32_t*, int, double, double, int, uint64_t, uint32_t, int, double*) {
        throw Error(BM_EINVAL, "this DBM has no label layer (bm_dbm_cfg.n_classes)");
    }
    virtual void predict_proba(const void*, int, float*) { throw Error(BM_EINVAL, "this DBM has no label layer (bm_dbm_cfg.n_classes)"); }
    // clamped Gibbs chains (DESIGN.md §5.9): rows of X [rows, V] with mask [rows, V], labels [rows] or NULL -> out [rows, V]
    virtual void fill(const void* X, const uint8_t* mask, const int32_t* labels, int rows, uint32_t row0, int k, uint64_t seed,
                      uint32_t tick, void* out) = 0;
    virtual void fill_debug(const char* name, void* host, size_t bytes) = 0;
    virtual void sample_v_debug(const char* name, void* host, size_t bytes) = 0;
    // exact log Z and log p*(v) by enumerating the odd layers (DESIGN.md §5.4f): the tensor-core engine's (bm_dbm_exact.cuh)
    virtual void exact(const void*, int, double*, double*) {
        throw Error(BM_EUNSUPPORTED, "exact log Z runs on the tensor-core engine (float32 models, BM_COMPUTE_BF16), not on the "
                                     "CUDA-core engine");
    }
    // AIS over the hidden layers with v clamped to each row of X (DESIGN.md §5.4g): the tensor-core engine's (DbmTC)
    virtual void ais_clamped(const void*, int, uint32_t, int, int, int, uint64_t, double*) {
        throw Error(BM_EUNSUPPORTED, "AIS with v clamped runs on the tensor-core engine (float32 models, BM_COMPUTE_BF16), not on "
                                     "the CUDA-core engine");
    }
};

// Parallel tempering (bm_dbm_cfg.n_temps / betas): what the engines refuse before anything is allocated.  0 / NULL is off.
static void check_pt_cfg(const Ctx* ctx, const bm_dbm_cfg& f) {
    if (f.n_temps == 0 && f.betas == nullptr) return;
    BM_REQUIRE(f.n_temps >= 1 && f.betas != nullptr, "parallel tempering: n_temps >= 1 inverse temperatures are needed in betas");
    BM_REQUIRE(f.betas[0] == 1.0, "parallel tempering: betas[0] must be 1");
    for (int m = 1; m < f.n_temps; ++m)
        BM_REQUIRE(std::isfinite(f.betas[m]) && f.betas[m] < f.betas[m - 1] && f.betas[m] >= 0.0,
                   "parallel tempering: betas must decrease strictly from 1 and stay >= 0");
    if (f.dtype != BM_DTYPE_F32 || f.compute != BM_COMPUTE_BF16)
        throw Error(BM_EUNSUPPORTED, "parallel tempering runs on the tensor-core engine only (float32 models, compute bf16)");
    if (f.v_kind != BM_UNIT_BERNOULLI)
        throw Error(BM_EUNSUPPORTED, "parallel tempering is not supported with gaussian visibles (a tempered gaussian needs variance sigma^2 / beta)");
    for (int i = 0; i < f.n_layers; ++i)
        if (f.h_kinds[i] != BM_UNIT_BERNOULLI) throw Error(BM_EUNSUPPORTED, "parallel tempering is not supported with multinomial hidden layers");
    if (ctx->nranks > 1) throw Error(BM_EUNSUPPORTED, "parallel tempering is not supported on a context with a communicator");
    BM_REQUIRE(f.sample_v != 0, "parallel tempering needs sampled visible states (sample_v): the swap compares energies of states");
    for (int i = 0; i < f.n_layers; ++i)
        BM_REQUIRE(f.sample_h[i] != 0, "parallel tempering needs sampled hidden states (sample_h of every layer): the swap compares energies of states");
}

template <typename T>
struct Dbm : DbmBase {
    int L, V, M, B;
    std::vector<int> Hs, h_kinds, sample_h;
    std::vector<double> h_n_samples, sp_target, sp_cost;
    int v_kind, sample_vis, max_mf;
    double mf_tol, l2, max_norm, damping;
    DevBuf<T> vb, dvb, sigma, v, v2, v3, Xd, xsum, vsum, recon, rowtmp;
    std::vector<DevBuf<T>> h3;
    std::vector<DevBuf<T>> W, dW, hb, dhb, qm, mm, pen, norm, G, musum, hsum;
    std::vector<DevBuf<T>> mu, mu2, h, h2, t;
    DevBuf<unsigned int> flag;
    DevBuf<double> scal, rowd;
    int xcap = 0;
    DevBuf<T> dpbuf;        // data parallelism: the step's statistics packed for ONE sum-allreduce

    static int size_of(int idx, int V, const std::vector<int>& Hs) { return idx == 0 ? V : Hs[idx - 1]; }
    int nranks() const { return ctx->nranks > 1 ? ctx->nranks : 1; }
    uint32_t particle_row0() const { return ctx->nranks > 1 ? (uint32_t)ctx->rank * (uint32_t)M : 0u; }   // global index of local particle 0

    // [G_0 | ... | musum_0 | hsum_0 | ... | xsum | vsum] -> one allreduce -> back (no-op on a single rank)
    void allreduce_step_statistics() {
        if (ctx->nranks <= 1) return;
        std::vector<std::pair<T*, size_t>> parts;
        int in = V;
        for (int i = 0; i < L; ++i) { parts.push_back({G[i].p, (size_t)in * Hs[i]}); in = Hs[i]; }
        for (int i = 0; i < L; ++i) { parts.push_back({musum[i].p, (size_t)Hs[i]}); parts.push_back({hsum[i].p, (size_t)Hs[i]}); }
        parts.push_back({xsum.p, (size_t)V}); parts.push_back({vsum.p, (size_t)V});
        size_t total = 0;
        for (auto& p : parts) total += p.second;
        dpbuf.ensure(total);
        size_t off = 0;
        for (auto& p : parts) { BM_CUDA(cudaMemcpyAsync(dpbuf.p + off, p.first, p.second * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream)); off += p.second; }
        allreduce_sum(ctx, dpbuf.p, total, sizeof(T) == 8);
        off = 0;
        for (auto& p : parts) { BM_CUDA(cudaMemcpyAsync(p.first, dpbuf.p + off, p.second * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream)); off += p.second; }
    }
    // mean of a per-rank mean over equally sized shards
    double allreduce_mean(double local) {
        if (ctx->nranks <= 1) return local;
        BM_CUDA(cudaMemcpyAsync(scal.p + 2, &local, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        allreduce_sum(ctx, scal.p + 2, 1, true);
        double out = 0.0;
        BM_CUDA(cudaMemcpyAsync(&out, scal.p + 2, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        return out / ctx->nranks;
    }

    Dbm(Ctx* c, const bm_dbm_cfg& f) {
        ctx = c; L = f.n_layers; V = f.n_visible; M = f.n_particles; B = f.batch_size;
        for (int i = 0; i < L; ++i) {
            Hs.push_back(f.n_hiddens[i]); h_kinds.push_back(f.h_kinds[i]); sample_h.push_back(f.sample_h[i]);
            h_n_samples.push_back(f.h_n_samples ? f.h_n_samples[i] : 100.0);
            sp_target.push_back(f.sparsity_target[i]); sp_cost.push_back(f.sparsity_cost[i]);
        }
        v_kind = f.v_kind; sample_vis = f.sample_v; max_mf = f.max_mf_updates;
        mf_tol = f.mf_tol; l2 = f.l2; max_norm = f.max_norm; damping = f.sparsity_damping;
        W.resize(L); dW.resize(L); hb.resize(L); dhb.resize(L); qm.resize(L); mm.resize(L); pen.resize(L); norm.resize(L);
        G.resize(L); musum.resize(L); hsum.resize(L); mu.resize(L); mu2.resize(L); h.resize(L); h2.resize(L); t.resize(L);
        vb.ensure(V); dvb.ensure(V); xsum.ensure(V); vsum.ensure(V);
        v.ensure((size_t)M * V); v2.ensure((size_t)M * V);
        for (DevBuf<T>* b : {&vb, &dvb, &v, &v2}) b->zero(ctx->stream);
        int in = V;
        for (int i = 0; i < L; ++i) {
            const int H = Hs[i];
            W[i].ensure((size_t)in * H); dW[i].ensure((size_t)in * H); G[i].ensure((size_t)in * H);
            for (DevBuf<T>* b : {&hb[i], &dhb[i], &qm[i], &mm[i], &pen[i], &norm[i], &musum[i], &hsum[i]}) { b->ensure(H); b->zero(ctx->stream); }
            mu[i].ensure((size_t)B * H); mu2[i].ensure((size_t)B * H); h[i].ensure((size_t)M * H); h2[i].ensure((size_t)M * H);
            for (DevBuf<T>* b : {&W[i], &dW[i], &mu[i], &mu2[i], &h[i], &h2[i]}) b->zero(ctx->stream);
            in = H;
        }
        if (f.sigma) {
            std::vector<T> s(V);
            for (int i = 0; i < V; ++i) s[i] = (T)f.sigma[i];
            sigma.ensure(V);
            BM_CUDA(cudaMemcpyAsync(sigma.p, s.data(), V * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        }
        flag.ensure(1); scal.ensure(8);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        reserve_x(B);
    }

    void reserve_x(int rows) {
        if (rows <= xcap) return;
        BM_REQUIRE(rows <= B, "a DBM batch may not exceed batch_size (the variational parameters are [batch_size, H])");
        xcap = rows;
        Xd.ensure((size_t)rows * V); recon.ensure((size_t)rows * V); rowtmp.ensure(rows);
        rowd.ensure(rows);
        for (int i = 0; i < L; ++i) t[i].ensure((size_t)rows * Hs[i]);
    }

    static std::string sfx(int i) { return i == 0 ? std::string() : "_" + std::to_string(i); }

    DevBuf<T>* by_name(const std::string& name, size_t* count) {
        if (name == "vb") { *count = V; return &vb; }
        if (name == "dvb") { *count = V; return &dvb; }
        if (name == "v") { *count = (size_t)M * V; return &v; }
        if (name == "sigma") { *count = V; return &sigma; }
        int in = V;
        for (int i = 0; i < L; ++i) {
            const std::string s = sfx(i);
            const int H = Hs[i];
            if (name == "W" + s) { *count = (size_t)in * H; return &W[i]; }
            if (name == "dW" + s) { *count = (size_t)in * H; return &dW[i]; }
            if (name == "hb" + s) { *count = H; return &hb[i]; }
            if (name == "dhb" + s) { *count = H; return &dhb[i]; }
            if (name == "q_means" + s) { *count = H; return &qm[i]; }
            if (name == "mu_means" + s) { *count = H; return &mm[i]; }
            if (name == "mu" + s) { *count = (size_t)B * H; return &mu[i]; }
            if (name == "h" + s) { *count = (size_t)M * H; return &h[i]; }
            in = H;
        }
        throw Error(BM_EINVAL, "unknown variable '" + name + "'");
    }
    void set_param(const char* name, const void* host, size_t bytes) override {
        size_t cnt; DevBuf<T>* b = by_name(name, &cnt);
        BM_REQUIRE(b->p != nullptr && bytes == cnt * sizeof(T), std::string("size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpyAsync(b->p, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void get_param(const char* name, void* host, size_t bytes) override {
        size_t cnt; DevBuf<T>* b = by_name(name, &cnt);
        BM_REQUIRE(b->p != nullptr && bytes == cnt * sizeof(T), std::string("size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpyAsync(host, b->p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    void init_particles(uint64_t seed) override {
        // layer.init(batch_size=n_particles): dbm.py:362-383, layers.py:43-45,59-63,78-82
        for (int idx = 0; idx <= L; ++idx) {
            const int n = size_of(idx, V, Hs);
            const int kind = idx == 0 ? v_kind : h_kinds[idx - 1];
            T* dst = idx == 0 ? v.p : h[idx - 1].p;
            for (int r0 = 0; r0 < M; r0 += 32768) {          // grid.y (the particle) is limited to 65535
                const int rows = M - r0 < 32768 ? M - r0 : 32768;
                dim3 grid(((n + 3) / 4 + 127) / 128, rows);
                particle_init_kernel<T><<<grid, 128, 0, ctx->stream>>>(dst + (size_t)r0 * n, rows, n, kind, sigma.p,
                                                                       make_rng(seed, SITE_PARTICLE_INIT, idx, 0, particle_row0() + (uint32_t)r0));
                count_launch(ctx);
            }
            BM_REQUIRE(kind != BM_UNIT_MULTINOMIAL || ctx->nranks <= 1, "multinomial layers are not supported with sharded particles");
            if (kind == BM_UNIT_MULTINOMIAL) {       // t /= reduce_sum(t) over the whole tensor
                launch_mean_combine<T>(ctx, dst, (const T*)nullptr, 0.0, (int)((size_t)M * n), scal.p);   // mean
                // total = mean * count: fold the count into the divisor on the host side of the kernel
                double mean = 0.0;
                BM_CUDA(cudaMemcpyAsync(&mean, scal.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
                BM_CUDA(cudaStreamSynchronize(ctx->stream));
                const double total = mean * (double)M * n;
                BM_CUDA(cudaMemcpyAsync(scal.p + 1, &total, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
                scale_all_kernel<T><<<592, 256, 0, ctx->stream>>>(dst, (size_t)M * n, scal.p + 1);
                count_launch(ctx);
            }
        }
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // ---- one fused conditional: act(scale_a * (A1 W_i [+ A2 W_{i+1}^T]) + scale_b * b_i) -----------------
    void hidden_op(int i, const T* below, const T* above, T* means_out, T* states_out, bool sample, int rows,
                   T acc_scale, T bias_scale, RngKey rng) {
        LayerOp<T> op;
        const int in = size_of(i, V, Hs), H = Hs[i];
        op.M = rows; op.N = H;
        op.A1 = below; op.lda1 = in; op.K1 = in; op.B1 = W[i].p; op.ldb1 = H; op.b1_trans = 0;
        if (above) { op.A2 = above; op.lda2 = Hs[i + 1]; op.K2 = Hs[i + 1]; op.B2 = W[i + 1].p; op.ldb2 = Hs[i + 1]; op.b2_trans = 1; }
        op.acc_scale = acc_scale; op.bias_scale = bias_scale; op.bias = hb[i].p;
        op.means = means_out; op.ldm = H; op.rng = rng;
        if (h_kinds[i] == BM_UNIT_BERNOULLI) {
            op.act = ACT_SIGMOID;
            if (sample) { op.sample = SMP_BERNOULLI; op.states = states_out; op.lds = H; }
            launch_layer_op<T>(ctx, op);
        } else if (h_kinds[i] == BM_UNIT_MULTINOMIAL) {
            op.act = ACT_LINEAR;
            launch_layer_op<T>(ctx, op);
            launch_softmax_rows<T>(ctx, means_out, H, rows, H, (T)h_n_samples[i]);
            if (sample) launch_multinomial_rows<T>(ctx, means_out, H, rows, H, (int)h_n_samples[i], states_out, H, rng);
        } else {
            throw Error(BM_EUNSUPPORTED, "gaussian hidden layers are not supported");
        }
    }
    void visible_op(const T* h0, T* means_out, T* states_out, bool sample, int rows, RngKey rng) {
        LayerOp<T> op;
        op.M = rows; op.N = V;
        op.A1 = h0; op.lda1 = Hs[0]; op.K1 = Hs[0]; op.B1 = W[0].p; op.ldb1 = Hs[0]; op.b1_trans = 1;
        op.bias = vb.p; op.means = means_out; op.ldm = V; op.rng = rng;
        if (v_kind == BM_UNIT_BERNOULLI) {
            op.act = ACT_SIGMOID;
            if (sample) { op.sample = SMP_BERNOULLI; op.states = states_out; op.lds = V; }
        } else if (v_kind == BM_UNIT_GAUSSIAN) {
            op.act = ACT_LINEAR; op.sigma = sigma.p;
            if (sample) { op.sample = SMP_GAUSSIAN; op.noise_sigma = sigma.p; op.states = states_out; op.lds = V; }
        } else throw Error(BM_EUNSUPPORTED, "multinomial visible layers are not supported");
        launch_layer_op<T>(ctx, op);
    }

    // dbm.py:385-427.  Hn[i] receive the new hidden values (states when sampled, else means)
    void gibbs_step(const T* vin, std::vector<const T*> Hin, std::vector<T*> Hn, T* v_new, bool update_v, bool sample,
                    int rows, uint64_t seed, uint32_t tstep, uint32_t tick) {
        for (int i = 0; i < L; ++i) {
            const T* below = i == 0 ? vin : Hn[i - 1];
            const T* above = (i + 1 < L) ? Hin[i + 1] : nullptr;
            const bool smp = sample && sample_h[i];
            // when sampling, means go to the scratch t[] (rows <= M may exceed xcap: use h2 as mean target)
            hidden_op(i, below, above, Hn[i], Hn[i], smp, rows, T(1), T(1), make_rng(seed, SITE_DBM_H + i, tstep, tick, particle_row0()));
        }
        if (update_v) {
            const bool smp = sample && sample_vis;
            visible_op(Hn[0], v_new, v_new, smp, rows, make_rng(seed, SITE_DBM_V, tstep, tick, particle_row0()));
        }
    }

    const T* upload(const void* X, int rows) {
        reserve_x(rows);
        BM_CUDA(cudaMemcpyAsync(Xd.p, X, (size_t)rows * V * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        return Xd.p;
    }

    // ---- E-step (dbm.py:429-478) ------------------------------------------------------------------------
    int mean_field(const T* X, int rows) {
        // approximate-inference initialisation of mu_new: only enters the first convergence test
        for (int i = 0; i < L; ++i) {
            const T* below = i == 0 ? X : mu2[i - 1].p;
            const T sc = (i == 0 || i < L - 1) ? T(2) : T(1);            // :438, :441-442
            hidden_op(i, below, nullptr, mu2[i].p, nullptr, false, rows, sc, T(1), RngKey{});
        }
        std::vector<T*> cur(L), nxt(L);
        for (int i = 0; i < L; ++i) { cur[i] = mu[i].p; nxt[i] = mu2[i].p; }
        int step = 0;
        while (step < max_mf) {
            BM_CUDA(cudaMemsetAsync(flag.p, 0, sizeof(unsigned int), ctx->stream));
            for (int i = 0; i < L; ++i) {
                const size_t n = (size_t)rows * Hs[i];
                max_abs_diff_kernel<T><<<ctx->sm_count, 256, 0, ctx->stream>>>(cur[i], nxt[i], n, flag.p);
                count_launch(ctx);
            }
            allreduce_max_u32(ctx, flag.p, 1);           // sharded rows: every rank runs the same number of sweeps
            unsigned int bits = 0;
            BM_CUDA(cudaMemcpyAsync(&bits, flag.p, sizeof(bits), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
            float diff; memcpy(&diff, &bits, sizeof(diff));
            if (!((T)diff > (T)mf_tol)) break;                            // :451-452
            std::vector<const T*> Hin(cur.begin(), cur.end());
            gibbs_step(X, Hin, nxt, nullptr, false, false, rows, 0, 0, 0);
            std::swap(cur, nxt);                                          // :457
            ++step;
        }
        for (int i = 0; i < L; ++i)
            if (cur[i] != mu[i].p)
                BM_CUDA(cudaMemcpyAsync(mu[i].p, cur[i], (size_t)rows * Hs[i] * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
        return step;
    }

    // ---- PCD particle update (dbm.py:480-509) --------------------------------------------------------------
    void particles_update(int n_steps, bool sample, uint64_t seed, uint32_t tick, int t0, bool commit, T** v_final) {
        sv_k = 0;                                     // h2 / v2 are about to be overwritten: no sample_v chain to report
        std::vector<T*> cur(L), nxt(L), spare(L);
        for (int i = 0; i < L; ++i) { cur[i] = h[i].p; nxt[i] = h2[i].p; spare[i] = nullptr; }
        T* vc = v.p; T* vn = v2.p; T* vspare = nullptr;
        if (!commit) {      // an uncommitted run must never write the persistent particles: ping-pong on scratch
            v3.ensure((size_t)M * V); vspare = v3.p;
            if (h3.size() != (size_t)L) h3.resize(L);
            for (int i = 0; i < L; ++i) { h3[i].ensure((size_t)M * Hs[i]); spare[i] = h3[i].p; }
        }
        for (int s = 0; s < n_steps; ++s) {
            std::vector<const T*> Hin(cur.begin(), cur.end());
            gibbs_step(vc, Hin, nxt, vn, true, sample, M, seed, (uint32_t)(t0 + s + 1), tick);
            if (!commit && s == 0) {                 // from now on alternate between the two scratch sets
                cur = nxt; nxt = spare; vc = vn; vn = vspare;
            } else { std::swap(cur, nxt); std::swap(vc, vn); }
        }
        if (commit) {
            for (int i = 0; i < L; ++i)
                if (cur[i] != h[i].p) BM_CUDA(cudaMemcpyAsync(h[i].p, cur[i], (size_t)M * Hs[i] * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
            if (vc != v.p) BM_CUDA(cudaMemcpyAsync(v.p, vc, (size_t)M * V * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
            if (v_final) *v_final = v.p;
        } else if (v_final) *v_final = vc;
    }

    void reconstruction(int rows) { visible_op(mu[0].p, recon.p, nullptr, false, rows, RngKey{}); }    // :626-628

    double msre(const T* X, int rows) {
        reconstruction(rows);
        launch_sqdiff_mean<T>(ctx, X, V, recon.p, V, rows, V, (double)rows * V, scal.p);
        double hval = 0.0;
        BM_CUDA(cudaMemcpyAsync(&hval, scal.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        return allreduce_mean(hval);
    }

    void train_step(const void* Xh, int rows, double lr, double mom, int k, uint64_t seed, uint32_t tick, int want, double* out) override {
        BM_REQUIRE(rows >= 1, "empty batch");
        const T* X = upload(Xh, rows);
        const int n_mf = mean_field(X, rows);
        particles_update(k, true, seed, tick, 0, true, nullptr);
        if (want) { BM_REQUIRE(out, "metrics requested without a buffer"); out[0] = msre(X, rows); out[1] = (double)n_mf; }
        const int nr = nranks();
        const T N = (T)((double)B * nr), Mp = (T)((double)M * nr);      // configured (global) sizes, as the reference (dbm.py:254-255)
        const T rows_g = (T)((double)rows * nr);                         // rows present in this step on all ranks
        // gradients (dbm.py:558-568): G_i = pos/N - neg/M
        for (int i = 0; i < L; ++i) {
            LayerOp<T> g;
            const int in = size_of(i, V, Hs), H = Hs[i];
            g.M = in; g.N = H; g.a_trans = 1;
            g.A1 = i == 0 ? X : mu[i - 1].p; g.lda1 = in; g.K1 = rows; g.B1 = mu[i].p; g.ldb1 = H;
            g.A2 = i == 0 ? v.p : h[i - 1].p; g.lda2 = in; g.K2 = M; g.B2 = h[i].p; g.ldb2 = H;
            g.s1 = T(1) / N; g.s2 = T(-1) / Mp;
            g.means = G[i].p; g.ldm = H;
            launch_layer_op<T>(ctx, g);
            launch_colsum<T>(ctx, mu[i].p, H, (const T*)nullptr, 0, rows, H, T(1), T(0), musum[i].p);
            launch_colsum<T>(ctx, h[i].p, H, (const T*)nullptr, 0, M, H, T(1), T(0), hsum[i].p);
        }
        launch_colsum<T>(ctx, X, V, (const T*)nullptr, 0, rows, V, T(1), T(0), xsum.p);
        launch_colsum<T>(ctx, v.p, V, (const T*)nullptr, 0, M, V, T(1), T(0), vsum.p);
        allreduce_step_statistics();
        dbm_vbias_kernel<T><<<(V + 255) / 256, 256, 0, ctx->stream>>>(V, xsum.p, vsum.p, rows_g, Mp, vb.p, dvb.p, (T)lr, (T)mom);
        count_launch(ctx);
        for (int i = 0; i < L; ++i) {
            const int in = size_of(i, V, Hs), H = Hs[i];
            BM_REQUIRE(i < H, "the reference's sparsity update indexes element i of layer i's unit vector");
            // dhb uses reduce_mean over the rows present (mu) and over the particles (H)
            dbm_sparsity_bias_kernel<T><<<(H + 255) / 256, 256, 0, ctx->stream>>>(
                H, i, musum[i].p, hsum[i].p, rows_g, Mp, qm[i].p, mm[i].p, pen[i].p, hb[i].p, dhb[i].p,
                (T)damping, (T)sp_cost[i], (T)sp_target[i], (T)lr, (T)mom);
            count_launch(ctx);
            launch_weight_update<T>(ctx, G[i].p, H, T(1), W[i].p, dW[i].p, in, H, pen[i].p, (T)l2, (T)lr, (T)mom, nullptr, 0);
            colnorm_kernel<T><<<(H + 31) / 32, dim3(32, 8), 0, ctx->stream>>>(W[i].p, in, H, norm[i].p);       // :511-513
            count_launch(ctx);
            max_norm_scale_kernel<T><<<dim3((H + 255) / 256, in < 32768 ? in : 32768), 256, 0, ctx->stream>>>(W[i].p, in, H, norm[i].p, (T)max_norm);
            count_launch(ctx);
        }
    }

    void val_metrics(const void* Xh, int rows, int k, uint64_t seed, uint32_t tick, double* out) override {
        const T* X = upload(Xh, rows);
        const int n_mf = mean_field(X, rows);
        particles_update(k, true, seed, tick, 0, true, nullptr);          // dbm.py:523 control dependencies
        out[0] = msre(X, rows); out[1] = (double)n_mf;
    }
    void transform(const void* Xh, int rows, void* out) override {
        const T* X = upload(Xh, rows);
        mean_field(X, rows);
        BM_CUDA(cudaMemcpyAsync(out, mu[L - 1].p, (size_t)rows * Hs[L - 1] * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void reconstruct(const void* Xh, int rows, void* out) override {
        const T* X = upload(Xh, rows);
        mean_field(X, rows);
        reconstruction(rows);
        BM_CUDA(cudaMemcpyAsync(out, recon.p, (size_t)rows * V * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void log_proba(const void* Xh, int rows, double* out) override {
        BM_REQUIRE(L == 2, "log_proba is defined for 2 hidden layers");
        const T* X = upload(Xh, rows);
        mean_field(X, rows);
        LayerOp<T> a;                       // t1 = X W_0
        a.M = rows; a.N = Hs[0]; a.A1 = X; a.lda1 = V; a.K1 = V; a.B1 = W[0].p; a.ldb1 = Hs[0]; a.means = t[0].p; a.ldm = Hs[0];
        launch_layer_op<T>(ctx, a);
        LayerOp<T> b;                       // t2 = mu_0 W_1
        b.M = rows; b.N = Hs[1]; b.A1 = mu[0].p; b.lda1 = Hs[0]; b.K1 = Hs[0]; b.B1 = W[1].p; b.ldb1 = Hs[1]; b.means = t[1].p; b.ldm = Hs[1];
        launch_layer_op<T>(ctx, b);
        dbm_bound_rows_kernel<T><<<(rows + 7) / 8, dim3(32, 8), 0, ctx->stream>>>(X, V, mu[0].p, Hs[0], mu[1].p, Hs[1], t[0].p, t[1].p,
                                                                                 vb.p, hb[0].p, hb[1].p, rows, rowd.p);
        count_launch(ctx);
        BM_CUDA(cudaMemcpyAsync(out, rowd.p, (size_t)rows * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void sample_v(int k, uint64_t seed, uint32_t tick, void* out) override {
        // dbm.py:641-648: k sampled sweeps (committed), k more without sampling; v <- their visible means
        particles_update(k, true, seed, tick, 0, true, nullptr);
        T* vf = nullptr;
        particles_update(k, false, seed, tick, k, false, &vf);
        if (vf != v.p) BM_CUDA(cudaMemcpyAsync(v.p, vf, (size_t)M * V * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
        BM_CUDA(cudaMemcpyAsync(out, v.p, (size_t)M * V * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        sv_k = k;
    }
    // The uncommitted sweeps of the last sample_v ping-pong on scratch: sweep t (1..k) is in h2 / v2 for odd t, h3 / v3 for even
    // t, untouched until the next particle update.  "v", "h", "h_1", ...: sweep k; + "_prev": sweep k - 1 (k >= 2).  [M, n].
    int sv_k = 0;                                 // sweeps of the last sample_v's uncommitted run (0: none to report)
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
        const T* src = nullptr; int width = 0;
        if (n == "v") { src = odd ? v2.p : v3.p; width = V; }
        else
            for (int i = 0; i < L; ++i)
                if (n == "h" + sfx(i)) { src = odd ? h2[i].p : h3[i].p; width = Hs[i]; }
        BM_REQUIRE(src, std::string("sample_v_debug: unknown name '") + name + "'");
        BM_REQUIRE(bytes == (size_t)M * width * sizeof(T), std::string("sample_v_debug: size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpyAsync(host, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // ---- clamped Gibbs chains (DESIGN.md §5.9) ---------------------------------------------------------------------------
    // Scratch of its own ([batch_size, n] per layer, allocated on first use): two chain states per layer -- index t % 2 holds
    // sweep t, 0 the start -- the batch, its mask and the visible means.  Nothing the model or the particles hold is touched.
    DevBuf<T> fX, fmean, fout, fv[2];
    std::vector<DevBuf<T>> fh[2];
    DevBuf<uint8_t> fmask;
    int f_rows = 0, f_k = 0;                     // the last fill (0: none yet)
    void fill(const void* Xh, const uint8_t* mask, const int32_t* labels, int rows, uint32_t row0, int k, uint64_t seed,
              uint32_t tick, void* out) override {
        check_fill_args(mask, labels, rows, k, B, V, 0);
        if (fh[0].empty()) {
            for (DevBuf<T>* b : {&fX, &fmean, &fout, &fv[0], &fv[1]}) b->ensure((size_t)B * V);
            fmask.ensure((size_t)B * V);
            for (int s = 0; s < 2; ++s) { fh[s].resize(L); for (int i = 0; i < L; ++i) fh[s][i].ensure((size_t)B * Hs[i]); }
        }
        f_rows = 0;
        BM_CUDA(cudaMemcpyAsync(fX.p, Xh, (size_t)rows * V * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        BM_CUDA(cudaMemcpyAsync(fmask.p, mask, (size_t)rows * V, cudaMemcpyHostToDevice, ctx->stream));
        // start: v0 = X where observed, the visible mean with nothing above it (act(0 W_0' + b)) elsewhere
        BM_CUDA(cudaMemsetAsync(fh[1][0].p, 0, (size_t)rows * Hs[0] * sizeof(T), ctx->stream));
        visible_op(fh[1][0].p, fv[0].p, nullptr, false, rows, RngKey{});
        launch_dbm_fill_clamp<T>(ctx, fmask.p, fX.p, V, fv[0].p, V, rows, V);
        for (int i = 0; i < L; ++i) {                // h0: the E-step's approximate-inference pass on v0 (dbm.py:434-446)
            const T sc = (i == 0 || i < L - 1) ? T(2) : T(1);
            hidden_op(i, i == 0 ? fv[0].p : fh[0][i - 1].p, nullptr, fh[0][i].p, nullptr, false, rows, sc, T(1), RngKey{});
        }
        for (int t = 1; t <= k; ++t) {               // the particle sweep of gibbs_step, drawing at rows row0 + r
            const int c = (t - 1) & 1, n = t & 1;
            for (int i = 0; i < L; ++i) {
                const T* below = i == 0 ? fv[c].p : fh[n][i - 1].p;
                const T* above = (i + 1 < L) ? fh[c][i + 1].p : nullptr;
                hidden_op(i, below, above, fh[n][i].p, fh[n][i].p, sample_h[i] != 0, rows, T(1), T(1), make_rng(seed, SITE_DBM_H + i, t, tick, row0));
            }
            visible_op(fh[n][0].p, fv[n].p, fv[n].p, sample_vis != 0, rows, make_rng(seed, SITE_DBM_V, t, tick, row0));
            launch_dbm_fill_clamp<T>(ctx, fmask.p, fX.p, V, fv[n].p, V, rows, V);
        }
        visible_op(fh[k & 1][0].p, fmean.p, nullptr, false, rows, RngKey{});        // p(v | h_1 of the last sweep)
        launch_dbm_fill_out<T, T>(ctx, fmask.p, fX.p, fmean.p, V, fout.p, rows, V);
        BM_CUDA(cudaMemcpyAsync(out, fout.p, (size_t)rows * V * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        f_rows = rows; f_k = k;
    }
    // "v", "h", "h_1", ...: the last sweep; the same with "_prev": the sweep before it (the start after one sweep); "mean": the
    // visible means before the observed units are put back.  [rows, n] in the storage dtype.
    void fill_debug(const char* name, void* host, size_t bytes) override {
        BM_REQUIRE(f_rows > 0, "fill_debug: no fill has run on this DBM");
        std::string n(name);
        int which = f_k & 1;
        const std::string suffix = "_prev";
        if (n.size() > suffix.size() && n.compare(n.size() - suffix.size(), suffix.size(), suffix) == 0) {
            n = n.substr(0, n.size() - suffix.size()); which = 1 - which;
        }
        const T* src = nullptr; int width = 0;
        if (n == "v") { src = fv[which].p; width = V; }
        else if (n == "mean" && std::string(name) == "mean") { src = fmean.p; width = V; }
        else for (int i = 0; i < L; ++i) if (n == "h" + sfx(i)) { src = fh[which][i].p; width = Hs[i]; }
        BM_REQUIRE(src, std::string("fill_debug: unknown name '") + name + "'");
        BM_REQUIRE(bytes == (size_t)f_rows * width * sizeof(T), std::string("fill_debug: size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpyAsync(host, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // ---- AIS (dbm.py:650-736) ---------------------------------------------------------------------------------
    // The runs are independent chains: run r draws from row r of the AIS sites whichever rank or call computes it
    // (row0 = first_run), so a ladder sharded over ranks, or cut into several calls, reproduces the unsharded one.
    bool has_base(const float* const* base) const {
        for (int j = 0; base && j <= L; ++j)
            if (base[j]) return true;
        return false;
    }
    virtual void ais_check(int R, int n_betas, int k, const float* const* base) const {
        if (has_base(base))
            throw Error(BM_EUNSUPPORTED, "AIS from a base-rate model runs on the tensor-core engine (float32 models, BM_COMPUTE_BF16), "
                                         "not on the CUDA-core engine");
        BM_REQUIRE(L == 2 && v_kind == BM_UNIT_BERNOULLI && h_kinds[0] == BM_UNIT_BERNOULLI && h_kinds[1] == BM_UNIT_BERNOULLI,
                   "AIS is defined for a 2-layer binary DBM");
        BM_REQUIRE(R >= 1 && n_betas >= 2 && k >= 1, "bad AIS arguments");
    }
    // runs [first, first + n) of a ladder of `total` runs -> out[0..n)
    void ais_slice(int n, uint32_t first, int n_betas, int k, uint64_t seed, const float* const* base, double* out, bool reduce,
                   int total, int offset) {
        DevBuf<double> all;
        all.ensure(total);
        all.zero(ctx->stream);
        // the unit kernels index the run with grid.y (limit 65535) and the workspaces grow with the runs: long ladders go in
        // chunks -- run r draws from row r whatever the chunking
        const int chunk = 32768;
        for (int done = 0; done < n; done += chunk)
            ais_local(std::min(chunk, n - done), first + (uint32_t)done, n_betas, k, seed, base, all.p + offset + done);
        if (reduce) allreduce_sum(ctx, all.p, (size_t)total, true);        // every rank ends with every run
        std::vector<double> hw(total);
        BM_CUDA(cudaMemcpyAsync(hw.data(), all.p, (size_t)total * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        // :731-734 -- the reference multiplies by `tf.cast(tf.log(2.), dtype)`: the FLOAT32 value of log 2 in every dtype
        int units = V;
        for (int i = 0; i < L; ++i) units += Hs[i];
        double logZ0 = (double)units * 0.693147182464599609375;
        if (has_base(base)) {               // log Z_A = sum_j sum_n softplus(a_{j,n}) in float64 (a layer without a base: a = 0)
            logZ0 = 0.0;
            for (int j = 0; j <= L; ++j)
                for (int c = 0, w = j == 0 ? V : Hs[j - 1]; c < w; ++c) {
                    const double a = base[j] ? (double)base[j][c] : 0.0;
                    logZ0 += std::max(a, 0.0) + std::log1p(std::exp(-std::fabs(a)));
                }
        }
        for (int r = 0; r < total; ++r) out[r] = hw[r] + logZ0;
    }
    void ais(int R, int n_betas, int k, uint64_t seed, const float* const* base, double* out) override {
        ais_check(R, n_betas, k, base);
        // with a communicator the runs are sharded over the ranks (SURVEY 8e) and gathered by one sum-allreduce of R doubles
        const int nr = ctx->nranks > 1 ? ctx->nranks : 1, rk = ctx->nranks > 1 ? ctx->rank : 0;
        const int lo = (int)((long long)R * rk / nr), hi = (int)((long long)R * (rk + 1) / nr);
        ais_slice(hi - lo, (uint32_t)lo, n_betas, k, seed, base, out, nr > 1, R, lo);
    }
    void ais_rows(int R, int n_betas, int k, uint64_t seed, uint32_t first_run, const float* const* base, double* out) override {
        ais_check(R, n_betas, k, base);
        ais_slice(R, first_run, n_betas, k, seed, base, out, false, R, 0);
    }
    // R chains starting at global run `row0`; their log-weights (without log Z_0) are ADDED to logw_out[0..R) (device, zeroed).
    // This engine has no base (ais_check refuses one).
    virtual void ais_local(int R, uint32_t row0, int n_betas, int k, uint64_t seed, const float* const*, double* logw_out) {
        const int H0 = Hs[0], H1 = Hs[1];
        DevBuf<T> x, xn, va, hc, pa, pb;
        struct { double* p; } logw{logw_out};
        x.ensure((size_t)R * H0); xn.ensure((size_t)R * H0); va.ensure((size_t)R * V); hc.ensure((size_t)R * H1);
        pa.ensure((size_t)R * V); pb.ensure((size_t)R * H1);
        const dim3 rgrid((R + 7) / 8), rblock(32, 8);
        auto pre = [&](const T* xs) {          // pa = x W_0^T + b ; pb = x W_1 + c_2   (beta-free, shared)
            LayerOp<T> a; a.M = R; a.N = V; a.A1 = xs; a.lda1 = H0; a.K1 = H0; a.B1 = W[0].p; a.ldb1 = H0; a.b1_trans = 1;
            a.bias = vb.p; a.means = pa.p; a.ldm = V; launch_layer_op<T>(ctx, a);
            LayerOp<T> b; b.M = R; b.N = H1; b.A1 = xs; b.lda1 = H0; b.K1 = H0; b.B1 = W[1].p; b.ldb1 = H1;
            b.bias = hb[1].p; b.means = pb.p; b.ldm = H1; launch_layer_op<T>(ctx, b);
        };
        auto accum = [&](const T* xs, double sign, double beta) {
            ais_accum_kernel<T><<<rgrid, rblock, 0, ctx->stream>>>(logw.p, sign, beta, xs, H0, hb[0].p, pa.p, V, pb.p, H1, R);
            count_launch(ctx);
        };
        T* xc = x.p; T* xo = xn.p;
        int it = 0;
        // transition T_beta(x): n_gibbs_steps times  v ~ p(v|x), h2 ~ p(h2|x), x' ~ p(x|v,h2)  at temperature beta.
        // `have_pre`: pa/pb already hold the pre-activations of the current x.
        auto transition = [&](T beta, bool have_pre) {
            for (int s = 0; s < k; ++s) {
                const uint32_t tick = (uint32_t)(it * k + s);
                if (!(have_pre && s == 0)) pre(xc);
                dim3 gv(((V + 3) / 4 + 127) / 128, R), gh(((H1 + 3) / 4 + 127) / 128, R);
                ais_unit_kernel<T><<<gv, 128, 0, ctx->stream>>>(pa.p, beta, va.p, R, V, sample_vis, make_rng(seed, SITE_AIS_V, 0, tick, row0));
                ais_unit_kernel<T><<<gh, 128, 0, ctx->stream>>>(pb.p, beta, hc.p, R, H1, sample_h[1], make_rng(seed, SITE_AIS_H2, 0, tick, row0));
                count_launch(ctx); count_launch(ctx);
                LayerOp<T> o;                 // x' = act(beta (v W_0 + h2 W_1^T), beta c_1)
                o.M = R; o.N = H0; o.A1 = va.p; o.lda1 = V; o.K1 = V; o.B1 = W[0].p; o.ldb1 = H0;
                o.A2 = hc.p; o.lda2 = H1; o.K2 = H1; o.B2 = W[1].p; o.ldb2 = H1; o.b2_trans = 1;
                o.acc_scale = beta; o.bias_scale = beta; o.bias = hb[0].p; o.act = ACT_SIGMOID;
                o.means = xo; o.ldm = H0; o.rng = make_rng(seed, SITE_AIS_H1, 0, tick, row0);
                if (sample_h[0]) { o.sample = SMP_BERNOULLI; o.states = xo; o.lds = H0; }
                launch_layer_op<T>(ctx, o);
                std::swap(xc, xo);
            }
            ++it;
        };
        // x_0 ~ Ber(1/2)   (:700-702)
        {
            dim3 g(((H0 + 3) / 4 + 127) / 128, R);
            launch_fill<T>(ctx, pb.p, (size_t)R * H1, T(0));
            launch_fill<T>(ctx, xo, (size_t)R * H0, T(0));          // pre-activation 0 -> p = 1/2
            ais_unit_kernel<T><<<g, 128, 0, ctx->stream>>>(xo, T(0), xc, R, H0, 1, make_rng(seed, SITE_AIS_INIT, 0, 0, row0));
            count_launch(ctx);
        }
        const T delta = (T)(1.0 / n_betas);
        transition(delta, false);                               // x_1 ~ T_1(x_1 | x_0)            :705
        pre(xc); accum(xc, -1.0, 0.0);                          // -log p_0(x_1)                  :708
        T beta = delta;
        while (beta < T(1) - delta + T(1e-5)) {                 // :710-711 (beta accumulates in the storage dtype)
            accum(xc, +1.0, (double)beta);                      // + log p_i(x_i)   (pa/pb of x_i are current)
            transition((T)(beta + delta), true);                // x_{i+1} ~ T_{i+1}
            pre(xc); accum(xc, -1.0, (double)beta);             // - log p_i(x_{i+1})
            beta = (T)(beta + delta);
        }
        accum(xc, +1.0, 1.0);                                   // + log p_M(x_M)                 :728
        BM_CUDA(cudaStreamSynchronize(ctx->stream));            // the workspaces above are released on return
    }
};

}  // namespace bm

#include "bm_dbm_tc.cuh"     // DbmTC: the same engine with every GEMM on the tensor cores (opt-in)
#include "bm_crbm_tc.cuh"    // ClassRbmTC: the classification RBM, a DbmTC of shape x - h - label (bm_crbm_*)
#include "bm_cdbm_tc.cuh"    // ClassDbmTC: the classification DBM, a DbmTC with a label layer on top (bm_dbm_cfg.n_classes)
#include "bm_dbm_exact.cuh"   // DbmTC::exact: exact log Z and log p*(v) over the odd layers' states (bm_dbm_exact)

using namespace bm;

// Centering (bm_dbm_cfg.centering / offset_rate): what is refused before anything is allocated.  0 is off.
static void check_centering_cfg(const Ctx* ctx, const bm_dbm_cfg& f) {
    if (f.centering == 0) return;
    BM_REQUIRE(std::isfinite(f.offset_rate) && f.offset_rate >= 0.0 && f.offset_rate <= 1.0, "centering: offset_rate must lie in [0, 1]");
    if (f.n_classes != 0) throw Error(BM_EUNSUPPORTED, "centering is not supported for classification DBMs (n_classes)");
    if (f.dtype != BM_DTYPE_F32 || f.compute != BM_COMPUTE_BF16)
        throw Error(BM_EUNSUPPORTED, "centering runs on the tensor-core engine only (float32 models, compute bf16)");
    if (!DbmTC::supports(f)) throw Error(BM_EUNSUPPORTED, "centering: the model does not run on the tensor-core engine");
    if (ctx->nranks > 1) throw Error(BM_EUNSUPPORTED, "centering is not supported on a context with a communicator");
}

extern "C" {

int bm_dbm_create(bm_ctx* hctx, const bm_dbm_cfg* cfg, bm_dbm** out) {
    BM_API_BEGIN
    Ctx* ctx = reinterpret_cast<Ctx*>(hctx);
    BM_REQUIRE(ctx && cfg && out, "null argument");
    BM_REQUIRE(cfg->n_layers >= 1 && cfg->n_layers <= 8 && cfg->n_visible > 0, "bad DBM shape");
    BM_REQUIRE(cfg->n_hiddens && cfg->h_kinds && cfg->sample_h && cfg->sparsity_target && cfg->sparsity_cost, "missing per-layer arrays");
    BM_REQUIRE(cfg->n_particles > 0 && cfg->batch_size > 0, "n_particles and batch_size must be positive");
    BM_REQUIRE(cfg->v_kind != BM_UNIT_GAUSSIAN || cfg->sigma, "gaussian visible layer needs sigma");
    BM_REQUIRE(cfg->n_classes >= 0 && cfg->n_classes != 1, "classification DBM: n_classes must be 0 (no label layer) or at least 2");
    check_centering_cfg(ctx, *cfg);
    if (cfg->n_classes >= 2) ClassDbmTC::check_cfg(ctx, *cfg);      // then n_temps <= 1: at most [1.0], no tempering
    check_pt_cfg(ctx, *cfg);
    if (cfg->n_temps >= 1 && !DbmTC::supports(*cfg)) throw Error(BM_EUNSUPPORTED, "parallel tempering: the model does not run on the tensor-core engine");
    BM_CUDA(cudaSetDevice(ctx->device));
    // BM_COMPUTE_BF16 (the Python mirror's default): float32 models with Bernoulli hidden layers run their GEMMs on the tensor
    // cores; every other combination keeps the storage-precision CUDA-core engine (as bm_rbm_create does for unit kinds the
    // tensor-core epilogue does not implement)
    DbmBase* d;
    CdbmShape s;
    if (cfg->n_classes >= 2) d = new ClassDbmTC(ctx, *cfg, s);
    else if (cfg->dtype == BM_DTYPE_F64) d = new Dbm<double>(ctx, *cfg);
    else if (cfg->compute == BM_COMPUTE_BF16 && DbmTC::supports(*cfg)) d = new DbmTC(ctx, *cfg);
    else d = new Dbm<float>(ctx, *cfg);
    *out = reinterpret_cast<bm_dbm*>(d);
    BM_API_END
}
void bm_dbm_destroy(bm_dbm* h) {
    if (!h) return;
    DbmBase* d = reinterpret_cast<DbmBase*>(h);
    cudaSetDevice(d->ctx->device);
    cudaStreamSynchronize(d->ctx->stream);
    delete d;
}
#define DBM(h) (reinterpret_cast<DbmBase*>(h))
#define DBM_ENTER(h) BM_REQUIRE((h) != nullptr, "null dbm handle"); BM_CUDA(cudaSetDevice(DBM(h)->ctx->device));

int bm_dbm_set_param(bm_dbm* h, const char* name, const void* host, size_t bytes) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(name && host, "null argument"); DBM(h)->set_param(name, host, bytes); BM_API_END
}
int bm_dbm_get_param(bm_dbm* h, const char* name, void* host, size_t bytes) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(name && host, "null argument"); DBM(h)->get_param(name, host, bytes); BM_API_END
}
int bm_dbm_init_particles(bm_dbm* h, uint64_t seed) { BM_API_BEGIN DBM_ENTER(h) DBM(h)->init_particles(seed); BM_API_END }
int bm_dbm_train_step(bm_dbm* h, const void* X, int32_t rows, double lr, double momentum, int32_t k, uint64_t seed,
                      uint32_t tick, int32_t want_metrics, double* out2) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X, "null batch");
    DBM(h)->train_step(X, rows, lr, momentum, k, seed, tick, want_metrics, out2);
    BM_API_END
}
int bm_dbm_train_step_labeled(bm_dbm* h, const void* X, const int32_t* labels, int32_t rows, double lr, double momentum,
                              int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, int32_t want_metrics, double* out2) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X && labels, "null argument");
    DBM(h)->train_step_labeled(X, labels, rows, lr, momentum, n_gibbs_steps, seed, tick, want_metrics, out2);
    BM_API_END
}
int bm_dbm_predict_proba(bm_dbm* h, const void* X, int32_t rows, float* out) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X && out, "null argument"); DBM(h)->predict_proba(X, rows, out); BM_API_END
}
int bm_dbm_val_metrics(bm_dbm* h, const void* X, int32_t rows, int32_t k, uint64_t seed, uint32_t tick, double* out2) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X && out2, "null argument"); DBM(h)->val_metrics(X, rows, k, seed, tick, out2); BM_API_END
}
int bm_dbm_transform(bm_dbm* h, const void* X, int32_t rows, void* out) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X && out, "null argument"); DBM(h)->transform(X, rows, out); BM_API_END
}
int bm_dbm_reconstruct(bm_dbm* h, const void* X, int32_t rows, void* out) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X && out, "null argument"); DBM(h)->reconstruct(X, rows, out); BM_API_END
}
int bm_dbm_log_proba(bm_dbm* h, const void* X, int32_t rows, double* out) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X && out, "null argument"); DBM(h)->log_proba(X, rows, out); BM_API_END
}
int bm_dbm_sample_v(bm_dbm* h, int32_t k, uint64_t seed, uint32_t tick, void* out) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(out, "null argument"); DBM(h)->sample_v(k, seed, tick, out); BM_API_END
}
int bm_dbm_ais_base(bm_dbm* h, int32_t n_runs, int32_t n_betas, int32_t k, uint64_t seed, const float* const* base, double* logZ) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(logZ, "null argument"); DBM(h)->ais(n_runs, n_betas, k, seed, base, logZ); BM_API_END
}
int bm_dbm_ais_base_rows(bm_dbm* h, int32_t n_runs, int32_t n_betas, int32_t k, uint64_t seed, uint32_t first_run,
                         const float* const* base, double* logZ) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(logZ, "null argument"); DBM(h)->ais_rows(n_runs, n_betas, k, seed, first_run, base, logZ); BM_API_END
}
int bm_dbm_ais(bm_dbm* h, int32_t n_runs, int32_t n_betas, int32_t k, uint64_t seed, double* logZ) {
    return bm_dbm_ais_base(h, n_runs, n_betas, k, seed, nullptr, logZ);
}
int bm_dbm_ais_rows(bm_dbm* h, int32_t n_runs, int32_t n_betas, int32_t k, uint64_t seed, uint32_t first_run, double* logZ) {
    return bm_dbm_ais_base_rows(h, n_runs, n_betas, k, seed, first_run, nullptr, logZ);
}
int bm_dbm_pt_counts(bm_dbm* h, int64_t* accepted, int64_t* proposed) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(accepted && proposed, "null argument"); DBM(h)->pt_counts(accepted, proposed); BM_API_END
}
int bm_dbm_fill(bm_dbm* h, const void* X, const uint8_t* mask, const int32_t* labels, int32_t rows, uint32_t row0,
                int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, void* out) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(X && mask && out, "null argument");
    DBM(h)->fill(X, mask, labels, rows, row0, n_gibbs_steps, seed, tick, out);
    BM_API_END
}
int bm_dbm_debug_last_fill(bm_dbm* h, const char* name, void* host, size_t bytes) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(name && host, "null argument"); DBM(h)->fill_debug(name, host, bytes); BM_API_END
}
int bm_dbm_exact(bm_dbm* h, const void* X, int32_t rows, double* log_p_star, double* log_Z) {
    BM_API_BEGIN DBM_ENTER(h) DBM(h)->exact(X, rows, log_p_star, log_Z); BM_API_END
}
int bm_dbm_ais_clamped(bm_dbm* h, const void* X, int32_t rows, uint32_t row0, int32_t n_runs, int32_t n_betas,
                       int32_t n_gibbs_steps, uint64_t seed, double* log_w) {
    BM_API_BEGIN DBM_ENTER(h) DBM(h)->ais_clamped(X, rows, row0, n_runs, n_betas, n_gibbs_steps, seed, log_w); BM_API_END
}
int bm_dbm_debug_exact_chunk(bm_dbm* h, int32_t log2_states) {
    BM_API_BEGIN DBM_ENTER(h)
    DbmTC* d = dynamic_cast<DbmTC*>(DBM(h));
    if (!d) throw Error(BM_EUNSUPPORTED, "exact log Z runs on the tensor-core engine");
    BM_REQUIRE(log2_states == 0 || (log2_states >= 1 && log2_states <= 30), "exact chunk: log2 of the states per launch in [1, 30], or 0");
    d->exact_chunk_bits = log2_states == 0 ? DbmTC::EXACT_CHUNK_BITS : log2_states;
    BM_API_END
}
int bm_dbm_debug_last_sample_v(bm_dbm* h, const char* name, void* host, size_t bytes) {
    BM_API_BEGIN DBM_ENTER(h) BM_REQUIRE(name && host, "null argument"); DBM(h)->sample_v_debug(name, host, bytes); BM_API_END
}

int bm_debug_dbm_multinomial_rows(bm_ctx* hctx, const float* pre, int32_t rows, int32_t cols, double n_samples, int32_t n_draws,
                                  uint64_t seed, uint32_t site, uint32_t t, uint32_t tick, uint16_t* out_bf, float* out_f32,
                                  float* ref_means, float* ref_counts) {
    BM_API_BEGIN
    Ctx* ctx = reinterpret_cast<Ctx*>(hctx);
    BM_REQUIRE(ctx && pre && out_bf && out_f32 && ref_means && rows > 0 && cols > 0 && n_draws >= 0, "bad argument");
    BM_REQUIRE(n_draws == 0 || ref_counts, "bad argument");
    BM_CUDA(cudaSetDevice(ctx->device));
    const size_t n = (size_t)rows * cols;
    DevBuf<float> x, ref, cnt, f32;
    DevBuf<bf16_t> bf;
    x.ensure(n); ref.ensure(n); cnt.ensure(n); f32.ensure(n); bf.ensure(n);
    BM_CUDA(cudaMemcpyAsync(x.p, pre, n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    BM_CUDA(cudaMemcpyAsync(ref.p, pre, n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    const RngKey rng = make_rng(seed, site, t, tick, 0);
    launch_dbm_multinomial_rows(ctx, x.p, cols, rows, cols, (float)n_samples, n_draws, bf.p, cols, f32.p, cols, rng);
    launch_softmax_rows<float>(ctx, ref.p, cols, rows, cols, (float)n_samples);
    if (n_draws > 0) launch_multinomial_rows<float>(ctx, ref.p, cols, rows, cols, n_draws, cnt.p, cols, rng);
    BM_CUDA(cudaMemcpyAsync(out_bf, bf.p, n * sizeof(bf16_t), cudaMemcpyDeviceToHost, ctx->stream));
    BM_CUDA(cudaMemcpyAsync(out_f32, f32.p, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    BM_CUDA(cudaMemcpyAsync(ref_means, ref.p, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    if (n_draws > 0) BM_CUDA(cudaMemcpyAsync(ref_counts, cnt.p, n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    BM_CUDA(cudaStreamSynchronize(ctx->stream));
    BM_API_END
}

}  // extern "C"
