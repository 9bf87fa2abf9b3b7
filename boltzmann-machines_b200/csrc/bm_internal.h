// Internal declarations shared by the translation units of libbm.so.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <stdexcept>
#include <vector>

#include "bm_rng.cuh"
#include "../../include/bm.h"

namespace bm {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define BM_CUDA(expr)                                                                         \
    do {                                                                                      \
        cudaError_t e__ = (expr);                                                             \
        if (e__ != cudaSuccess)                                                               \
            throw ::bm::Error(BM_ECUDA, std::string(#expr " failed: ") + cudaGetErrorString(e__) + \
                                        " (" __FILE__ ":" + std::to_string(__LINE__) + ")");  \
    } while (0)

#define BM_REQUIRE(cond, msg)                                                \
    do {                                                                     \
        if (!(cond)) throw ::bm::Error(BM_EINVAL, std::string(msg));         \
    } while (0)

extern thread_local std::string g_last_error;

// Every C-ABI entry point is an NVTX range named after the function when BM_NVTX=1 (ncu --nvtx --nvtx-include "bm_rbm_train_step/",
// timeline tools): header-only NVTX v3, a no-op unless a tool injects itself.
struct NvtxRange {
    bool on;
    explicit NvtxRange(const char* name);
    ~NvtxRange();
};
#define BM_API_BEGIN try { ::bm::NvtxRange nvtx_range__(__func__);
#define BM_API_END                                                                   \
    return BM_OK;                                                                    \
    }                                                                                \
    catch (const ::bm::Error& e) { ::bm::g_last_error = e.what(); return e.code; }   \
    catch (const std::exception& e) { ::bm::g_last_error = e.what(); return BM_ECUDA; }

struct Ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;       // compute stream: every kernel of the library
    cudaStream_t copy_stream = nullptr;  // H2D prefetch of the next batch
    cudaEvent_t t0 = nullptr, t1 = nullptr, copy_done = nullptr;
    uint64_t launches = 0;
    void* l2_scratch = nullptr;
    size_t l2_scratch_bytes = 0;
    // optional per-launch timing of the tensor-core kernel (bm_ctx_profile_tc)
    bool profile_tc = false;
    std::vector<cudaEvent_t> prof_events;     // pairs (start, stop)
    size_t prof_used = 0;
    double prof_flops = 0.0, prof_ms = 0.0;
    uint64_t prof_launches = 0;
    // scratch of the small reduction kernels: per CONTEXT (two contexts on one device run on different streams)
    double* sqdiff_scratch = nullptr;
    double* reduce_scratch = nullptr;    // partial sums of sqdiff_mean / sumsq (bm_simt.cu)
    float* colsum_scratch = nullptr;
    size_t colsum_scratch_floats = 0;
    // NCCL (resolved at run time with dlopen; see bm_comm.cu)
    void* nccl_comm = nullptr;
    int rank = 0, nranks = 1;
};

// called right after every kernel launch: counts it, and turns a launch the runtime refused (invalid configuration, too
// much shared memory, ...) into an error -- unchecked, such a launch simply does not happen and its output stays stale
inline void count_launch(Ctx* c) {
    c->launches++;
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) throw Error(BM_ECUDA, std::string("kernel launch failed: ") + cudaGetErrorString(e));
}
void profile_drain(Ctx* c);      // fold recorded event pairs into prof_ms (synchronises the stream)
cudaEvent_t profile_event(Ctx* c);
void allreduce_sum(Ctx* ctx, void* buf, size_t count, bool is_double);
void allreduce_max_u32(Ctx* ctx, unsigned int* buf, size_t count);
void allreduce_sum_u32(Ctx* ctx, unsigned int* buf, size_t count);

// ---- activation / sampling selectors of the fused epilogue ------------------------
enum Act : int { ACT_LINEAR = 0, ACT_SIGMOID = 1, ACT_SOFTPLUS = 2 };
enum Smp : int { SMP_NONE = 0, SMP_BERNOULLI = 1, SMP_GAUSSIAN = 2 };

// C[M,N] = s1 * op(A1) * op(B1) + s2 * op(A2) * op(B2)           (pair 2 optional: K2 == 0)
//   a_trans == 0: A is [M,K] row-major (lda);   a_trans == 1: A is [K,M] row-major
//   b_trans == 0: B is [K,N] row-major (ldb);   b_trans == 1: B is [N,K] row-major
// then  pre = acc_scale * C * sigma[n] + bias_scale * bias[n]   (sigma/bias nullable)
//       mean = act(pre);  state = sample(mean)
template <typename T>
struct LayerOp {
    int M = 0, N = 0;
    const T* A1 = nullptr; int lda1 = 0; int K1 = 0; const T* B1 = nullptr; int ldb1 = 0; int b1_trans = 0;
    const T* A2 = nullptr; int lda2 = 0; int K2 = 0; const T* B2 = nullptr; int ldb2 = 0; int b2_trans = 0;
    int a_trans = 0;
    T s1 = 1, s2 = 1;
    T acc_scale = 1, bias_scale = 1;
    const T* bias = nullptr;
    const T* sigma = nullptr;      // per-column scale of the accumulator (gaussian visible units)
    const T* noise_sigma = nullptr;  // per-column std of gaussian sampling noise
    int act = ACT_LINEAR;
    int sample = SMP_NONE;
    RngKey rng{};
    T* means = nullptr; int ldm = 0;
    T* states = nullptr; int lds = 0;
};

template <typename T> void launch_layer_op(Ctx* ctx, const LayerOp<T>& op);

// column statistics: out[n] = s1 * sum_r P[r,n] + s2 * sum_r Q[r,n]   (Q nullable)
template <typename T>
void launch_colsum(Ctx* ctx, const T* P, int ldp, const T* Q, int ldq, int rows, int cols,
                   T s1, T s2, T* out);

// out[r] = sum_n P[r,n] * (w ? w[n] : 1)
template <typename T>
void launch_rowdot(Ctx* ctx, const T* P, int ldp, const T* w, int rows, int cols, T* out);

// per-row free-energy visible term: kind 0: -sum_v x*vb ; kind 2 (gaussian): 0.5*sum_v (x - vb/sigma)^2
template <typename T>
void launch_fe_visible(Ctx* ctx, const T* X, int ldx, const T* vb, const T* sigma, int kind,
                       int rows, int cols, T* out);

// mean over i of (a[i] + b_sign * b[i]) in double -> out (device double)
template <typename T>
void launch_mean_combine(Ctx* ctx, const T* a, const T* b, double b_sign, int n, double* out);

// sum over all elements of (P - Q)^2 (Q nullable) / denom -> out (device double)
template <typename T>
void launch_sqdiff_mean(Ctx* ctx, const T* P, int ldp, const T* Q, int ldq, int rows, int cols,
                        double denom, double* out);

// input preparation: Xp = X / sigma (gaussian) then dropout x/keep*floor(keep+u)
template <typename T>
void launch_prepare_input(Ctx* ctx, const T* X, int ldx, T* Xp, int ldxp, int rows, int cols,
                          const T* sigma, double keep, RngKey rng);

// PLL corruption: Xc = X with element (r, idx_r) replaced by 1 - x, idx_r = word(r,0) % cols
template <typename T>
void launch_pll_corrupt(Ctx* ctx, const T* X, int ldx, T* Xc, int ldxc, int rows, int cols, RngKey rng);

// bias + sparsity step (base_rbm.py:451-462, 470-474)
template <typename T>
struct BiasUpdate {
    int V, H;
    const T* dvb_raw;    // sum_b (X - v)          [V]
    const T* dhb_raw;    // sum_b (h0 - hk)        [H]
    const T* qsum;       // sum_b hk               [H]
    T *vb, *hb, *dvb, *dhb, *q_means, *pen;   // pen [H] written for the W update
    T n_div;             // the three statistics above arrive as raw sums; dvb/dhb divide by n_div
    T lr, mom, damp, cost, target;
};
template <typename T> void launch_bias_update(Ctx* ctx, const BiasUpdate<T>& u);

// W step (base_rbm.py:445-449, 462, 467-468): g = G - l2*W - pen[n]; dW = lr*(mom*dW + g); W += dW
// G is the positive-minus-negative statistic, divided here by g_div (the batch size N).
template <typename T>
void launch_weight_update(Ctx* ctx, const T* G, int ldg, T g_div, T* W, T* dW, int V, int H,
                          const T* pen, T l2, T lr, T mom, __nv_bfloat16* Wb, int ldwb);

// sum(W^2) in double
template <typename T> void launch_sumsq(Ctx* ctx, const T* W, size_t n, double* out);

// row-wise n_samples*softmax (in place on means) and multinomial counts
template <typename T>
void launch_softmax_rows(Ctx* ctx, T* X, int ldx, int rows, int cols, T scale);
template <typename T>
void launch_multinomial_rows(Ctx* ctx, const T* means, int ldm, int rows, int cols, int n_draws,
                             T* counts, int ldc, RngKey rng);

// W[i] = stddev * normal_i with tf.random_normal's Philox stream
template <typename T>
void launch_tf_normal_fill(Ctx* ctx, T* W, size_t n, double stddev, uint64_t op_seed);

template <typename T> void launch_fill(Ctx* ctx, T* p, size_t n, T v);

}  // namespace bm
