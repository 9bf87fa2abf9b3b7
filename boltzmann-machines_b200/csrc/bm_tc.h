// Tensor-core (wgmma / TMA) path of libbm.so: host-side description of fused
// "layer ops" and of multi-phase programs (a whole Gibbs chain + dW in ONE persistent launch).
// Kernel in bm_tc.cu.
#pragma once
#include "bm_internal.h"
#include "bm_tc_desc.h"
#include <vector>

namespace bm {

// A row-major bf16 matrix in HBM: `rows` x `cols`, leading dimension `ld` (elements, multiple of 8),
// 16-byte aligned base.
struct TcMat {
    const __nv_bfloat16* ptr = nullptr;
    int rows = 0, cols = 0, ld = 0;
};

// C[M,N] (fp32, registers) = sum over pairs of  (+/-) A_p[M,K_p] * B_p[N,K_p]^T
//   a_t == false: A_p is stored [M, K] (K contiguous, "K-major");  true: stored [K, M] (M contiguous, "MN-major")
//   b_t == false: B_p is stored [N, K] (K-major);                 true: stored [K, N] (MN-major)
// then the same fused epilogue as the CUDA-core LayerOp (bias, scale, activation, Philox sampling),
// writing bf16 (operands of the next GEMM) and/or fp32 (host-visible results, dW partials).
struct TcGemm {
    int M = 0, N = 0;
    int n_pairs = 1;
    TcMat A[2], B[2];
    bool a_t[2] = {false, false}, b_t[2] = {false, false};
    bool neg[2] = {false, false};     // subtract this pair (wgmma scale-a = -1)
    int K[2] = {0, 0};
    int a_row0[2] = {0, 0};           // first row of A_p inside its buffer (resident dataset slices; !a_t only)
    int a_k0[2] = {0, 0};             // first K row of A_p inside its buffer (a_t only)
    bool a_batch[2] = {false, false}; // add the launch's batch_row to a_row0 / a_k0 (resident dataset cursor)
    unsigned long long* dbg = nullptr;     // device buffer of 64 timestamps (debug timeline)
    int force_bn = 0, force_cluster = 0;   // tests: override the tile heuristic (width; CTA pairs or single CTAs)
    // split-K: the concatenated K range is cut into `splits` parts; part s writes out_f32 + s * split_stride
    int splits = 1;
    size_t split_stride = 0;
    // epilogue
    float acc_scale = 1.f, bias_scale = 1.f;
    const float* bias = nullptr;
    const float* sigma = nullptr;
    const float* noise_sigma = nullptr;
    int act = ACT_LINEAR;
    int sample = SMP_NONE;
    RngKey rng{};                     // single launches: full key; programs: c2 (site | t << 8), and k0 / k1 with TcProgram::op_keys
    __nv_bfloat16* out_mean_bf = nullptr;  int ld_mean_bf = 0;
    __nv_bfloat16* out_state_bf = nullptr; int ld_state_bf = 0;
    float* out_f32 = nullptr;              int ld_f32 = 0;     // fp32 means (or raw accumulators)
    // dataflow inside a program: this op reads what ops dep[i] (indices into the program) wrote.
    //   dep_all[i] == false: row block g of this op needs row block g of dep[i]   (A rows = batch rows)
    //   dep_all[i] == true : every unit needs all of dep[i]                        (K runs over the batch: dW)
    int n_deps = 0;
    int dep[3] = {-1, -1, -1};
    bool dep_all[3] = {false, false, false};
    // which CTA pairs of a program run this op (see launch_tc_program):
    //   LANE_CHAIN: the first P pairs, P = the largest unit count of any chain op (fixed unit -> pair map)
    //   LANE_SPARE: the pairs the chain ops never use (falls back to LANE_ALL when there are none)
    //   LANE_ALL  : every pair
    int lane = 0;
    int pair_begin = 0, pair_count = 0;   // pair_count > 0: run on pairs [pair_begin, + pair_count) whatever the lane (training groups)
    // AIS in the epilogue (TcPhaseLite::ais_kind and friends)
    int ais_kind = 0;
    float ais_a = 0.f, ais_b = 0.f, ais_next = 0.f, ais_lin = 0.f;
    double* ais_logw = nullptr;
    const float* ais_base = nullptr;  // AIS ops: per-column base bias a, + a after the beta scaling (TcPhaseLite::ais_base)
    uint32_t tick_off = 0;
    uint32_t row_off = 0;             // draws of row r come from row rng.row0 + row_off + r (slot m of a tempered ladder: m * rows)
};
enum : int { LANE_CHAIN = 0, LANE_SPARE = 1, LANE_ALL = 2 };

// what a single-op launch runs (tc_describe in bm_tc.cu): the epilogue mode, the tile width, the row grouping (1 or 2), the
// number of units and the CTAs of the grid
struct TcPlan { int mode, bn, cluster, units, ctas; };
// `plan` (nullable) receives the description of the launch before it is issued
void launch_tc_gemm(Ctx* ctx, const TcGemm& g, TcPlan* plan = nullptr);
// number of (row-block pair, column block, split) units the tile heuristic cuts `g` into inside a program
int tc_plan_units(Ctx* ctx, const TcGemm& g);

// A program = ops executed by ONE persistent kernel: every CTA pair walks the same global list of
// (op, row-block pair, column block) units in order; a unit starts as soon as the row blocks it reads
// are complete (per-row-block counters in global memory), so the epilogue of one half-step overlaps
// the MMAs of the next and no kernel boundary separates the 2k+1 GEMMs of a CD-k chain and its dW.
// Ops the engines put into one program launch (the kernel's descriptor table holds 96); longer work goes in several launches.
constexpr int TC_PROGRAM_OPS = 90;
struct TcProgram {
    std::vector<TcGemm> ops;
    // device-side cache (owned by the program): descriptors + counters
    void* dev_phases = nullptr; size_t dev_phases_bytes = 0;
    int* dev_counters = nullptr; size_t n_counters = 0;
    std::vector<unsigned char> host_image;      // last uploaded descriptor image
    int epoch = 0;                              // launches since the dataflow counters were last zeroed
    int chain_units = -1;                       // largest unit count of the chain ops (planned once by the owner)
    bool op_keys = false;                       // ops draw with their own rng.k0 / k1 (training groups), not the launch key
    ~TcProgram();
};
// tick/row0 of `rng` are shared by all ops, and so is its key unless prog.op_keys; batch_row shifts the ops' a_batch operands.  `plan` (nullable, tests)
// receives one record per op of the launch, appended once the launch was issued (its `launch` field is left 0).
void launch_tc_program(Ctx* ctx, TcProgram& prog, RngKey rng, int batch_row, std::vector<bm_tc_op_plan>* plan = nullptr);

// helpers on bf16 activations
void launch_f32_to_bf16(Ctx* ctx, const float* src, int lds, __nv_bfloat16* dst, int ldd, int rows, int cols);
void launch_bf16_to_f32(Ctx* ctx, const __nv_bfloat16* src, int lds, float* dst, int ldd, int rows, int cols);
// byte-valued datasets (exact for 0..255) and the MSRE of the bf16 activations
void launch_u8_to_bf16(Ctx* ctx, const uint8_t* src, int lds, __nv_bfloat16* dst, int ldd, int rows, int cols,
                       cudaStream_t stream = nullptr);   // (nullptr: the context's stream)
template <typename T> void launch_u8_to_real(Ctx* ctx, const uint8_t* src, T* dst, size_t n);
void launch_sqdiff_mean_bf16(Ctx* ctx, const __nv_bfloat16* P, int ldp, const __nv_bfloat16* Q, int ldq, int rows, int cols,
                             double denom, double* out);
// out[n] = s1 * sum_r P[r,n] + s2 * sum_r Q[r,n]  (bf16 inputs, Q nullable, fp32 out)
void launch_colsum_bf16(Ctx* ctx, const __nv_bfloat16* P, int ldp, const __nv_bfloat16* Q, int ldq,
                        int rows, int cols, float s1, float s2, float* out);
// up to 3 plain column sums over the same number of rows in one pair of launches: out[i][c] = sum_r P[i][r, c]
void launch_colsums_bf16(Ctx* ctx, int n, const __nv_bfloat16* const* P, const int* ldp, const int* cols, float* const* out, int rows);
// the three column statistics of a CD step in one pass: sum(X - v), sum(h0 - hk), sum(hk)
void launch_cd_statistics_bf16(Ctx* ctx, const __nv_bfloat16* X, int ldx, const __nv_bfloat16* v, int ldv,
                               const __nv_bfloat16* h0, const __nv_bfloat16* hk, int ldh, int rows, int V, int H,
                               float* dvb_sum, float* dhb_sum, float* q_sum);
// G[i] = sum_s partial[s * stride + i]
void launch_reduce_partials(Ctx* ctx, const float* partial, size_t stride, int splits, float* G, size_t n);

// W += momentum step of (sum_s partial[s]) / g_div, plus the bf16 shadow, in one pass (n_hidden % 4 == 0)
void launch_weight_update_splitk(Ctx* ctx, const float* partial, size_t stride, int splits, float g_div, float* W, float* dW,
                                 int V, int H, const float* pen, float l2, float lr, float mom, __nv_bfloat16* Wb, int ldwb);

void launch_cd_tail(Ctx* ctx, const CdTail& t);
// the updates of n models of one shape in one launch: dev_tails[n] in device memory, `first` a host copy of its first entry
void launch_cd_tail_group(Ctx* ctx, const CdTail* dev_tails, const CdTail& first, int n);
// buf[r, col0] = a, buf[r, col0 + 1] = b for r < rows (the two constant columns of a batch buffer)
void launch_set_column_pair(Ctx* ctx, __nv_bfloat16* buf, int ld, size_t rows, int col0, float a, float b);
void launch_fill_bf16(Ctx* ctx, __nv_bfloat16* buf, size_t n, float v);

}  // namespace bm
