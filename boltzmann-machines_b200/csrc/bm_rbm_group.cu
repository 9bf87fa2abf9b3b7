// Training groups (bm_rbm_group_* in include/bm.h): the training steps of several tensor-core RBMs of one shape in shared
// launches.  A small RBM's step leaves most of the H100 idle -- a 48-row batch of a 192-300 model is a few units per op on a
// grid of 66 CTA pairs -- so the steps of the members run side by side: per step, ONE upload and conversion of every member's
// batch on the copy stream, program launches holding the chains of as many members as TC_PROGRAM_OPS allows (each member's
// chain ops on CTA pairs of its own, its statistics ops on all pairs), and ONE launch that updates every member.
//
// Every op is the op the member's own step builds (RbmTC::build_program: tile width, row grouping, splits and K order are its
// solo plan) and draws with the member's own key and tick (TcPhaseLite::k0 / k1, tick_off), so the grouped epoch ends
// bit-for-bit where each member's bm_rbm_train_epoch ends.
#include "bm_rbm.h"
#include <map>
#include <memory>

namespace bm {

template <typename S> __device__ __forceinline__ float group_in(S x) { return (float)x; }
template <> __device__ __forceinline__ float group_in<uint16_t>(uint16_t x) { return __uint_as_float((uint32_t)x << 16); }

// member g's rows r < rows of the staged upload [n][slot][V] -> fp32 (metrics) and bf16 (the chain's operand) at row g * slot + r of
// the half, divided by the member's sigma for Gaussian visibles -- the arithmetic of the solo step's staging (u8 / bf16 widening,
// prepare_input_kernel's x / sigma, the f32 -> bf16 rounding)
template <typename S>
__global__ void group_input_kernel(const S* __restrict__ src, int V, int rows, size_t slot, const float* __restrict__ sigma,
                                   float* __restrict__ Xf, __nv_bfloat16* __restrict__ Xb, int ldb) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y, g = blockIdx.z;
    if (c >= V || r >= rows) return;
    const size_t row = (size_t)g * slot + r;
    float x = group_in<S>(src[row * V + c]);
    if (sigma) x = x / sigma[(size_t)g * V + c];
    Xf[row * V + c] = x;
    Xb[row * ldb + c] = __float2bfloat16_rn(x);
}

struct RbmGroup {
    Ctx* ctx = nullptr;
    std::vector<RbmBase*> m;
    std::vector<TcGroupMember*> tc;
    int G = 0, V = 0, H = 0, ldv = 0, slot = 0;
    cudaStream_t copy = nullptr;
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_consumed[2] = {nullptr, nullptr};
    DevBuf<uint8_t> stage[2];
    DevBuf<__nv_bfloat16> Xb;        // [2 halves][G slots][slot rows] x ldv, the constant columns (1, 0) at VP (see RbmTC::VM)
    DevBuf<float> Xf;                // [2][G][slot] x V
    DevBuf<float> sigma;             // [G][V] (Gaussian visibles)
    std::map<std::pair<int, int>, std::unique_ptr<TcProgram>> progs;     // (rows, launch of the step)
    DevBuf<CdTail> tails;            // two tables of G updates; a step uses the one that matches the members' q buffers
    std::vector<CdTail> tail_img[2];
    int tail_next = 0;
    double* host = nullptr; size_t host_cap = 0;

    ~RbmGroup() {
        if (copy) { cudaStreamSynchronize(copy); cudaStreamDestroy(copy); }
        for (int b = 0; b < 2; ++b) { if (ev_copied[b]) cudaEventDestroy(ev_copied[b]); if (ev_consumed[b]) cudaEventDestroy(ev_consumed[b]); }
        if (host) cudaFreeHost(host);
    }
    int VP() const { return (V + 63) / 64 * 64; }

    // buffers for `batch` rows per member (grown before anything of the epoch is queued)
    void reserve(int batch) {
        if (batch <= slot) return;
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        if (copy) BM_CUDA(cudaStreamSynchronize(copy));
        slot = batch;
        const size_t rows = (size_t)2 * G * slot;
        Xb.ensure(rows * ldv); Xb.zero(ctx->stream);
        launch_set_column_pair(ctx, Xb.p, ldv, rows, VP(), 1.0f, 0.0f);
        Xf.ensure(rows * V); Xf.zero(ctx->stream);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // one step: the members' programs, their metrics, their updates
    void step(int b, int rows, int k, const double* lr, const double* mom, const uint64_t* seeds, const uint32_t* ticks,
              const uint32_t* masks, double* const* dst) {
        const size_t half = (size_t)b * G * slot;
        std::vector<TcProgram*> own(G);
        for (int g = 0; g < G; ++g) {
            own[g] = &tc[g]->group_step(Xb.p, ldv, 2 * G * slot, g * slot, (int)half, Xf.p + (half + (size_t)g * slot) * V, rows, k);
            BM_REQUIRE((int)own[g]->ops.size() <= TC_PROGRAM_OPS, "a member's step does not fit one program launch");
        }
        // launches: whole members, in order, up to TC_PROGRAM_OPS ops each
        const int total = ctx->sm_count / 2;
        int launch = 0;
        for (int g0 = 0; g0 < G; ++launch) {
            int g1 = g0, n_ops = 0;
            while (g1 < G && n_ops + (int)own[g1]->ops.size() <= TC_PROGRAM_OPS) n_ops += (int)own[g1++]->ops.size();
            std::unique_ptr<TcProgram>& slot_prog = progs[std::make_pair(rows, launch)];
            if (!slot_prog) { slot_prog.reset(new TcProgram()); slot_prog->op_keys = true; }
            TcProgram& prog = *slot_prog;
            prog.ops.clear();
            // chain ops first, member by member, each member's on CTA pairs of its own (disjoint while the members of the launch fit
            // the grid; after that the ranges start over at pair 0); then every statistics op on all pairs
            std::vector<std::vector<int>> where(g1 - g0);
            int next_pair = 0;
            for (int pass = 0; pass < 2; ++pass)
                for (int g = g0; g < g1; ++g) {
                    const std::vector<TcGemm>& ops = own[g]->ops;
                    std::vector<int>& w = where[g - g0];
                    w.resize(ops.size(), -1);
                    const int P = std::min(std::max(own[g]->chain_units, 1), total);
                    if (pass == 0 && next_pair + P > total) next_pair = 0;
                    for (size_t i = 0; i < ops.size(); ++i) {
                        if ((ops[i].lane == LANE_CHAIN) != (pass == 0)) continue;
                        TcGemm op = ops[i];
                        for (int d = 0; d < op.n_deps; ++d) op.dep[d] = w[op.dep[d]];
                        op.rng.k0 = (uint32_t)seeds[g]; op.rng.k1 = (uint32_t)(seeds[g] >> 32);
                        op.tick_off += ticks[g] - ticks[g0];
                        if (pass == 0) { op.pair_begin = next_pair; op.pair_count = P; }
                        w[i] = (int)prog.ops.size();
                        prog.ops.push_back(op);
                    }
                    if (pass == 0) next_pair += P;
                }
            std::vector<bm_tc_op_plan> plan;
            launch_tc_program(ctx, prog, make_rng(seeds[g0], 0, 0, ticks[g0], 0), (int)half, &plan);
            for (int g = g0; g < g1; ++g) {
                std::vector<bm_tc_op_plan>& mine = tc[g]->group_plan();
                for (int j : where[g - g0]) { mine.push_back(plan[j]); mine.back().launch = launch; }
            }
            g0 = g1;
        }
        for (int g = 0; g < G; ++g)
            if (masks[g]) tc[g]->group_metrics(masks[g], rows, seeds[g], ticks[g], dst[g]);
        // updates: one launch; the table is uploaded only when it changed (the members' q buffers alternate between two)
        std::vector<CdTail> cur(G);
        for (int g = 0; g < G; ++g) cur[g] = tc[g]->group_tail(rows, lr[g], mom[g]);
        int t = -1;
        for (int s = 0; s < 2 && t < 0; ++s)
            if (tail_img[s].size() == cur.size() && memcmp(tail_img[s].data(), cur.data(), cur.size() * sizeof(CdTail)) == 0) t = s;
        if (t < 0) {
            t = tail_next; tail_next ^= 1;
            BM_CUDA(cudaMemcpyAsync(tails.p + (size_t)t * G, cur.data(), cur.size() * sizeof(CdTail), cudaMemcpyHostToDevice, ctx->stream));
            tail_img[t] = cur;
        }
        launch_cd_tail_group(ctx, tails.p + (size_t)t * G, cur[0], G);
        for (int g = 0; g < G; ++g) tc[g]->group_step_done();
    }

    void train_epoch(const void* X, int64_t n_rows, int batch, const double* lr, const double* mom, int k, const uint64_t* seeds,
                     const uint32_t* tick0, const uint32_t* masks, const int32_t* every, const int64_t* iter0, double* out, int src) {
        BM_REQUIRE(X && n_rows >= 1 && batch >= 1 && batch <= 65535, "empty dataset or batch (1..65535 rows)");
        BM_REQUIRE(lr && mom && seeds && tick0 && masks && every && iter0, "null per-member argument");
        BM_REQUIRE(k >= 1, "n_gibbs_steps must be >= 1");
        if (2 * k + 3 > TC_PROGRAM_OPS)
            throw Error(BM_EUNSUPPORTED, "training groups: n_gibbs_steps above 43 (the chain needs several launches per member)");
        bool any = false;
        for (int g = 0; g < G; ++g) any = any || masks[g] != 0;
        BM_REQUIRE(!any || out != nullptr, "metrics requested without an output buffer");
        BM_REQUIRE(src != SRC_BF16 || m[0]->cfg.v_kind != BM_UNIT_GAUSSIAN,
                   "a bfloat16 feed needs models without sigma scaling (not Gaussian visibles)");
        const size_t es = src == SRC_U8 ? 1 : (src == SRC_BF16 ? 2 : sizeof(float));
        const int64_t nb = (n_rows + batch - 1) / batch;
        reserve(batch);
        for (int b = 0; b < 2; ++b) stage[b].ensure((size_t)G * slot * V * es);
        tails.ensure((size_t)2 * G);
        if ((size_t)G * nb * 8 > host_cap) {
            if (host) cudaFreeHost(host);
            host = nullptr; host_cap = 0;
            BM_CUDA(cudaMallocHost((void**)&host, (size_t)G * nb * 8 * sizeof(double)));
            host_cap = (size_t)G * nb * 8;
        }
        for (int b = 0; b < 2; ++b) BM_CUDA(cudaEventRecord(ev_consumed[b], ctx->stream));
        std::vector<uint32_t> ticks(G), step_masks(G);
        std::vector<double*> dst(G);
        try {
            for (int64_t i = 0; i < nb; ++i) {
                const int b = (int)(i & 1);
                const int rows = (int)std::min<int64_t>(batch, n_rows - i * batch);
                const size_t half = (size_t)b * G * slot;
                BM_CUDA(cudaStreamWaitEvent(copy, ev_consumed[b], 0));
                BM_CUDA(cudaMemcpy2DAsync(stage[b].p, (size_t)slot * V * es, (const char*)X + (size_t)i * batch * V * es,
                                          (size_t)n_rows * V * es, (size_t)rows * V * es, (size_t)G, cudaMemcpyHostToDevice, copy));
                const dim3 grid((unsigned)((V + 127) / 128), (unsigned)rows, (unsigned)G);
                float* xf = Xf.p + half * V;
                __nv_bfloat16* xb = Xb.p + half * ldv;
                if (src == SRC_U8)
                    group_input_kernel<uint8_t><<<grid, 128, 0, copy>>>(stage[b].p, V, rows, slot, sigma.p, xf, xb, ldv);
                else if (src == SRC_BF16)
                    group_input_kernel<uint16_t><<<grid, 128, 0, copy>>>((const uint16_t*)stage[b].p, V, rows, slot, sigma.p, xf, xb, ldv);
                else
                    group_input_kernel<float><<<grid, 128, 0, copy>>>((const float*)stage[b].p, V, rows, slot, sigma.p, xf, xb, ldv);
                count_launch(ctx);
                BM_CUDA(cudaEventRecord(ev_copied[b], copy));
                BM_CUDA(cudaStreamWaitEvent(ctx->stream, ev_copied[b], 0));
                for (int g = 0; g < G; ++g) {
                    ticks[g] = tick0[g] + (uint32_t)i;
                    const bool report = masks[g] && every[g] > 0 && ((iter0[g] + i + 1) % every[g] == 0);
                    step_masks[g] = report ? masks[g] : 0u;
                    dst[g] = host + ((size_t)g * nb + i) * 8;
                }
                step(b, rows, k, lr, mom, seeds, ticks.data(), step_masks.data(), dst.data());
                BM_CUDA(cudaEventRecord(ev_consumed[b], ctx->stream));
            }
        } catch (...) {
            cudaStreamSynchronize(copy); cudaStreamSynchronize(ctx->stream);
            throw;
        }
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        for (int g = 0; g < G && any; ++g)
            for (int64_t i = 0; i < nb; ++i) {
                double* o = out + ((size_t)g * nb + i) * 4;
                const bool report = masks[g] && every[g] > 0 && ((iter0[g] + i + 1) % every[g] == 0);
                if (report) tc[g]->group_finish_metrics(host + ((size_t)g * nb + i) * 8, masks[g], o);
                else for (int j = 0; j < 4; ++j) o[j] = 0.0;
            }
    }
};

}  // namespace bm

using namespace bm;

extern "C" {

int bm_rbm_group_create(bm_ctx* hctx, bm_rbm* const* members, int32_t n, bm_rbm_group** out) {
    BM_API_BEGIN
    Ctx* ctx = reinterpret_cast<Ctx*>(hctx);
    BM_REQUIRE(ctx && members && out && n >= 1, "bad argument");
    std::vector<RbmBase*> m(n);
    for (int g = 0; g < n; ++g) {
        m[g] = reinterpret_cast<RbmBase*>(members[g]);
        BM_REQUIRE(m[g] != nullptr, "null rbm handle");
    }
    const bm_rbm_cfg& c0 = m[0]->cfg;
    for (int g = 0; g < n; ++g) {
        const bm_rbm_cfg& c = m[g]->cfg;
        BM_REQUIRE(m[g]->ctx == ctx, "members must share the group's context");
        BM_REQUIRE(c.n_visible == c0.n_visible, "members must share n_visible");
        BM_REQUIRE(c.n_hidden == c0.n_hidden, "members must share n_hidden");
        BM_REQUIRE(c.v_kind == c0.v_kind, "members must share the visible unit kind (v_kind)");
        BM_REQUIRE(c.h_kind == c0.h_kind, "members must share the hidden unit kind (h_kind)");
        BM_REQUIRE(c.max_batch == c0.max_batch, "members must share max_batch");
        if (c.v_kind == BM_UNIT_MULTINOMIAL || c.h_kind == BM_UNIT_MULTINOMIAL)
            throw Error(BM_EUNSUPPORTED, "training groups: multinomial layers (their row kernels run between launches)");
        if (!m[g]->tc_group_member())
            throw Error(BM_EUNSUPPORTED, "training groups: the fp32 / fp64 engines (members need compute='bf16', float32)");
        if (c.dropout_keep >= 0) throw Error(BM_EUNSUPPORTED, "training groups: dropout");
    }
    if (ctx->nranks > 1) throw Error(BM_EUNSUPPORTED, "training groups: a context with a communicator");
    BM_CUDA(cudaSetDevice(ctx->device));
    std::unique_ptr<RbmGroup> grp(new RbmGroup());
    grp->ctx = ctx; grp->m = m; grp->G = n;
    for (RbmBase* r : m) grp->tc.push_back(r->tc_group_member());
    grp->V = c0.n_visible; grp->H = c0.n_hidden;
    grp->ldv = (c0.n_visible + 63) / 64 * 64 + 64;          // RbmTC::ldv
    if (c0.v_kind == BM_UNIT_GAUSSIAN) {
        grp->sigma.ensure((size_t)n * grp->V);
        for (int g = 0; g < n; ++g)        // (the tensor-core engine derives from the float32 storage engine, which holds sigma)
            BM_CUDA(cudaMemcpyAsync(grp->sigma.p + (size_t)g * grp->V, static_cast<RbmSimt<float>*>(m[g])->sigma.p,
                                    (size_t)grp->V * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    }
    BM_CUDA(cudaStreamCreateWithFlags(&grp->copy, cudaStreamNonBlocking));
    for (int b = 0; b < 2; ++b) {
        BM_CUDA(cudaEventCreateWithFlags(&grp->ev_copied[b], cudaEventDisableTiming));
        BM_CUDA(cudaEventCreateWithFlags(&grp->ev_consumed[b], cudaEventDisableTiming));
    }
    grp->reserve(c0.max_batch > 0 ? c0.max_batch : 1);
    *out = reinterpret_cast<bm_rbm_group*>(grp.release());
    BM_API_END
}

void bm_rbm_group_destroy(bm_rbm_group* h) {
    if (!h) return;
    RbmGroup* g = reinterpret_cast<RbmGroup*>(h);
    cudaSetDevice(g->ctx->device);
    cudaStreamSynchronize(g->ctx->stream);
    delete g;
}

#define GROUP_EPOCH(name, T, SRC)                                                                                              \
    int name(bm_rbm_group* h, const T* X, int64_t n_rows, int32_t batch, const double* lr, const double* momentum, int32_t k,  \
             const uint64_t* seeds, const uint32_t* tick0, const uint32_t* mask, const int32_t* every, const int64_t* iter0,    \
             double* out) {                                                                                                    \
        BM_API_BEGIN                                                                                                           \
        BM_REQUIRE(h != nullptr, "null group handle");                                                                         \
        RbmGroup* g = reinterpret_cast<RbmGroup*>(h);                                                                          \
        BM_CUDA(cudaSetDevice(g->ctx->device));                                                                                \
        g->train_epoch(X, n_rows, batch, lr, momentum, k, seeds, tick0, mask, every, iter0, out, SRC);                         \
        BM_API_END                                                                                                             \
    }
GROUP_EPOCH(bm_rbm_group_train_epoch, void, SRC_NATIVE)
GROUP_EPOCH(bm_rbm_group_train_epoch_u8, uint8_t, SRC_U8)
GROUP_EPOCH(bm_rbm_group_train_epoch_bf16, uint16_t, SRC_BF16)

}  // extern "C"
