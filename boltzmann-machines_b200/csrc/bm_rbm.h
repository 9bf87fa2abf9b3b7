// RBM engine classes (header so that the tensor-core engine can derive from the storage-precision one).
#pragma once
#include "bm_internal.h"
#include "bm_tc.h"
#include <vector>
#include <algorithm>
#include <string.h>
#include <math.h>

namespace bm {

template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    void ensure(size_t count) {
        if (count <= n) return;
        if (p) cudaFree(p);
        p = nullptr;
        BM_CUDA(cudaMalloc(&p, count * sizeof(T)));
        n = count;
    }
    void zero(cudaStream_t s) { if (p) BM_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), s)); }
    ~DevBuf() { if (p) cudaFree(p); }
};

enum : int { SRC_NATIVE = 0, SRC_U8 = 1, SRC_BF16 = 2 };

// What a training group (bm_rbm_group.cu) asks of a tensor-core model: the group runs the training steps of several models
// of one shape in shared program launches and updates them all in one launch.
struct TcGroupMember {
    virtual ~TcGroupMember() {}
    // builds the program of one training step exactly as the model's own step does, reading the batch from rows
    // [base, base + rows) of the bf16 input X (ld, rows_total rows) shifted by the launch's batch cursor `cursor`; Xf holds the
    // same rows in fp32 for the metrics.  The model's activations then describe this step.
    virtual TcProgram& group_step(const __nv_bfloat16* X, int ld, int rows_total, int base, int cursor, const float* Xf, int rows,
                                  int k) = 0;
    virtual CdTail group_tail(int rows, double lr, double mom) const = 0;     // the update of that step
    virtual void group_step_done() = 0;                                         // after the update was queued
    virtual std::vector<bm_tc_op_plan>& group_plan() = 0;                       // what bm_rbm_debug_tc_plan reports
    // the metrics of `mask` under the step's pre-update weights, read back asynchronously into dst[8] ...
    virtual void group_metrics(uint32_t mask, int rows, uint64_t seed, uint32_t tick, double* dst) = 0;
    // ... and turned into the four slots of bm_rbm_train_epoch once the stream has been synchronised
    virtual void group_finish_metrics(const double* h, uint32_t mask, double* out) const = 0;
};

struct RbmBase {
    Ctx* ctx = nullptr;
    bm_rbm_cfg cfg{};
    virtual ~RbmBase() {}
    virtual void set_param(const char* name, const void* host, size_t bytes) = 0;
    virtual void get_param(const char* name, void* host, size_t bytes) = 0;
    virtual void init_weights(double stddev, uint64_t op_seed) = 0;
    virtual void set_data(const void* X, int64_t n_rows) = 0;
    virtual void train_step(const void* X_host, int64_t first_row, int rows, double lr, double mom, int k,
                            uint64_t seed, uint32_t tick, uint32_t mask, double* out) = 0;
    // src: element type of X_host -- SRC_NATIVE: cfg.dtype; SRC_U8: one unsigned byte per visible unit (binary / byte-valued
    // data, exact); SRC_BF16: bfloat16 bit patterns (real-valued data for the bf16 engine, which rounds its input to bf16 anyway)
    virtual void train_epoch(const void* X_host, int64_t n_rows, int batch, double lr, double mom, int k, uint64_t seed,
                             uint32_t tick0, uint32_t mask, int every, int64_t iter0, double* out, int src) = 0;
    virtual void transform(const void* X, int rows, int k, uint64_t seed, uint32_t tick, void* H_out) = 0;
    virtual void metrics(const void* X, int rows, int k, uint64_t seed, uint32_t tick, uint32_t mask, double* out) = 0;
    virtual void get_activation(const char* name, void* host, size_t bytes) = 0;
    // test hook (bm_rbm_debug_tc_plan): the ops of the last tensor-core program
    virtual const std::vector<bm_tc_op_plan>& tc_plan() const { throw Error(BM_EINVAL, "this engine runs no tensor-core program"); }
    virtual TcGroupMember* tc_group_member() { return nullptr; }       // null: the engine cannot train in a group
};

// ------------------------------------------------------------------------------------------
// storage-precision engine (CUDA-core GEMMs): float32 or float64 end to end
// ------------------------------------------------------------------------------------------
template <typename T>
struct RbmSimt : RbmBase {
    int V, H;
    DevBuf<T> W, vb, hb, dW, dvb, dhb, q, sigma;
    DevBuf<T> stats;        // [G (V*H) | dvb_sum (V) | dhb_sum (H) | q_sum (H)] : one allreduce
    DevBuf<T> pen, hhat;
    DevBuf<T> Xin, Xp, Xc, h0m, h0s, vm, vs, hm, hs, tmpH, rowA, rowB;
    DevBuf<T> data;         // resident dataset
    int64_t data_rows = 0;
    DevBuf<double> scal;    // device scalars
    int cap = 0, last_rows = 0;
    const T* Xcur = nullptr;   // prepared batch of the last call
    const T* vs_cur = nullptr;
    const T* h0s_cur = nullptr;

    RbmSimt(Ctx* c, const bm_rbm_cfg& f) {
        ctx = c; cfg = f; V = f.n_visible; H = f.n_hidden;
        W.ensure((size_t)V * H); dW.ensure((size_t)V * H);
        vb.ensure(V); dvb.ensure(V); hb.ensure(H); dhb.ensure(H); q.ensure(H);
        pen.ensure(H); hhat.ensure(H);
        stats.ensure((size_t)V * H + V + 2 * (size_t)H);
        scal.ensure(16);
        for (DevBuf<T>* b : {&W, &dW, &vb, &dvb, &hb, &dhb, &q, &pen}) b->zero(ctx->stream);
        if (f.sigma) {
            std::vector<T> s(V);
            for (int i = 0; i < V; ++i) s[i] = (T)f.sigma[i];
            sigma.ensure(V);
            BM_CUDA(cudaMemcpyAsync(sigma.p, s.data(), V * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
        }
        cfg.sigma = nullptr;
        reserve(f.max_batch > 0 ? f.max_batch : 1);
    }

    void reserve(int rows) {
        if (rows <= cap) return;
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        cap = rows;
        const size_t rv = (size_t)rows * V, rh = (size_t)rows * H;
        Xin.ensure(rv); Xp.ensure(rv); Xc.ensure(rv); vm.ensure(rv); vs.ensure(rv);
        h0m.ensure(rh); h0s.ensure(rh); hm.ensure(rh); hs.ensure(rh); tmpH.ensure(rh);
        rowA.ensure(rows); rowB.ensure(rows);
    }

    DevBuf<T>* by_name(const char* name, size_t* count) {
        struct E { const char* n; DevBuf<T>* b; size_t c; };
        const E tab[] = {{"W", &W, (size_t)V * H}, {"vb", &vb, (size_t)V}, {"hb", &hb, (size_t)H},
                         {"dW", &dW, (size_t)V * H}, {"dvb", &dvb, (size_t)V}, {"dhb", &dhb, (size_t)H},
                         {"q_means", &q, (size_t)H}, {"sigma", &sigma, (size_t)V}};
        for (const E& e : tab)
            if (!strcmp(e.n, name)) { *count = e.c; return e.b; }
        throw Error(BM_EINVAL, std::string("unknown variable '") + name + "'");
    }

    void set_param(const char* name, const void* host, size_t bytes) override {
        size_t cnt; DevBuf<T>* b = by_name(name, &cnt);
        BM_REQUIRE(b->p != nullptr, std::string("variable '") + name + "' does not exist in this model");
        BM_REQUIRE(bytes == cnt * sizeof(T), std::string("size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpyAsync(b->p, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void get_param(const char* name, void* host, size_t bytes) override {
        size_t cnt; DevBuf<T>* b = by_name(name, &cnt);
        BM_REQUIRE(b->p != nullptr, std::string("variable '") + name + "' does not exist in this model");
        BM_REQUIRE(bytes == cnt * sizeof(T), std::string("size mismatch for '") + name + "'");
        BM_CUDA(cudaMemcpyAsync(host, b->p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void init_weights(double stddev, uint64_t op_seed) override {
        launch_tf_normal_fill<T>(ctx, W.p, (size_t)V * H, stddev, op_seed);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void set_data(const void* X, int64_t n_rows) override {
        data.ensure((size_t)n_rows * V);
        BM_CUDA(cudaMemcpyAsync(data.p, X, (size_t)n_rows * V * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        data_rows = n_rows;
    }

    // ---- one conditional: means (and states) of one layer given the other -----------------
    void layer(bool up, const T* in, T* means, T* states, bool sample, uint32_t site, uint32_t t,
               int rows, uint64_t seed, uint32_t tick, uint32_t row0) {
        LayerOp<T> op;
        op.M = rows; op.N = up ? H : V;
        op.A1 = in; op.lda1 = up ? V : H; op.K1 = up ? V : H;
        op.B1 = W.p; op.ldb1 = H; op.b1_trans = up ? 0 : 1;
        const T mult = (T)(up ? cfg.propup_mult : cfg.propdown_mult);   // base_rbm.py:342-343,356-357
        op.acc_scale = mult; op.bias_scale = mult;
        op.bias = up ? hb.p : vb.p;
        op.means = means; op.ldm = op.N;
        const int kind = up ? cfg.h_kind : cfg.v_kind;
        op.rng = make_rng(seed, site, t, tick, row0);
        if (kind == BM_UNIT_BERNOULLI) {
            op.act = ACT_SIGMOID;
            if (sample) { op.sample = SMP_BERNOULLI; op.states = states; op.lds = op.N; }
            launch_layer_op<T>(ctx, op);
        } else if (kind == BM_UNIT_GAUSSIAN) {
            op.act = ACT_LINEAR; op.sigma = sigma.p;             // layers.py:84-86
            if (sample) { op.sample = SMP_GAUSSIAN; op.noise_sigma = sigma.p; op.states = states; op.lds = op.N; }
            launch_layer_op<T>(ctx, op);
        } else {                                                 // multinomial, layers.py:65-70
            op.act = ACT_LINEAR;
            launch_layer_op<T>(ctx, op);
            const double M = up ? cfg.h_n_samples : cfg.v_n_samples;
            launch_softmax_rows<T>(ctx, means, op.N, rows, op.N, (T)M);
            if (sample) launch_multinomial_rows<T>(ctx, means, op.N, rows, op.N, (int)M, states, op.N, op.rng);
        }
    }

    // ---- input: upload (or slice of the resident data) -> sigma division -> dropout ----------
    const T* stage_input(const void* X_host, int64_t first_row, int rows, uint64_t seed, uint32_t tick, uint32_t row0) {
        reserve(rows);
        const T* src;
        if (staged_u8) {
            launch_u8_to_real<T>(ctx, staged_u8, Xin.p, (size_t)rows * V);     // byte-valued epoch data, exact
            src = Xin.p;
        } else if (staged_dev) {
            src = staged_dev;                       // already copied by train_epoch's copy stream
        } else if (X_host) {
            BM_CUDA(cudaMemcpyAsync(Xin.p, X_host, (size_t)rows * V * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
            src = Xin.p;
        } else {
            BM_REQUIRE(first_row >= 0 && first_row + rows <= data_rows, "row range outside the resident dataset");
            src = data.p + (size_t)first_row * V;
        }
        const bool gauss = cfg.v_kind == BM_UNIT_GAUSSIAN;
        if (gauss || cfg.dropout_keep >= 0) {
            launch_prepare_input<T>(ctx, src, V, Xp.p, V, rows, V, gauss ? sigma.p : nullptr, cfg.dropout_keep,
                                    make_rng(seed, SITE_DROPOUT, 0, tick, row0));
            src = Xp.p;
        }
        return src;
    }

    // ---- Gibbs chain (base_rbm.py:421-426, 367-384) ----------------------------------------------
    void chain(const T* X, int rows, int k, uint64_t seed, uint32_t tick, uint32_t row0) {
        BM_REQUIRE(k >= 1, "n_gibbs_steps must be >= 1");
        last_rows = rows; Xcur = X;
        const bool sh = cfg.sample_h != 0, sv = cfg.sample_v != 0;
        layer(true, X, h0m.p, h0s.p, sh, SITE_H0, 0, rows, seed, tick, row0);
        h0s_cur = sh ? h0s.p : h0m.p;
        const T* hstate = h0s_cur;
        for (int t = 1; t <= k; ++t) {
            layer(false, hstate, vm.p, vs.p, sv, SITE_V, t, rows, seed, tick, row0);
            vs_cur = sv ? vs.p : vm.p;
            const bool smp = sh && t < k;       // the last step's hidden states are never consumed
            layer(true, vs_cur, hm.p, hs.p, smp, SITE_H, t, rows, seed, tick, row0);
            hstate = smp ? hs.p : hm.p;
        }
    }

    // ---- free energy of a batch -> device scalar slot (rbm/rbm.py:17-22, 50-60, 109-116) ---------
    void free_energy(const T* X, int rows, int slot, uint64_t seed, uint32_t tick, uint32_t fe_idx) {
        LayerOp<T> op;
        op.M = rows; op.N = H; op.A1 = X; op.lda1 = V; op.K1 = V; op.B1 = W.p; op.ldb1 = H;
        op.means = tmpH.p; op.ldm = H;
        if (cfg.h_kind == BM_UNIT_MULTINOMIAL) {
            op.act = ACT_LINEAR;                      // T2 = -v W (sign applied below)
            launch_layer_op<T>(ctx, op);
            launch_fill<T>(ctx, pen.p, H, T(1));      // uniform logits (pen is rewritten by every update)
            launch_multinomial_rows<T>(ctx, pen.p, H, 1, H, (int)cfg.h_n_samples, hhat.p, H,
                                       make_rng(seed, SITE_MULTINOMIAL_FE, fe_idx, tick, 0));
            launch_rowdot<T>(ctx, tmpH.p, H, hhat.p, rows, H, rowA.p);
        } else {
            op.act = ACT_SOFTPLUS; op.bias = hb.p;    // softplus(v W + hb)
            launch_layer_op<T>(ctx, op);
            launch_rowdot<T>(ctx, tmpH.p, H, nullptr, rows, H, rowA.p);
        }
        launch_fe_visible<T>(ctx, X, V, vb.p, sigma.p, cfg.v_kind == BM_UNIT_GAUSSIAN ? BM_UNIT_GAUSSIAN : 0, rows, V, rowB.p);
        launch_mean_combine<T>(ctx, rowB.p, rowA.p, -1.0, rows, scal.p + slot);
    }

    // engines that keep the chain's activations in another format compute the MSRE from them directly
    virtual bool msre_from_activations(int /*rows*/, double* /*dst*/) { return false; }

    void run_metrics(uint32_t mask, int rows, uint64_t seed, uint32_t tick, uint32_t row0, double* out) {
        if (!mask) return;
        BM_REQUIRE(out != nullptr, "metrics requested without an output buffer");
        if (mask & BM_METRIC_L2_LOSS) launch_sumsq<T>(ctx, W.p, (size_t)V * H, scal.p + 0);
        if ((mask & BM_METRIC_MSRE) && !msre_from_activations(rows, scal.p + 1))
            launch_sqdiff_mean<T>(ctx, Xcur, V, vm.p, V, rows, V, (double)rows * V, scal.p + 1);
        if (mask & BM_METRIC_PLL) {
            launch_pll_corrupt<T>(ctx, Xcur, V, Xc.p, V, rows, V, make_rng(seed, SITE_PLL, 0, tick, row0));
            free_energy(Xc.p, rows, 4, seed, tick, 0);
            free_energy(Xcur, rows, 5, seed, tick, 1);
        }
        if (mask & BM_METRIC_FREE_ENERGY) free_energy(Xcur, rows, 3, seed, tick, 2);
        double h[8];
        if (defer_dst) {                            // train_epoch: read back without stalling the stream
            BM_CUDA(cudaMemcpyAsync(defer_dst, scal.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
            return;
        }
        BM_CUDA(cudaMemcpyAsync(h, scal.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        finish_metrics(h, mask, out);
    }
    void finish_metrics(const double* h, uint32_t mask, double* out) const {
        double fe_const = 0.0;
        if (cfg.h_kind == BM_UNIT_MULTINOMIAL) {
            const double M = cfg.h_n_samples, K = (double)H;
            fe_const = -lgamma(M + K) + lgamma(M + 1.0) + lgamma(K);
        }
        out[BM_SLOT_L2_LOSS] = (mask & BM_METRIC_L2_LOSS) ? cfg.l2 * 0.5 * h[0] : 0.0;   // base_rbm.py:483
        out[BM_SLOT_MSRE] = (mask & BM_METRIC_MSRE) ? h[1] : 0.0;                         // :487
        if (mask & BM_METRIC_PLL) {                                                       // :511-512
            const double d = h[4] - h[5];
            out[BM_SLOT_PLL] = (double)V * -(fmax(-d, 0.0) + log1p(exp(-fabs(d))));
        } else out[BM_SLOT_PLL] = 0.0;
        out[BM_SLOT_FREE_ENERGY] = (mask & BM_METRIC_FREE_ENERGY) ? h[3] + fe_const : 0.0;
    }

    void train_step(const void* X_host, int64_t first_row, int rows, double lr, double mom, int k,
                    uint64_t seed, uint32_t tick, uint32_t mask, double* out) override {
        BM_REQUIRE(rows >= 1, "empty batch");
        const uint32_t row0 = (uint32_t)(ctx->rank * rows);
        const T* X = stage_input(X_host, first_row, rows, seed, tick, row0);
        chain(X, rows, k, seed, tick, row0);
        run_metrics(mask, rows, seed, tick, row0, out);

        T* G = stats.p;
        T* dvb_sum = G + (size_t)V * H;
        T* dhb_sum = dvb_sum + V;
        T* q_sum = dhb_sum + H;
        // dW_positive - dW_negative (base_rbm.py:447-448): X^T h0_means - v^T h_means
        LayerOp<T> g;
        g.M = V; g.N = H; g.a_trans = 1;
        g.A1 = X; g.lda1 = V; g.K1 = rows; g.B1 = h0m.p; g.ldb1 = H;
        g.A2 = vs_cur; g.lda2 = V; g.K2 = rows; g.B2 = hm.p; g.ldb2 = H;
        g.s1 = T(1); g.s2 = T(-1);
        g.means = G; g.ldm = H;
        launch_layer_op<T>(ctx, g);
        launch_colsum<T>(ctx, X, V, vs_cur, V, rows, V, T(1), T(-1), dvb_sum);       // :451
        launch_colsum<T>(ctx, h0m.p, H, hm.p, H, rows, H, T(1), T(-1), dhb_sum);     // :453
        launch_colsum<T>(ctx, hm.p, H, (const T*)nullptr, 0, rows, H, T(1), T(0), q_sum);   // :457
        allreduce_sum(ctx, stats.p, (size_t)V * H + V + 2 * (size_t)H, sizeof(T) == 8);
        const T N = (T)((double)rows * ctx->nranks);

        BiasUpdate<T> u;
        u.V = V; u.H = H; u.dvb_raw = dvb_sum; u.dhb_raw = dhb_sum; u.qsum = q_sum;
        u.vb = vb.p; u.hb = hb.p; u.dvb = dvb.p; u.dhb = dhb.p; u.q_means = q.p; u.pen = pen.p;
        u.n_div = N; u.lr = (T)lr; u.mom = (T)mom;
        u.damp = (T)cfg.sparsity_damping; u.cost = (T)cfg.sparsity_cost; u.target = (T)cfg.sparsity_target;
        launch_bias_update<T>(ctx, u);
        launch_weight_update<T>(ctx, G, H, N, W.p, dW.p, V, H, pen.p, (T)cfg.l2, (T)lr, (T)mom, nullptr, 0);
    }

    // ---- one epoch over a host dataset (base_rbm.py:549-571) -----------------------------------
    // Batch i+1 is copied host->device on a second stream while batch i computes (two staging
    // buffers); requested metrics are read back asynchronously into pinned memory, so the compute
    // stream never waits for the host inside the epoch.
    ~RbmSimt() override {
        if (copy_stream) cudaStreamDestroy(copy_stream);
        for (int b = 0; b < 2; ++b) { if (ev_copied[b]) cudaEventDestroy(ev_copied[b]); if (ev_consumed[b]) cudaEventDestroy(ev_consumed[b]); }
        if (epoch_host) cudaFreeHost(epoch_host);
    }
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_consumed[2] = {nullptr, nullptr};
    DevBuf<T> epoch_stage[2];
    DevBuf<uint8_t> epoch_stage_u8[2];
    DevBuf<uint16_t> epoch_stage_bf16[2];
    const T* staged_dev = nullptr;
    const uint8_t* staged_u8 = nullptr;
    const uint16_t* staged_bf16 = nullptr;
    int staged_half = -1;             // >= 0: the engine converted the staged batch itself on the copy stream (convert_on_copy_stream)

    // An engine that keeps its input in another format may convert the batch the copy stream has just uploaded ON that stream
    // (off the compute stream's critical path), into half `b` of a double buffer of its own; it then reads `staged_half` in its
    // train_step instead of the staged pointers.  Called after the upload has been queued and before ev_copied[b] is recorded.
    virtual bool convert_on_copy_stream(int /*b*/, const void* /*staged*/, int /*rows*/, int /*batch*/, int /*src*/,
                                        cudaStream_t /*copy*/) { return false; }
    virtual bool accepts_bf16_feed() const { return false; }
    double* defer_dst = nullptr;
    double* epoch_host = nullptr;
    size_t epoch_host_cap = 0;

    void train_epoch(const void* X_host, int64_t n_rows, int batch, double lr, double mom, int k, uint64_t seed,
                     uint32_t tick0, uint32_t mask, int every, int64_t iter0, double* out, int src) override {
        BM_REQUIRE(X_host != nullptr && n_rows >= 1 && batch >= 1, "empty dataset or batch");
        const bool src_u8 = src == SRC_U8, src_bf16 = src == SRC_BF16;
        BM_REQUIRE(!src_bf16 || accepts_bf16_feed(), "a bfloat16 feed needs the bf16 tensor-core engine without dropout / sigma scaling");
        BM_REQUIRE(!mask || out != nullptr, "metrics requested without an output buffer");
        const int64_t nb = (n_rows + batch - 1) / batch;
        if (!copy_stream) {
            BM_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
            for (int b = 0; b < 2; ++b) {
                BM_CUDA(cudaEventCreateWithFlags(&ev_copied[b], cudaEventDisableTiming));
                BM_CUDA(cudaEventCreateWithFlags(&ev_consumed[b], cudaEventDisableTiming));
            }
        }
        for (int b = 0; b < 2; ++b) {
            if (src_u8) epoch_stage_u8[b].ensure((size_t)batch * V);
            else if (src_bf16) epoch_stage_bf16[b].ensure((size_t)batch * V);
            else epoch_stage[b].ensure((size_t)batch * V);
        }
        if ((size_t)nb * 8 > epoch_host_cap) {
            if (epoch_host) cudaFreeHost(epoch_host);
            epoch_host = nullptr; epoch_host_cap = 0;
            BM_CUDA(cudaMallocHost((void**)&epoch_host, (size_t)nb * 8 * sizeof(double)));
            epoch_host_cap = (size_t)nb * 8;
        }
        // the staging buffers may still be read by work already queued on the compute stream
        for (int b = 0; b < 2; ++b) BM_CUDA(cudaEventRecord(ev_consumed[b], ctx->stream));
        const T* Xh = (const T*)X_host;
        const uint8_t* Xh8 = (const uint8_t*)X_host;
        const uint16_t* Xh16 = (const uint16_t*)X_host;
        double unused[4];
        try {
            for (int64_t i = 0; i < nb; ++i) {
                const int b = (int)(i & 1);
                const int rows = (int)std::min<int64_t>(batch, n_rows - i * batch);
                BM_CUDA(cudaStreamWaitEvent(copy_stream, ev_consumed[b], 0));
                if (src_u8)
                    BM_CUDA(cudaMemcpyAsync(epoch_stage_u8[b].p, Xh8 + (size_t)i * batch * V, (size_t)rows * V,
                                            cudaMemcpyHostToDevice, copy_stream));
                else if (src_bf16)
                    BM_CUDA(cudaMemcpyAsync(epoch_stage_bf16[b].p, Xh16 + (size_t)i * batch * V, (size_t)rows * V * 2,
                                            cudaMemcpyHostToDevice, copy_stream));
                else
                    BM_CUDA(cudaMemcpyAsync(epoch_stage[b].p, Xh + (size_t)i * batch * V, (size_t)rows * V * sizeof(T),
                                            cudaMemcpyHostToDevice, copy_stream));
                const void* staged = src_u8 ? (const void*)epoch_stage_u8[b].p
                                            : (src_bf16 ? (const void*)epoch_stage_bf16[b].p : (const void*)epoch_stage[b].p);
                staged_half = convert_on_copy_stream(b, staged, rows, batch, src, copy_stream) ? b : -1;
                BM_CUDA(cudaEventRecord(ev_copied[b], copy_stream));
                BM_CUDA(cudaStreamWaitEvent(ctx->stream, ev_copied[b], 0));
                if (src_u8) staged_u8 = epoch_stage_u8[b].p;
                else if (src_bf16) staged_bf16 = epoch_stage_bf16[b].p;
                else staged_dev = epoch_stage[b].p;
                const bool report = mask && every > 0 && ((iter0 + i + 1) % every == 0);
                defer_dst = epoch_host + 8 * i;
                train_step(nullptr, 0, rows, lr, mom, k, seed, tick0 + (uint32_t)i, report ? mask : 0u, unused);
                BM_CUDA(cudaEventRecord(ev_consumed[b], ctx->stream));
            }
        } catch (...) {
            staged_dev = nullptr; staged_u8 = nullptr; staged_bf16 = nullptr; staged_half = -1; defer_dst = nullptr;
            cudaStreamSynchronize(copy_stream); cudaStreamSynchronize(ctx->stream);
            throw;
        }
        staged_dev = nullptr; staged_u8 = nullptr; staged_bf16 = nullptr; staged_half = -1; defer_dst = nullptr;
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        for (int64_t i = 0; i < nb && mask; ++i) {
            const bool report = every > 0 && ((iter0 + i + 1) % every == 0);
            if (report) finish_metrics(epoch_host + 8 * i, mask, out + 4 * i);
            else for (int j = 0; j < 4; ++j) out[4 * i + j] = 0.0;
        }
    }

    void transform(const void* X_host, int rows, int k, uint64_t seed, uint32_t tick, void* H_out) override {
        BM_REQUIRE(rows >= 1, "empty batch");
        const T* X = stage_input(X_host, 0, rows, seed, tick, 0);
        chain(X, rows, k, seed, tick, 0);
        BM_CUDA(cudaMemcpyAsync(H_out, hm.p, (size_t)rows * H * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    void metrics(const void* X_host, int rows, int k, uint64_t seed, uint32_t tick, uint32_t mask, double* out) override {
        BM_REQUIRE(rows >= 1, "empty batch");
        const T* X = stage_input(X_host, 0, rows, seed, tick, 0);
        Xcur = X; last_rows = rows;
        if (mask & BM_METRIC_MSRE) chain(X, rows, k, seed, tick, 0);
        run_metrics(mask, rows, seed, tick, 0, out);
    }

    void get_activation(const char* name, void* host, size_t bytes) override {
        const T* src = nullptr; int n = 0;
        if (!strcmp(name, "X")) { src = Xcur; n = V; }
        else if (!strcmp(name, "h0_means")) { src = h0m.p; n = H; }
        else if (!strcmp(name, "h0_states")) { src = h0s_cur; n = H; }
        else if (!strcmp(name, "v_means")) { src = vm.p; n = V; }
        else if (!strcmp(name, "v_states")) { src = vs_cur; n = V; }
        else if (!strcmp(name, "h_means")) { src = hm.p; n = H; }
        else throw Error(BM_EINVAL, std::string("unknown activation '") + name + "'");
        BM_REQUIRE(src != nullptr && last_rows > 0, "no step has run yet");
        BM_REQUIRE(bytes == (size_t)last_rows * n * sizeof(T), "size mismatch");
        BM_CUDA(cudaMemcpyAsync(host, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
};

RbmBase* make_rbm_tc(Ctx* ctx, const bm_rbm_cfg& cfg);   // bm_rbm_tc.cu

}  // namespace bm
