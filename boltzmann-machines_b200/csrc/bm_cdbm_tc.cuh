// Classification DBM on the tensor cores (DESIGN.md §5.7): included by bm_dbm.cu after bm_crbm_tc.cuh.
//
// Units v - h_1 - ... - h_L - y with a one-of-C label y connected to h_L only; energy = the plain DBM energy - e_y'U h_L - yb'e_y
// (U [C, H_L], yb [C]).  The label is hidden layer L + 1 of a DbmTC: a multinomial layer with n_samples 1 whose weight is
// W_{L+1} = U^T ([H_L, C]), as in ClassRbmTC.  What the label adds to the plain engine:
//   E-step    the label slot of a row labelled t >= 0 is the one-hot e_t in every history slot and is never updated; a row
//             labelled -1 updates it like any multinomial layer (softmax, n_samples 1).  A batch without -1 runs no label op at
//             all (DbmTC::CLAMP_ALL: the top hidden op's second operand pair reads the one-hot slots, one program per chunk); a
//             mixed batch follows the label's row kernel with cdbm_clamp_labels_kernel (CLAMP_ROWS); a batch of -1 only is the
//             plain engine op for op (CLAMP_NONE).
//   particles k sweeps over v, h_1 .. h_L, y exactly as the plain engine: y is one categorical draw at site SITE_DBM_H + L.
//   update    as the plain engine for L + 1 layers; U takes l2, momentum and max-norm like any W; yb the plain momentum update
//             from sum q(y) / rows - sum y / M (DbmTC::top_is_label), without a sparsity term.
//   queries   predict_proba: the E-step with y free, then softmax(yb + mu_L U^T) from the final mu_L (one raw fp32 op and the
//             multinomial row kernel's fp32 output); transform: mu_L with y free.  log_proba and AIS are refused.
#pragma once

namespace bm {

struct CdbmShape {       // the arrays the engine's bm_dbm_cfg points into, alive while DbmTC's constructor reads them
    int32_t Hs[9], kinds[9], smp[9];
    double ns[9], spt[9], spc[9];
};

// the model's configuration plus the label layer on top
static inline bm_dbm_cfg cdbm_as_dbm(const bm_dbm_cfg& f, CdbmShape& s) {
    bm_dbm_cfg d = f;
    const int L = f.n_layers;
    for (int i = 0; i < L; ++i) {
        s.Hs[i] = f.n_hiddens[i]; s.kinds[i] = f.h_kinds[i]; s.smp[i] = f.sample_h[i];
        s.ns[i] = f.h_n_samples ? f.h_n_samples[i] : 100.0;
        s.spt[i] = f.sparsity_target[i]; s.spc[i] = f.sparsity_cost[i];
    }
    s.Hs[L] = f.n_classes; s.kinds[L] = BM_UNIT_MULTINOMIAL; s.smp[L] = 1;    // the label particles are always drawn
    s.ns[L] = 1.0; s.spt[L] = 0.0; s.spc[L] = 0.0;                          // one draw of a one-of-C group; no sparsity
    d.n_layers = L + 1;
    d.n_hiddens = s.Hs; d.h_kinds = s.kinds; d.sample_h = s.smp; d.h_n_samples = s.ns;
    d.sparsity_target = s.spt; d.sparsity_cost = s.spc;
    d.n_temps = 0; d.betas = nullptr; d.n_classes = 0;
    return d;
}

struct ClassDbmTC : DbmTC {
    int C, Lm;                               // classes; the model's hidden layers (the engine has Lm + 1, the label on top)
    DevBuf<int> lab;                         // [B] labels of the step (-1: unlabelled)
    DevBuf<float> proba;                     // [B, C] softmax(yb + mu_L U^T) of a predict_proba chunk
    DevBuf<bf16_t> proba_b;                  // the row kernel's bf16 output beside it (not read)

    // BM_EINVAL for shapes and n_classes; BM_EUNSUPPORTED naming the option otherwise.  Before anything is allocated.
    static void check_cfg(const Ctx* ctx, const bm_dbm_cfg& f) {
        BM_REQUIRE(f.n_classes >= 2, "classification DBM: n_classes must be 0 (no label layer) or at least 2");
        BM_REQUIRE(f.n_layers + 1 <= 8, "classification DBM: at most 7 hidden layers (the label layer is the 8th)");
        if (f.dtype != BM_DTYPE_F32)
            throw Error(BM_EUNSUPPORTED, "classification DBM: float32 models only, on the tensor-core engine (dtype float64 requested)");
        if (f.compute != BM_COMPUTE_BF16)
            throw Error(BM_EUNSUPPORTED, "classification DBM: runs on the tensor-core engine only (compute fp32 requested)");
        if (f.n_temps > 1) throw Error(BM_EUNSUPPORTED, "classification DBM: parallel tempering (n_temps > 1) is not supported");
        if (ctx->nranks > 1) throw Error(BM_EUNSUPPORTED, "classification DBM: a context with a communicator is not supported");
        CdbmShape s;
        if (!DbmTC::supports(cdbm_as_dbm(f, s)))
            throw Error(BM_EUNSUPPORTED, "classification DBM: the model does not run on the tensor-core engine (unit kinds)");
    }
    ClassDbmTC(Ctx* c, const bm_dbm_cfg& f, CdbmShape& s) : DbmTC(c, cdbm_as_dbm(f, s)) {
        C = f.n_classes; Lm = f.n_layers;
        top_is_label = true;
        lab.ensure(B); proba.ensure((size_t)B * C); proba_b.ensure((size_t)B * ldn[Lm + 1]);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    // ---- variables: the plain DBM's names for layers 0..L-1, plus U [C, H_L], yb, dU, dyb, y [M, C] and mu_y [B, C] ------
    // The engine's own names of the label layer ("W_L", "hb_L", ...) are not variables of the model.
    std::string engine_name(const std::string& n) const {
        const std::string s = sfx(Lm);
        for (const char* stem : {"W", "dW", "hb", "dhb", "q_means", "mu_means", "mu", "h"})
            if (n == stem + s) throw Error(BM_EINVAL, "unknown variable '" + n + "'");
        if (n == "U") return "W" + s;
        if (n == "dU") return "dW" + s;
        if (n == "yb") return "hb" + s;
        if (n == "dyb") return "dhb" + s;
        if (n == "y") return "h" + s;
        if (n == "mu_y") return "mu" + s;
        return n;
    }
    void set_param(const char* name, const void* host, size_t bytes) override {
        const std::string n(name);
        const int H = Hs[Lm - 1];
        if (n == "U" || n == "dU") {                           // [C, H_L] <-> W_{L+1} = U^T [H_L, C]
            BM_REQUIRE(bytes == (size_t)C * H * sizeof(float), "size mismatch for '" + n + "'");
            const float* src = static_cast<const float*>(host);
            std::vector<float> t((size_t)H * C);
            for (int y = 0; y < C; ++y) for (int j = 0; j < H; ++j) t[(size_t)j * C + y] = src[(size_t)y * H + j];
            DbmTC::set_param(engine_name(n).c_str(), t.data(), bytes);
            return;
        }
        DbmTC::set_param(engine_name(n).c_str(), host, bytes);
    }
    void get_param(const char* name, void* host, size_t bytes) override {
        const std::string n(name);
        const int H = Hs[Lm - 1];
        if (n == "U" || n == "dU") {
            BM_REQUIRE(bytes == (size_t)C * H * sizeof(float), "size mismatch for '" + n + "'");
            std::vector<float> t((size_t)H * C);
            DbmTC::get_param(engine_name(n).c_str(), t.data(), bytes);
            float* dst = static_cast<float*>(host);
            for (int y = 0; y < C; ++y) for (int j = 0; j < H; ++j) dst[(size_t)y * H + j] = t[(size_t)j * C + y];
            return;
        }
        DbmTC::get_param(engine_name(n).c_str(), host, bytes);
    }

    // ---- training -----------------------------------------------------------------------------------------------------
    // labels [rows] in [-1, C): checked, like the batch size, before anything is launched
    void train_step_labeled(const void* Xh, const int32_t* labels, int rows, double lr, double mom, int k, uint64_t seed,
                            uint32_t tick, int want, double* out) override {
        BM_REQUIRE(rows >= 1 && rows <= B, "a batch must have 1..batch_size rows");
        BM_REQUIRE(labels, "null labels");
        int unlabelled = 0;
        for (int r = 0; r < rows; ++r) {
            if (labels[r] < -1 || labels[r] >= C)
                throw Error(BM_EINVAL, "label " + std::to_string(labels[r]) + " of row " + std::to_string(r) + " is outside [-1, n_classes)");
            unlabelled += labels[r] == -1;
        }
        BM_REQUIRE(!want || out, "metrics requested without a buffer");
        if (unlabelled == rows) { DbmTC::train_step(Xh, rows, lr, mom, k, seed, tick, want, out); return; }
        BM_CUDA(cudaMemcpyAsync(lab.p, labels, (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
        mf_clamp = unlabelled ? CLAMP_ROWS : CLAMP_ALL;
        mf_labels = lab.p;
        try {
            DbmTC::train_step(Xh, rows, lr, mom, k, seed, tick, want, out);
        } catch (...) {
            mf_clamp = CLAMP_NONE;
            throw;
        }
        mf_clamp = CLAMP_NONE;
    }

    // ---- queries (y free in every row) ----------------------------------------------------------------------------------
    // q(y|x) = softmax(yb + mu_L U^T) in fp32 from the E-step's final mu_L, in chunks of batch_size rows
    void predict_proba(const void* Xh, int rows, float* out) override {
        BM_REQUIRE(rows >= 1, "empty batch");
        const float* X = static_cast<const float*>(Xh);
        for (int r0 = 0; r0 < rows; r0 += B) {
            const int n = std::min(B, rows - r0);
            upload_tc(X + (size_t)r0 * V, n);
            mean_field_tc(n);
            launch_tc_gemm(ctx, hidden_gemm(Lm, mu_b[Lm - 1].p, nullptr, proba_b.p, false, n, 1.f, 1.f, RngKey{}));   // -> pre_f32
            launch_dbm_multinomial_rows(ctx, pre_f32.p, C, n, C, 1.f, 0, proba_b.p, ldn[Lm + 1], proba.p, C, RngKey{});
            BM_CUDA(cudaMemcpyAsync(out + (size_t)r0 * C, proba.p, (size_t)n * C * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
            BM_CUDA(cudaStreamSynchronize(ctx->stream));
        }
    }
    void transform(const void* Xh, int rows, void* out) override {         // mu_L, the top hidden layer below the label
        upload_tc(Xh, rows);
        mean_field_tc(rows);
        BM_CUDA(cudaMemcpyAsync(out, mu[Lm - 1].p, (size_t)rows * Hs[Lm - 1] * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void exact(const void*, int, double*, double*) override {
        throw Error(BM_EUNSUPPORTED, "classification DBM: exact log Z is not supported (the enumeration has no label layer)");
    }
    void log_proba(const void*, int, double*) override {
        throw Error(BM_EUNSUPPORTED, "classification DBM: log_proba is not supported (the variational bound has no label layer)");
    }
    void ais_clamped(const void*, int, uint32_t, int, int, int, uint64_t, double*) override {
        throw Error(BM_EUNSUPPORTED, "classification DBM: AIS with v clamped is not supported (the AIS ladder has no label layer)");
    }
    void ais(int, int, int, uint64_t, const float* const*, double*) override {
        throw Error(BM_EUNSUPPORTED, "classification DBM: AIS is not supported (the AIS ladder has no label layer)");
    }
    void ais_rows(int, int, int, uint64_t, uint32_t, const float* const*, double*) override {
        throw Error(BM_EUNSUPPORTED, "classification DBM: AIS is not supported (the AIS ladder has no label layer)");
    }
};

}  // namespace bm
