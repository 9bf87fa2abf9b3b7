// Tensor-core RBM engine (BM_COMPUTE_BF16): the product path for float32 models.
//
// Variables (W, biases, momentum accumulators, q_means) stay in fp32 exactly as in the
// reference; every GEMM of the CD-k step -- h0, the 2k chain half-steps and the fused
// positive-minus-negative dW -- runs on the tensor cores (wgmma) with bf16 operands and fp32 accumulation, as ONE
// persistent dataflow launch (bm_tc.cu: TcProgram).  Activations live in L2/HBM as bf16 only
// (binary samples are exact in bf16).  A bf16 shadow of W is refreshed by the weight-update
// kernel.  Metrics (free energy / PLL) are evaluated in fp32 by the inherited CUDA-core kernels.
#include "bm_rbm.h"
#include "bm_peer.h"
#include <stdlib.h>
#include <string.h>
#include <map>
#include <memory>
#include <tuple>

namespace bm {

static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

struct RbmTC : RbmSimt<float> {
    typedef __nv_bfloat16 bf16;
    int ldw, ldv, ldh;
    DevBuf<bf16> Wb, Xb, h0m_b, h0s_b, vm_b, vs_b, hm_b, hs_b, data_b;
    DevBuf<float> partials, vparts, tstats, widen, q_alt;
    DevBuf<bf16> ones;             // [rows, 64] of 1.0: the B operand that turns a GEMM over the batch rows into column sums
    int tc_cap = 0;
    bool tc_kinds;
    // state of the last chain
    const bf16* X_b = nullptr; int X_ld = 0; int X_row0 = 0; int X_rows_total = 0;
    int X_mode = 0;       // 0: a buffer of exactly this batch; 1: rows [X_row0, ..) of the resident dataset; 2: a half of the epoch double buffer (1, 2: the program takes the row as its batch cursor)
    const bf16* vstate_b = nullptr;
    const bf16* h0state_b = nullptr;
    bool last_was_tc = false;
    // cached programs, keyed by (rows, k, with_dw, input buffer is the resident dataset)
    std::map<std::tuple<int, int, int, int>, std::unique_ptr<TcProgram>> progs;
    int dw_splits = 1, v_splits = 1;
    std::vector<bm_tc_op_plan> last_plan;          // the ops of the last run_program, all its launches (bm_rbm_debug_tc_plan)
    PeerExchange peer;             // data parallelism over NVLink peer memory (inactive on one rank / without peer access)
    // The batch buffers (X, v_k) carry two constant columns behind their V data columns -- (1, 0) for X, (1, 1) for v_k --
    // so that the dW GEMMs, run over V + 2 rows, also deliver sum(h0 - h_k) (row V) and -sum(h_k) (row V + 1): the
    // column statistics of base_rbm.py:453,457 cost no pass of their own.  sum(X - v_k) (:451) is two more ops of the
    // program ([V x 1] = X^T 1 - v_k^T 1).  Everything is summed and applied by ONE kernel (launch_cd_tail).
    // The constant columns sit at VP = V rounded up to 64, i.e. behind the last 64-column box a TMA store of the visible
    // activations can touch (seen on an earlier GPU: a store box that is clipped by the tensor edge inside a 16-byte unit
    // overwrites the rest of that unit).  Rows V .. VP-1 of the statistics are don't-cares.
    int VP() const { return (V + 63) / 64 * 64; }
    int VM() const { return VP() + 2; }
    // distance between two split-K slices: rounded up to 8 floats, so that every slice starts on a 32-byte boundary
    // whatever the shape (the vector paths of the epilogue, reduce_partials and the update rely on it)
    size_t gstride() const { return ((size_t)VM() * H + 7) & ~(size_t)7; }
    size_t vstride() const { return ((size_t)V + 7) & ~(size_t)7; }

    RbmTC(Ctx* c, const bm_rbm_cfg& f) : RbmSimt<float>(c, f) {
        ldw = round_up(H, 64); ldv = round_up(V, 64) + 64; ldh = round_up(H, 64);
        Wb.ensure((size_t)V * ldw);
        Wb.zero(ctx->stream);
        q_alt.ensure(H); q_alt.zero(ctx->stream);
        if (tc_kinds_of(f)) peer.setup(ctx, V, H, W.p, dW.p, Wb.p, ldw);      // collective when the context has peers
        tc_kinds = tc_kinds_of(f);
        reserve_tc(f.max_batch > 0 ? f.max_batch : 1);
    }

    bool accepts_bf16_feed() const override { return tc_kinds && cfg.v_kind != BM_UNIT_GAUSSIAN && cfg.dropout_keep < 0; }
    // every built-in unit kind runs its GEMMs on the tensor cores.  Bernoulli / Gaussian conditionals are fused into the
    // GEMM's epilogue and the whole chain is one program; a multinomial layer needs the whole row for its softmax
    // (layers.py:65-70), so its conditional is GEMM (raw fp32 pre-activations) -> row softmax -> categorical draws as
    // separate launches (`mixed`), the other layer's conditional staying fused.
    static bool tc_kinds_of(const bm_rbm_cfg& f) {
        auto ok = [](int k) { return k == BM_UNIT_BERNOULLI || k == BM_UNIT_MULTINOMIAL; };
        return ok(f.h_kind) && (ok(f.v_kind) || f.v_kind == BM_UNIT_GAUSSIAN);
    }
    bool mixed() const { return cfg.h_kind == BM_UNIT_MULTINOMIAL || cfg.v_kind == BM_UNIT_MULTINOMIAL; }

    void reserve_tc(int rows) {
        if (rows <= tc_cap) return;
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        tc_cap = rows;
        Xb.ensure((size_t)2 * rows * ldv);        // two halves: epochs convert batch i+1 on the copy stream while batch i is in use
        vm_b.ensure((size_t)rows * ldv); vs_b.ensure((size_t)rows * ldv);
        h0m_b.ensure((size_t)rows * ldh); h0s_b.ensure((size_t)rows * ldh);
        hm_b.ensure((size_t)rows * ldh); hs_b.ensure((size_t)rows * ldh);
        widen.ensure((size_t)rows * (V > H ? V : H));
        ones.ensure((size_t)rows * 64);
        launch_fill_bf16(ctx, ones.p, (size_t)rows * 64, 1.0f);
        for (DevBuf<bf16>* b : {&Xb, &vm_b, &vs_b}) b->zero(ctx->stream);       // (columns V .. VP-1 are read by the dW ops)
        launch_set_column_pair(ctx, Xb.p, ldv, (size_t)2 * rows, VP(), 1.0f, 0.0f);
        launch_set_column_pair(ctx, vm_b.p, ldv, (size_t)rows, VP(), 1.0f, 1.0f);
        launch_set_column_pair(ctx, vs_b.p, ldv, (size_t)rows, VP(), 1.0f, 1.0f);
        progs.clear();                         // buffers moved: cached descriptors are stale
    }

    // epochs (bm_rbm.h train_epoch): the uploaded batch becomes the bf16 operand on the copy stream, in the half of Xb the step
    // before last has finished with (ev_consumed[b], which the copy stream has already waited for)
    bool convert_on_copy_stream(int b, const void* staged, int rows, int batch, int src, cudaStream_t copy) override {
        static int enabled = -1;
        if (enabled < 0) { const char* e = getenv("BM_EPOCH_CONVERT_ON_COPY_STREAM"); enabled = e ? atoi(e) : 1; }
        const bool plain = (cfg.v_kind != BM_UNIT_GAUSSIAN) && (cfg.dropout_keep < 0);
        if (!enabled || !plain || !tc_kinds || (src != SRC_U8 && src != SRC_BF16)) return false;
        if (batch > tc_cap) {
            reserve_tc(batch);
            BM_CUDA(cudaStreamSynchronize(ctx->stream));      // the buffers' constant columns are written on the compute stream
        }
        bf16* dst = Xb.p + (size_t)b * tc_cap * ldv;
        if (src == SRC_U8) launch_u8_to_bf16(ctx, (const uint8_t*)staged, V, dst, ldv, rows, V, copy);
        else BM_CUDA(cudaMemcpy2DAsync(dst, (size_t)ldv * 2, staged, (size_t)V * 2, (size_t)V * 2, (size_t)rows,
                                       cudaMemcpyDeviceToDevice, copy));
        return true;
    }

    void refresh_shadow() { launch_f32_to_bf16(ctx, W.p, H, Wb.p, ldw, V, H); }
    void get_param(const char* name, void* host, size_t bytes) override {
        if (!strcmp(name, "W") || !strcmp(name, "dW")) peer.pull_replicas();      // (data parallel: rows of the other ranks' shards)
        RbmSimt<float>::get_param(name, host, bytes);
    }

    void set_param(const char* name, const void* host, size_t bytes) override {
        RbmSimt<float>::set_param(name, host, bytes);
        if (!strcmp(name, "W")) { refresh_shadow(); BM_CUDA(cudaStreamSynchronize(ctx->stream)); }
    }
    void init_weights(double stddev, uint64_t op_seed) override {
        RbmSimt<float>::init_weights(stddev, op_seed);
        refresh_shadow();
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    void set_data(const void* X, int64_t n_rows) override {
        RbmSimt<float>::set_data(X, n_rows);
        data_b.ensure((size_t)n_rows * ldv);
        data_b.zero(ctx->stream);
        launch_f32_to_bf16(ctx, data.p, V, data_b.p, ldv, (int)n_rows, V);
        launch_set_column_pair(ctx, data_b.p, ldv, (size_t)n_rows, VP(), 1.0f, 0.0f);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        progs.clear();
    }

    TcMat mat(const bf16* p, int rows, int cols, int ld) const { TcMat m; m.ptr = p; m.rows = rows; m.cols = cols; m.ld = ld; return m; }

    // one conditional (a Gibbs half-step) as a tensor-core op
    TcGemm layer_op(bool up, TcMat in, bool in_is_batch_cursor, bf16* means, bf16* states, bool sample,
                    uint32_t site, uint32_t t, int rows) {
        TcGemm g;
        g.M = rows; g.N = up ? H : V;
        g.A[0] = in; g.a_batch[0] = in_is_batch_cursor; g.K[0] = up ? V : H;
        g.B[0] = mat(Wb.p, V, H, ldw);
        g.b_t[0] = up;                 // v W: W is [K=V, N=H] (N contiguous); h W^T: W is [N=V, K=H] (K contiguous)
        const float mult = (float)(up ? cfg.propup_mult : cfg.propdown_mult);    // base_rbm.py:342-343,356-357
        g.acc_scale = mult; g.bias_scale = mult;
        g.bias = up ? hb.p : vb.p;
        g.rng = make_rng(0, site, t, 0, 0);
        { const char* e = getenv(up ? "BM_TC_BN_UP" : "BM_TC_BN_DOWN"); if (e) g.force_bn = atoi(e); }
        g.out_mean_bf = means; g.ld_mean_bf = up ? ldh : ldv;
        const int kind = up ? cfg.h_kind : cfg.v_kind;
        if (kind == BM_UNIT_BERNOULLI) {
            g.act = ACT_SIGMOID;
            if (sample) { g.sample = SMP_BERNOULLI; g.out_state_bf = states; g.ld_state_bf = g.ld_mean_bf; }
        } else {
            g.act = ACT_LINEAR; g.sigma = sigma.p;                                // layers.py:84-86
            if (sample) { g.sample = SMP_GAUSSIAN; g.noise_sigma = sigma.p; g.out_state_bf = states; g.ld_state_bf = g.ld_mean_bf; }
        }
        return g;
    }

    // input staging: fp32 prepared batch (inherited) -> bf16, or a slice of the resident bf16 dataset
    void stage_tc(const void* X_host, int64_t first_row, int rows, uint64_t seed, uint32_t tick, uint32_t row0) {
        reserve_tc(rows);
        const bool plain = (cfg.v_kind != BM_UNIT_GAUSSIAN) && (cfg.dropout_keep < 0);
        X_mode = 0;
        if (staged_half >= 0) {
            // epoch data already converted into a half of Xb by the copy stream (convert_on_copy_stream)
            reserve(rows);
            X_b = Xb.p; X_ld = ldv; X_row0 = staged_half * tc_cap; X_rows_total = 2 * tc_cap; X_mode = 2;
            Xcur = nullptr;
        } else if (staged_bf16) {
            // real-valued epoch data fed as bfloat16 (accepted only when `plain`): the bits the fp32 -> bf16 conversion of the
            // float feed would produce, so the chain is bit-identical at half the host->device bytes
            BM_REQUIRE(plain, "a bfloat16 feed needs a model without dropout / sigma scaling");
            reserve(rows);
            BM_CUDA(cudaMemcpy2DAsync(Xb.p, (size_t)ldv * 2, staged_bf16, (size_t)V * 2, (size_t)V * 2, (size_t)rows,
                                      cudaMemcpyDeviceToDevice, ctx->stream));
            X_b = Xb.p; X_ld = ldv; X_row0 = 0; X_rows_total = rows;
            Xcur = nullptr;
        } else if (staged_u8 && plain) {
            // byte-valued epoch data goes straight to the bf16 operand buffer; the fp32 copy the CUDA-core
            // metric kernels read is made only when such a metric is requested (ensure_fp32_input)
            reserve(rows);
            launch_u8_to_bf16(ctx, staged_u8, V, Xb.p, ldv, rows, V);
            X_b = Xb.p; X_ld = ldv; X_row0 = 0; X_rows_total = rows;
            Xcur = nullptr;
        } else if (!X_host && !staged_dev && !staged_u8 && plain) {
            BM_REQUIRE(first_row >= 0 && first_row + rows <= data_rows, "row range outside the resident dataset");
            reserve(rows);
            X_b = data_b.p; X_ld = ldv; X_row0 = (int)first_row; X_rows_total = (int)data_rows; X_mode = 1;
            Xcur = data.p + (size_t)first_row * V;
        } else {
            const float* X = stage_input(X_host, first_row, rows, seed, tick, row0);
            launch_f32_to_bf16(ctx, X, V, Xb.p, ldv, rows, V);
            X_b = Xb.p; X_ld = ldv; X_row0 = 0; X_rows_total = rows;
            Xcur = X;
        }
        last_rows = rows;
    }

    // fp32 view of the current batch for the free-energy / PLL kernels (exact: bf16 holds 0..255 and the
    // resident/converted inputs were rounded to bf16 once already)
    void ensure_fp32_input(int rows) {
        if (Xcur) return;
        launch_bf16_to_f32(ctx, X_b + (size_t)X_row0 * X_ld, X_ld, Xin.p, V, rows, V);
        Xcur = Xin.p;
    }
    // MSRE straight from the bf16 activations of the last chain (no widened copies)
    bool msre_from_activations(int rows, double* dst) override {
        if (!last_was_tc) return false;
        launch_sqdiff_mean_bf16(ctx, X_b + (size_t)X_row0 * X_ld, X_ld, vm_b.p, ldv, rows, V, (double)rows * V, dst);
        return true;
    }

    // The whole chain (base_rbm.py:421-426, 367-384) -- and, for training, the fused dW
    // (base_rbm.py:447-448) -- as ONE persistent launch.
    void run_program(int rows, int k, bool with_dw, uint64_t seed, uint32_t tick, uint32_t row0) {
        BM_REQUIRE(k >= 1, "n_gibbs_steps must be >= 1");
        last_plan.clear();
        const bool resident = X_mode != 0;           // the input is addressed through the launch's batch cursor
        auto key = std::make_tuple(rows, k, with_dw ? 1 : 0, X_mode);
        std::unique_ptr<TcProgram>& slot = progs[key];
        if (!slot) slot.reset(new TcProgram());
        TcProgram& prog = *slot;
        const bool sh = cfg.sample_h != 0, sv = cfg.sample_v != 0;
        std::vector<TcGemm>& ops = prog.ops;
        ops.clear();
        const bool in_program = !mixed();          // mixed: the chain has just run launch by launch (chain_mixed)
        const bf16* hstate = nullptr;
        if (in_program) {
            // rows of the resident dataset beyond this batch only produce output rows >= M, which are masked
            ops.push_back(layer_op(true, mat(X_b, X_rows_total, V, X_ld), resident, h0m_b.p, h0s_b.p, sh, SITE_H0, 0, rows));
            if (!resident) ops.back().a_row0[0] = X_row0;
            h0state_b = sh ? h0s_b.p : h0m_b.p;
            hstate = h0state_b;
            int prev = 0;
            for (int t = 1; t <= k; ++t) {
                // outputs nobody reads are not written: sampled visibles need their means only at the
                // last step (MSRE), sampled mid-chain hiddens never need theirs
                const bool last = (t == k);
                TcGemm gv = layer_op(false, mat(hstate, rows, H, ldh), false, (sv && !last) ? nullptr : vm_b.p, vs_b.p, sv, SITE_V, t, rows);
                gv.n_deps = 1; gv.dep[0] = prev;
                ops.push_back(gv); prev = (int)ops.size() - 1;
                vstate_b = sv ? vs_b.p : vm_b.p;
                const bool smp = sh && !last;
                TcGemm gh = layer_op(true, mat(vstate_b, rows, V, ldv), false, smp ? nullptr : hm_b.p, hs_b.p, smp, SITE_H, t, rows);
                gh.n_deps = 1; gh.dep[0] = prev;
                ops.push_back(gh); prev = (int)ops.size() - 1;
                hstate = smp ? hs_b.p : hm_b.p;
            }
        }
        if (with_dw) {
            // dW_positive - dW_negative (base_rbm.py:447-448): G = X^T h0_means - v_k^T h_k_means, K = the batch rows,
            // split over K so that every CTA pair gets a slice; the slices are summed by the update kernel.  The operands'
            // constant columns add the rows V, V + 1 (see VM()).
            const int total_pairs = ctx->sm_count / 2;
            const int pair_tiles = ((VM() + 255) / 256) * ((H + 255) / 256);
            const int v_groups = (V + 255) / 256;
            const int row_chunks = (rows + 63) / 64;
            auto operand_x = [&](TcGemm& g, int pr, int cols) {
                g.A[pr] = mat(X_b, X_rows_total, cols, X_ld); g.a_t[pr] = true; g.a_batch[pr] = resident;
                if (!resident) g.a_k0[pr] = X_row0;
                g.K[pr] = rows;
            };
            auto operand_v = [&](TcGemm& g, int pr, int cols) {
                g.A[pr] = mat(vstate_b, rows, cols, ldv); g.a_t[pr] = true; g.neg[pr] = true; g.K[pr] = rows;
            };
            auto dw_op = [&](bool pos, bool neg) {
                TcGemm g;
                g.M = VM(); g.N = H; g.n_pairs = (pos && neg) ? 2 : 1;
                int pr = 0;
                if (pos) { operand_x(g, pr, VM()); g.B[pr] = mat(h0m_b.p, rows, H, ldh); g.b_t[pr] = true; ++pr; }
                if (neg) { operand_v(g, pr, VM()); g.B[pr] = mat(hm_b.p, rows, H, ldh); g.b_t[pr] = true; }
                g.split_stride = gstride(); g.ld_f32 = H;
                return g;
            };
            auto colsum_op = [&](bool pos, bool neg) {            // [V x 1] = X^T 1 - v_k^T 1
                TcGemm g;
                g.M = V; g.N = 1; g.n_pairs = (pos && neg) ? 2 : 1;
                int pr = 0;
                if (pos) { operand_x(g, pr, V); g.B[pr] = mat(ones.p, rows, 64, 64); g.b_t[pr] = true; ++pr; }
                if (neg) { operand_v(g, pr, V); g.B[pr] = mat(ones.p, rows, 64, 64); g.b_t[pr] = true; }
                g.split_stride = vstride(); g.ld_f32 = 1;
                return g;
            };
            // The positive statistics depend on the input and h0 only.  When the chain leaves CTA pairs idle and is long enough
            // to hide them, they run on those pairs BESIDE the chain and only the negative ones are left for the end of the step.
            // The cycle counts below (per K chunk of a statistics unit, per chain half-step) are rough estimates carried over
            // from an earlier GPU; they are not measured on the H100.
            if (prog.chain_units < 0)            // shapes are fixed per cached program: plan once
                for (const TcGemm& o : ops) prog.chain_units = std::max(prog.chain_units, tc_plan_units(ctx, o));
            const int chain_units = prog.chain_units;
            const int spare = in_program ? total_pairs - chain_units : 0;
            int pos_splits = 0;
            if (spare >= 2 && pair_tiles > 0) {
                pos_splits = std::max(1, std::min(spare / pair_tiles, row_chunks));
                const int rounds = (pair_tiles * pos_splits + spare - 1) / spare;
                const double pos_cycles = (double)rounds * ((double)(row_chunks / pos_splits + 1) * 600.0 + 10000.0);
                const double chain_cycles = (double)(2 * k) * 20000.0;
                if (pos_cycles > 0.8 * chain_cycles) pos_splits = 0;
            }
            { const char* e = getenv("BM_TC_DW_OVERLAP"); if (e && !atoi(e)) pos_splits = 0; }
            if ((int)ops.size() + 4 > TC_PROGRAM_OPS) pos_splits = 0;      // a chain cut into several launches keeps its statistics at the end
            const int last_v = (int)ops.size() - 2, last_h = (int)ops.size() - 1;
            if (pos_splits > 0) {
                const int neg_splits = std::max(1, std::min(total_pairs / pair_tiles, row_chunks));
                const int xs = std::max(1, std::min(spare / v_groups, row_chunks));
                const int vs = std::max(1, std::min(2 * spare / v_groups, row_chunks));
                dw_splits = pos_splits + neg_splits;
                v_splits = xs + vs;
                partials.ensure((size_t)dw_splits * gstride());
                vparts.ensure((size_t)v_splits * vstride());
                TcGemm gx = colsum_op(true, false);                // no dependency: the input is there from the start
                gx.splits = xs; gx.out_f32 = vparts.p; gx.lane = LANE_SPARE;
                TcGemm gp = dw_op(true, false);
                gp.splits = pos_splits; gp.out_f32 = partials.p;
                gp.n_deps = 1; gp.dep[0] = 0; gp.dep_all[0] = true;
                gp.lane = LANE_SPARE;
                // program order: right after h0, so that the spare pairs meet them first
                ops.insert(ops.begin() + 1, gp);
                ops.insert(ops.begin() + 1, gx);
                for (size_t i = 3; i < ops.size(); ++i)
                    for (int d = 0; d < ops[i].n_deps; ++d) if (ops[i].dep[d] >= 1) ops[i].dep[d] += 2;
                TcGemm gv = colsum_op(false, true);                // beside the last hidden half-step
                gv.splits = vs; gv.out_f32 = vparts.p + (size_t)xs * vstride();
                gv.n_deps = 1; gv.dep[0] = last_v + 2; gv.dep_all[0] = true;
                gv.lane = LANE_SPARE;
                ops.push_back(gv);
                TcGemm gn = dw_op(false, true);
                gn.splits = neg_splits; gn.out_f32 = partials.p + (size_t)pos_splits * gstride();
                gn.n_deps = 2; gn.dep[0] = last_v + 2; gn.dep[1] = last_h + 2; gn.dep_all[0] = gn.dep_all[1] = true;
                gn.lane = LANE_ALL;
                ops.push_back(gn);
            } else {
                TcGemm gc = colsum_op(true, true);
                int vs = std::max(1, std::min(total_pairs / v_groups, 2 * row_chunks));
                v_splits = vs;
                gc.splits = vs;
                vparts.ensure((size_t)vs * vstride());
                gc.out_f32 = vparts.p;
                if (in_program) { gc.n_deps = 1; gc.dep[0] = last_v; gc.dep_all[0] = true; }
                gc.lane = LANE_ALL;
                ops.push_back(gc);
                TcGemm g = dw_op(true, true);
                int splits = total_pairs / (pair_tiles > 0 ? pair_tiles : 1);
                if (splits < 1) splits = 1;
                if (splits > 2 * row_chunks) splits = 2 * row_chunks;
                dw_splits = splits;
                g.splits = splits;
                partials.ensure((size_t)splits * gstride());
                g.out_f32 = partials.p;
                if (in_program) {
                    g.n_deps = 3;
                    g.dep[0] = 0; g.dep[1] = last_v; g.dep[2] = last_h;
                    g.dep_all[0] = g.dep_all[1] = g.dep_all[2] = true;
                }
                g.lane = LANE_ALL;
                ops.push_back(g);
            }
        }
        if ((int)ops.size() <= TC_PROGRAM_OPS) {
            if (!ops.empty()) launch_tc_program(ctx, prog, make_rng(seed, 0, 0, tick, row0), resident ? X_row0 : 0, &last_plan);
        } else {
            // a chain longer than one program holds (CD-k with 2k + 3 > 96 ops; the reference has no such limit,
            // base_rbm.py:386-405): consecutive launches of up to TC_PROGRAM_OPS ops -- a dependency on an op of an earlier launch is
            // the kernel boundary
            const std::vector<TcGemm> all = ops;
            ops.clear();                         // (the cached whole-chain program object only keeps the plan)
            for (size_t lo = 0, c = 1; lo < all.size(); lo += (size_t)TC_PROGRAM_OPS, ++c) {
                const size_t hi = std::min(all.size(), lo + (size_t)TC_PROGRAM_OPS);
                std::unique_ptr<TcProgram>& part = progs[std::make_tuple(rows, k, (with_dw ? 1 : 0) | (int)(c << 1), X_mode)];
                if (!part) part.reset(new TcProgram());
                part->ops.assign(all.begin() + lo, all.begin() + hi);
                for (TcGemm& g : part->ops) {
                    int n = 0;
                    for (int d = 0; d < g.n_deps; ++d)
                        if (g.dep[d] >= (int)lo) { g.dep[n] = g.dep[d] - (int)lo; g.dep_all[n] = g.dep_all[d]; ++n; }
                    g.n_deps = n;
                    if (g.lane == LANE_SPARE) g.lane = LANE_ALL;
                }
                const size_t first = last_plan.size();
                launch_tc_program(ctx, *part, make_rng(seed, 0, 0, tick, row0), resident ? X_row0 : 0, &last_plan);
                for (size_t i = first; i < last_plan.size(); ++i) last_plan[i].launch = (int32_t)(c - 1);
            }
        }
        last_was_tc = true;
    }

    // One conditional of a model with a multinomial layer, launch by launch: the GEMM on the tensor cores, then (multinomial
    // side) M * softmax over the row and the categorical draws on the fp32 pre-activations (layers.py:65-70; sampling reads the
    // UNROUNDED means, like the oracle), bf16 copies for the next GEMM.
    void half_step_mixed(bool up, TcMat in, bool in_is_batch_cursor, bf16* means_b, bf16* states_b, bool sample,
                         uint32_t site, uint32_t t, int rows, uint64_t seed, uint32_t tick, uint32_t row0) {
        const int kind = up ? cfg.h_kind : cfg.v_kind;
        const int N = up ? H : V, ldo = up ? ldh : ldv;
        const RngKey rng = make_rng(seed, site, t, tick, row0);
        if (kind != BM_UNIT_MULTINOMIAL) {
            TcGemm g = layer_op(up, in, in_is_batch_cursor, means_b, states_b, sample, site, t, rows);
            g.rng = rng;
            if (in_is_batch_cursor) { g.a_batch[0] = false; g.a_row0[0] = X_row0; }       // single launches carry no batch cursor
            launch_tc_gemm(ctx, g);
            return;
        }
        float* pre = up ? hm.p : vm.p;             // fp32 workspaces of the storage-precision engine (reserve())
        float* st = up ? hs.p : vs.p;
        TcGemm g;
        g.M = rows; g.N = N;
        g.A[0] = in; g.K[0] = up ? V : H;
        if (in_is_batch_cursor) g.a_row0[0] = X_row0;
        g.B[0] = mat(Wb.p, V, H, ldw); g.b_t[0] = up;
        const float mult = (float)(up ? cfg.propup_mult : cfg.propdown_mult);
        g.acc_scale = mult; g.bias_scale = mult; g.bias = up ? hb.p : vb.p;
        g.act = ACT_LINEAR;
        g.out_f32 = pre; g.ld_f32 = N;
        launch_tc_gemm(ctx, g);
        const double M = up ? cfg.h_n_samples : cfg.v_n_samples;
        launch_softmax_rows<float>(ctx, pre, N, rows, N, (float)M);
        if (sample) {
            launch_multinomial_rows<float>(ctx, pre, N, rows, N, (int)M, st, N, rng);
            launch_f32_to_bf16(ctx, st, N, states_b, ldo, rows, N);
        }
        if (means_b) launch_f32_to_bf16(ctx, pre, N, means_b, ldo, rows, N);
    }
    void chain_mixed(int rows, int k, uint64_t seed, uint32_t tick, uint32_t row0) {
        BM_REQUIRE(k >= 1, "n_gibbs_steps must be >= 1");
        reserve(rows);
        const bool resident = (X_b == data_b.p);
        const bool sh = cfg.sample_h != 0, sv = cfg.sample_v != 0;
        half_step_mixed(true, mat(X_b, X_rows_total, V, X_ld), true, h0m_b.p, h0s_b.p, sh, SITE_H0, 0, rows, seed, tick, row0);
        (void)resident;
        h0state_b = sh ? h0s_b.p : h0m_b.p;
        const bf16* hstate = h0state_b;
        for (int t = 1; t <= k; ++t) {
            const bool last = (t == k);
            half_step_mixed(false, mat(hstate, rows, H, ldh), false, vm_b.p, vs_b.p, sv, SITE_V, t, rows, seed, tick, row0);
            vstate_b = sv ? vs_b.p : vm_b.p;
            const bool smp = sh && !last;
            half_step_mixed(true, mat(vstate_b, rows, V, ldv), false, hm_b.p, hs_b.p, smp, SITE_H, t, rows, seed, tick, row0);
            hstate = smp ? hs_b.p : hm_b.p;
        }
    }

    void train_step(const void* X_host, int64_t first_row, int rows, double lr, double mom, int k,
                    uint64_t seed, uint32_t tick, uint32_t mask, double* out) override {
        if (!tc_kinds) { last_was_tc = false; RbmSimt<float>::train_step(X_host, first_row, rows, lr, mom, k, seed, tick, mask, out); refresh_shadow(); return; }
        BM_REQUIRE(rows >= 1, "empty batch");
        const uint32_t row0 = (uint32_t)(ctx->rank * rows);
        stage_tc(X_host, first_row, rows, seed, tick, row0);
        if (mixed()) chain_mixed(rows, k, seed, tick, row0);
        run_program(rows, k, true, seed, tick, row0);
        if (mask) {
            if (mask & (BM_METRIC_PLL | BM_METRIC_FREE_ENERGY | BM_METRIC_L2_LOSS)) peer.pull_replicas();   // these read the fp32 W
            if (mask & (BM_METRIC_PLL | BM_METRIC_FREE_ENERGY)) ensure_fp32_input(rows);
            run_metrics(mask, rows, seed, tick, row0, out);
        }

        if (peer.active) {
            // with NVLink peers: reduce-scatter, sharded update and all-gather of the weights as stores to peer memory (bm_peer.h)
            DpStep s{};
            peer.fill(s);
            s.part = partials.p; s.stride = gstride(); s.splits = dw_splits; s.srow = VP();
            s.vpart = vparts.p; s.vstride = vstride(); s.vsplits = v_splits;
            s.n_div = (float)((double)rows * ctx->nranks);
            s.lr = (float)lr; s.mom = (float)mom; s.l2 = (float)cfg.l2;
            s.damp = (float)cfg.sparsity_damping; s.cost = (float)cfg.sparsity_cost; s.target = (float)cfg.sparsity_target;
            s.vb = vb.p; s.hb = hb.p; s.dvb = dvb.p; s.dhb = dhb.p;
            s.q_old = q.p; s.q_new = q_alt.p; s.pen = pen.p;
            peer.run(s);
            std::swap(q.p, q_alt.p);
            return;
        }
        CdTail t{};
        t.V = V; t.H = H;
        t.part = partials.p; t.stride = gstride(); t.splits = dw_splits; t.srow = VP();
        t.vpart = vparts.p; t.vstride = vstride(); t.vsplits = v_splits;
        if (ctx->nranks > 1) {
            // with peers: sum this rank's slices, one all-reduce over [G' | sum(X - v_k)], then the same update on every rank
            tstats.ensure(gstride() + vstride());
            launch_reduce_partials(ctx, partials.p, gstride(), dw_splits, tstats.p, (size_t)VM() * H);
            launch_reduce_partials(ctx, vparts.p, vstride(), v_splits, tstats.p + gstride(), (size_t)V);
            allreduce_sum(ctx, tstats.p, gstride() + vstride(), false);
            t.part = tstats.p; t.splits = 1; t.vpart = tstats.p + gstride(); t.vsplits = 1;
        }
        t.n_div = (float)((double)rows * ctx->nranks);
        t.lr = (float)lr; t.mom = (float)mom; t.l2 = (float)cfg.l2;
        t.damp = (float)cfg.sparsity_damping; t.cost = (float)cfg.sparsity_cost; t.target = (float)cfg.sparsity_target;
        t.W = W.p; t.dW = dW.p; t.vb = vb.p; t.hb = hb.p; t.dvb = dvb.p; t.dhb = dhb.p;
        t.q_old = q.p; t.q_new = q_alt.p; t.pen = pen.p;
        t.Wb = Wb.p; t.ldwb = ldw;
        launch_cd_tail(ctx, t);
        std::swap(q.p, q_alt.p);               // (same size; "q_means" names the current one)
    }

    void transform(const void* X_host, int rows, int k, uint64_t seed, uint32_t tick, void* H_out) override {
        if (!tc_kinds) { last_was_tc = false; RbmSimt<float>::transform(X_host, rows, k, seed, tick, H_out); return; }
        BM_REQUIRE(rows >= 1, "empty batch");
        stage_tc(X_host, 0, rows, seed, tick, 0);
        if (mixed()) chain_mixed(rows, k, seed, tick, 0);
        run_program(rows, k, false, seed, tick, 0);
        launch_bf16_to_f32(ctx, hm_b.p, ldh, widen.p, H, rows, H);
        BM_CUDA(cudaMemcpyAsync(H_out, widen.p, (size_t)rows * H * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    void metrics(const void* X_host, int rows, int k, uint64_t seed, uint32_t tick, uint32_t mask, double* out) override {
        if (!tc_kinds) { last_was_tc = false; RbmSimt<float>::metrics(X_host, rows, k, seed, tick, mask, out); return; }
        BM_REQUIRE(rows >= 1, "empty batch");
        stage_tc(X_host, 0, rows, seed, tick, 0);
        if (mask & (BM_METRIC_PLL | BM_METRIC_FREE_ENERGY | BM_METRIC_L2_LOSS)) peer.pull_replicas();
        if ((mask & BM_METRIC_MSRE) && mixed()) chain_mixed(rows, k, seed, tick, 0);
        if (mask & BM_METRIC_MSRE) run_program(rows, k, false, seed, tick, 0);
        if (mask & (BM_METRIC_PLL | BM_METRIC_FREE_ENERGY)) ensure_fp32_input(rows);
        run_metrics(mask, rows, seed, tick, 0, out);
    }

    const std::vector<bm_tc_op_plan>& tc_plan() const override { return last_plan; }

    void get_activation(const char* name, void* host, size_t bytes) override {
        if (!last_was_tc) { RbmSimt<float>::get_activation(name, host, bytes); return; }
        const bf16* src = nullptr; int n = 0, ld = 0;
        if (!strcmp(name, "X")) { src = X_b + (size_t)X_row0 * X_ld; n = V; ld = X_ld; }
        else if (!strcmp(name, "h0_means")) { src = h0m_b.p; n = H; ld = ldh; }
        else if (!strcmp(name, "h0_states")) { src = h0state_b; n = H; ld = ldh; }
        else if (!strcmp(name, "v_means")) { src = vm_b.p; n = V; ld = ldv; }
        else if (!strcmp(name, "v_states")) { src = vstate_b; n = V; ld = ldv; }
        else if (!strcmp(name, "h_means")) { src = hm_b.p; n = H; ld = ldh; }
        else throw Error(BM_EINVAL, std::string("unknown activation '") + name + "'");
        BM_REQUIRE(src != nullptr && last_rows > 0, "no step has run yet");
        BM_REQUIRE(bytes == (size_t)last_rows * n * sizeof(float), "size mismatch");
        launch_bf16_to_f32(ctx, src, ld, widen.p, n, last_rows, n);
        BM_CUDA(cudaMemcpyAsync(host, widen.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
    }
};

RbmBase* make_rbm_tc(Ctx* ctx, const bm_rbm_cfg& cfg) { return new RbmTC(ctx, cfg); }

}  // namespace bm

using namespace bm;

extern "C" int bm_debug_tc_gemm(bm_ctx* hctx, int32_t M, int32_t N, int32_t K, const float* A, int32_t a_t,
                                const float* B, int32_t b_t, int32_t K2, const float* A2, const float* B2,
                                int32_t neg2, int32_t splits, int32_t force_bn, int32_t force_cluster, float* C) {
    BM_API_BEGIN
    Ctx* ctx = reinterpret_cast<Ctx*>(hctx);
    BM_REQUIRE(ctx && A && B && C && M > 0 && N > 0 && K > 0, "bad argument");
    BM_CUDA(cudaSetDevice(ctx->device));
    TcGemm g;
    g.M = M; g.N = N; g.n_pairs = (K2 > 0) ? 2 : 1;
    DevBuf<float> stage; DevBuf<__nv_bfloat16> bufs[4]; DevBuf<float> out;
    const float* hosts[4] = {A, B, A2, B2};
    for (int i = 0; i < 2 * g.n_pairs; ++i) {
        const int pr = i / 2; const bool isA = (i % 2) == 0;
        const int Kp = pr ? K2 : K;
        const bool t = isA ? (a_t != 0) : (b_t != 0);
        const int mn = isA ? M : N;
        const int rows = t ? Kp : mn, cols = t ? mn : Kp;
        const int ld = round_up(cols, 8);
        stage.ensure((size_t)rows * cols);
        bufs[i].ensure((size_t)rows * ld);
        BM_CUDA(cudaMemcpyAsync(stage.p, hosts[i], (size_t)rows * cols * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        launch_f32_to_bf16(ctx, stage.p, cols, bufs[i].p, ld, rows, cols);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        TcMat m; m.ptr = bufs[i].p; m.rows = rows; m.cols = cols; m.ld = ld;
        if (isA) { g.A[pr] = m; g.a_t[pr] = t; } else { g.B[pr] = m; g.b_t[pr] = t; }
        g.K[pr] = Kp;
    }
    g.neg[1] = neg2 != 0;
    g.splits = splits > 0 ? splits : 1;
    g.force_bn = force_bn; g.force_cluster = force_cluster;
    DevBuf<unsigned long long> dbg;
    const char* tl = getenv("BM_TC_TIMELINE");
    if (tl) { dbg.ensure(64); dbg.zero(ctx->stream); g.dbg = dbg.p; }
    g.split_stride = (size_t)M * N;
    const int ldc = round_up(N, 4);
    g.split_stride = (size_t)M * ldc;
    out.ensure((size_t)g.splits * M * ldc);
    g.out_f32 = out.p; g.ld_f32 = ldc;
    // BM_TC_EPI=1|2|3: time the hot bf16 epilogues instead of the raw fp32 one (results are not returned)
    DevBuf<__nv_bfloat16> obf1, obf2;
    const char* epi = getenv("BM_TC_EPI");
    if (epi && g.splits == 1) {
        const int md = atoi(epi);
        const int ldo = round_up(N, 8);
        obf1.ensure((size_t)M * ldo); obf2.ensure((size_t)M * ldo);
        g.out_f32 = nullptr; g.act = ACT_SIGMOID;
        if (md == 1 || md == 3) { g.out_mean_bf = obf1.p; g.ld_mean_bf = ldo; }
        if (md == 1 || md == 2) { g.out_state_bf = obf2.p; g.ld_state_bf = ldo; g.sample = SMP_BERNOULLI; g.rng = make_rng(1, 1, 0, 0, 0); }
    }
    const char* reps = getenv("BM_TC_REPS");
    for (int i = 0, n = reps ? atoi(reps) : 0; i < n; ++i) { g.dbg = nullptr; launch_tc_gemm(ctx, g); }
    g.dbg = tl ? dbg.p : nullptr;
    launch_tc_gemm(ctx, g);
    DevBuf<float> red;
    const float* res = out.p;
    if (g.splits > 1) {
        red.ensure((size_t)M * ldc);
        launch_reduce_partials(ctx, out.p, (size_t)M * ldc, g.splits, red.p, (size_t)M * ldc);
        res = red.p;
    }
    if (g.out_f32) BM_CUDA(cudaMemcpy2DAsync(C, (size_t)N * sizeof(float), res, (size_t)ldc * sizeof(float), (size_t)N * sizeof(float), M,
                                             cudaMemcpyDeviceToHost, ctx->stream));
    BM_CUDA(cudaStreamSynchronize(ctx->stream));
    if (tl) {
        unsigned long long h[64];
        BM_CUDA(cudaMemcpy(h, dbg.p, sizeof(h), cudaMemcpyDeviceToHost));
        fprintf(stderr, "timeline(SM cycles from kernel start): setup=%llu mma_done=%llu epi_start=%llu epi_done=%llu exit=%llu\n",
                h[1] - h[0], h[2] - h[0], h[3] - h[0], h[4] - h[0], h[5] - h[0]);
        fprintf(stderr, "  sm clock: %llu cycles over %llu ns = %.0f MHz\n", h[5] - h[0], h[7] - h[6], 1e3 * (double)(h[5] - h[0]) / (double)(h[7] - h[6]));
        fprintf(stderr, "  tma_issue:");
        for (int i = 0; i < 24 && h[8 + i]; ++i) fprintf(stderr, " %llu", h[8 + i] - h[0]);
        fprintf(stderr, "\n  mma iteration 12: wait_full=%llu mma_x4=%llu commit=%llu", h[57] - h[56], h[58] - h[57], h[59] - h[58]);
        fprintf(stderr, "\n  mma_ready:");
        for (int i = 0; i < 24 && h[32 + i]; ++i) fprintf(stderr, " %llu", h[32 + i] - h[0]);
        fprintf(stderr, "\n");
    }
    BM_API_END
}

extern "C" int bm_debug_tc_op(bm_ctx* hctx, bm_tc_op_args* a) {
    BM_API_BEGIN
    Ctx* ctx = reinterpret_cast<Ctx*>(hctx);
    BM_REQUIRE(ctx && a && a->M > 0 && a->N > 0 && (a->n_pairs == 1 || a->n_pairs == 2), "bad argument");
    BM_CUDA(cudaSetDevice(ctx->device));
    const int M = a->M, N = a->N, n8 = round_up(N, 8);
    TcGemm g;
    g.M = M; g.N = N; g.n_pairs = a->n_pairs;
    // operands: bf16 bit patterns, copied into buffers whose leading dimension is a multiple of 8 (TMA)
    DevBuf<__nv_bfloat16> ops[4];
    std::vector<uint16_t> staged;
    for (int i = 0; i < 2 * g.n_pairs; ++i) {
        const int pr = i / 2; const bool isA = (i % 2) == 0;
        const uint16_t* src = isA ? a->A[pr] : a->B[pr];
        const bool t = (isA ? a->a_t[pr] : a->b_t[pr]) != 0;
        const int Kp = a->K[pr];
        BM_REQUIRE(src && Kp > 0, "bad operand");
        const int mn = isA ? M : N;
        const int rows = t ? Kp : mn, cols = t ? mn : Kp, ld = round_up(cols, 8);
        staged.assign((size_t)rows * ld, 0);
        for (int r = 0; r < rows; ++r) memcpy(&staged[(size_t)r * ld], src + (size_t)r * cols, (size_t)cols * 2);
        ops[i].ensure(staged.size());
        BM_CUDA(cudaMemcpyAsync(ops[i].p, staged.data(), staged.size() * 2, cudaMemcpyHostToDevice, ctx->stream));
        TcMat m; m.ptr = ops[i].p; m.rows = rows; m.cols = cols; m.ld = ld;
        if (isA) { g.A[pr] = m; g.a_t[pr] = t; g.neg[pr] = a->neg[pr] != 0; } else { g.B[pr] = m; g.b_t[pr] = t; }
        g.K[pr] = Kp;
    }
    g.splits = a->splits > 0 ? a->splits : 1;
    g.force_bn = a->force_bn; g.force_cluster = a->force_cluster;
    // epilogue vectors
    DevBuf<float> vec[3];
    const float* vsrc[3] = {a->bias, a->sigma, a->noise_sigma};
    for (int i = 0; i < 3; ++i) {
        if (!vsrc[i]) continue;
        vec[i].ensure((size_t)N);
        BM_CUDA(cudaMemcpyAsync(vec[i].p, vsrc[i], (size_t)N * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    }
    g.bias = vec[0].p; g.sigma = vec[1].p; g.noise_sigma = vec[2].p;
    g.acc_scale = a->acc_scale; g.bias_scale = a->bias_scale;
    g.act = a->act; g.sample = a->sample;
    g.rng = make_rng(a->seed, a->site, a->t, a->tick, a->row0);
    g.tick_off = a->tick_off;
    g.ais_kind = a->ais_kind; g.ais_a = a->ais_a; g.ais_b = a->ais_b; g.ais_next = a->ais_next; g.ais_lin = a->ais_lin;
    // outputs and log-weights: whole buffers in, whole buffers out
    DevBuf<double> logw;
    if (a->logw) {
        BM_REQUIRE(a->logw_len > M, "log-weights need a guard entry past M");
        logw.ensure((size_t)a->logw_len);
        BM_CUDA(cudaMemcpyAsync(logw.p, a->logw, (size_t)a->logw_len * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        g.ais_logw = logw.p;
    }
    DevBuf<__nv_bfloat16> mean, state;
    DevBuf<float> f32;
    const size_t mean_n = (size_t)a->mean_rows * a->mean_ld, state_n = (size_t)a->state_rows * a->state_ld;
    const size_t f32_n = (size_t)g.splits * a->f32_rows * a->f32_ld;
    if (a->mean_bf) {
        BM_REQUIRE(a->mean_rows > M && a->mean_ld > n8 && a->mean_ld % 8 == 0, "bf16 means need guard rows and columns");
        mean.ensure(mean_n);
        BM_CUDA(cudaMemcpyAsync(mean.p, a->mean_bf, mean_n * 2, cudaMemcpyHostToDevice, ctx->stream));
        g.out_mean_bf = mean.p; g.ld_mean_bf = a->mean_ld;
    }
    if (a->state_bf) {
        BM_REQUIRE(a->state_rows > M && a->state_ld > n8 && a->state_ld % 8 == 0, "bf16 states need guard rows and columns");
        state.ensure(state_n);
        BM_CUDA(cudaMemcpyAsync(state.p, a->state_bf, state_n * 2, cudaMemcpyHostToDevice, ctx->stream));
        g.out_state_bf = state.p; g.ld_state_bf = a->state_ld;
    }
    if (a->f32) {
        BM_REQUIRE(a->f32_rows > M && a->f32_ld > n8, "fp32 outputs need guard rows and columns");
        f32.ensure(f32_n);
        BM_CUDA(cudaMemcpyAsync(f32.p, a->f32, f32_n * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        g.out_f32 = f32.p; g.ld_f32 = a->f32_ld;
        g.split_stride = (size_t)a->f32_rows * a->f32_ld;
    }
    TcPlan plan;
    launch_tc_gemm(ctx, g, &plan);          // refuses an op it does not run before launching anything
    a->mode = plan.mode; a->bn = plan.bn; a->cluster = plan.cluster; a->units = plan.units; a->ctas = plan.ctas;
    if (a->mean_bf) BM_CUDA(cudaMemcpyAsync(a->mean_bf, mean.p, mean_n * 2, cudaMemcpyDeviceToHost, ctx->stream));
    if (a->state_bf) BM_CUDA(cudaMemcpyAsync(a->state_bf, state.p, state_n * 2, cudaMemcpyDeviceToHost, ctx->stream));
    if (a->f32) BM_CUDA(cudaMemcpyAsync(a->f32, f32.p, f32_n * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    if (a->logw) BM_CUDA(cudaMemcpyAsync(a->logw, logw.p, (size_t)a->logw_len * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    BM_CUDA(cudaStreamSynchronize(ctx->stream));
    BM_API_END
}
