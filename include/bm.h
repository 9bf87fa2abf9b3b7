/* bm.h -- C-ABI of libbm.so: the H100-native RBM/DBM engine.
 *
 * This is the drop-in boundary.  In the reference (yell/boltzmann-machines) the
 * operator boundary of the hot path is "a TensorFlow graph with named
 * collections executed by Session.run(fetches, feed_dict)"; each entry point
 * below names the reference interface it replaces (paths relative to
 * /root/reference/boltzmann_machines/).  Plain C types only: handles, pointers to
 * caller-owned host buffers (C-contiguous), sizes.  Every function returns
 * BM_OK (0) or a negative BM_E* code; bm_last_error() gives the thread-local
 * message.  Handles are not thread-safe; one context per GPU / per process rank.
 *
 * Random numbers: every stochastic call takes (seed, tick).  Element (row r,
 * column c) of draw site s at Gibbs index t uses Philox-4x32-10 with
 * key = (seed & 0xffffffff, seed >> 32) and counter = (c / 4, row0 + r,
 * s | t << 8, tick), word lane c % 4 -- see DESIGN.md "RNG layout".  Results do
 * not depend on tile shapes or on the number of GPUs.
 */
#ifndef BM_H_
#define BM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BM_OK            0
#define BM_EINVAL       -1   /* bad argument / shape / name                     */
#define BM_ECUDA        -2   /* CUDA runtime or driver error                    */
#define BM_ENOGPU       -3   /* no usable sm_90 device                          */
#define BM_ENCCL        -4   /* NCCL missing or failed                          */
#define BM_EUNSUPPORTED -5   /* configuration not implemented by the engine     */

typedef struct bm_ctx bm_ctx;   /* device + streams (+ NCCL communicator)          */
typedef struct bm_rbm bm_rbm;   /* one RBM: parameters, accumulators, workspaces    */
typedef struct bm_dbm bm_dbm;   /* one DBM: layers, variational params, particles   */

enum { BM_UNIT_BERNOULLI = 0, BM_UNIT_MULTINOMIAL = 1, BM_UNIT_GAUSSIAN = 2 };  /* layers.py:39-89 */
enum { BM_DTYPE_F32 = 0, BM_DTYPE_F64 = 1 };                                     /* base/mixin.py:14-25 */
enum { BM_COMPUTE_FP32 = 0,   /* CUDA-core FMA, storage dtype everywhere (parity anchor) */
       BM_COMPUTE_BF16 = 1 }; /* wgmma bf16 operands, fp32 accumulate (F32 models only)   */

/* metric selection bits / slots of the double[4] result (base_rbm.py:482-517) */
enum { BM_METRIC_L2_LOSS = 1, BM_METRIC_MSRE = 2, BM_METRIC_PLL = 4, BM_METRIC_FREE_ENERGY = 8 };
enum { BM_SLOT_L2_LOSS = 0, BM_SLOT_MSRE = 1, BM_SLOT_PLL = 2, BM_SLOT_FREE_ENERGY = 3 };

/* Static configuration of an RBM: what BaseRBM._make_constants/_make_vars bake
 * into the graph (rbm/base_rbm.py:244-327) plus the layer classes' parameters. */
typedef struct bm_rbm_cfg {
    int32_t n_visible, n_hidden;
    int32_t v_kind, h_kind;          /* BM_UNIT_*                                   */
    int32_t dtype;                   /* BM_DTYPE_* : storage type of every variable  */
    int32_t compute;                 /* BM_COMPUTE_*                                 */
    int32_t sample_v, sample_h;      /* sample_v_states / sample_h_states            */
    int32_t max_batch;               /* sizing hint (workspaces grow on demand)      */
    int32_t reserved0;
    double  l2;
    double  dropout_keep;            /* < 0: no dropout; else keep probability       */
    double  sparsity_target, sparsity_cost, sparsity_damping;
    double  propup_mult, propdown_mult;   /* 1 or 2 (dbm_first / dbm_last)           */
    double  v_n_samples, h_n_samples;     /* MultinomialLayer.n_samples              */
    const double* sigma;             /* [n_visible] for a gaussian visible layer, else NULL */
} bm_rbm_cfg;

/* ---- library / context -------------------------------------------------------- */
const char* bm_version(void);
const char* bm_last_error(void);
int  bm_device_count(int* n);                                   /* 0 devices is BM_OK with *n = 0 */
int  bm_ctx_create(int device, bm_ctx** out);                   /* replaces tf.Session creation, base/tf_model.py:26,33 */
void bm_ctx_destroy(bm_ctx* ctx);
int  bm_ctx_sync(bm_ctx* ctx);
/* device-side stopwatch on the context's compute stream (CUDA events) */
int  bm_ctx_timer_start(bm_ctx* ctx);
int  bm_ctx_timer_stop(bm_ctx* ctx, float* ms);
int  bm_ctx_flush_l2(bm_ctx* ctx);                              /* writes a >L2-sized scratch buffer */
int  bm_host_alloc(void** p, size_t bytes);                     /* pinned host memory for the feed path */
int  bm_host_free(void* p);
/* packing of a host training set for the feed path (what BaseRBM.fit does once per call; multi-threaded, one pass):
 * bm_host_pack_u8: *exact = 1 and out[i] = X[i] if every value is an integer in 0..255 (dtype BM_DTYPE_F32 / F64), else
 * *exact = 0;  bm_host_pack_bf16: out[i] = round-to-nearest-even bfloat16 of X[i].  Replace the numpy casts feed_dict relied on
 * (rbm/base_rbm.py:533-547). */
int  bm_host_pack_u8(const void* X, int32_t dtype, size_t n, uint8_t* out, int32_t* exact);
int  bm_host_pack_bf16(const float* X, size_t n, uint16_t* out);
int  bm_ctx_launch_count(bm_ctx* ctx, uint64_t* n);             /* kernels launched by this library on ctx */
/* per-launch CUDA-event timing of the tensor-core layer kernel (the roofline's dominant kernel):
 * enable, run, then read the accumulated algorithmic FLOPs, device milliseconds and launch count */
int  bm_ctx_profile_tc(bm_ctx* ctx, int enable);
int  bm_ctx_profile_read(bm_ctx* ctx, double* flops, double* ms, uint64_t* launches);

/* ---- multi-GPU: one process per GPU, chains sharded by rows, sum-allreduce of the
 *      gradient statistics (no counterpart in the reference: it is single-device) */
int  bm_comm_unique_id(void* id128);                            /* 128-byte NCCL unique id (rank 0) */
int  bm_ctx_comm_init(bm_ctx* ctx, const void* id128, int rank, int nranks);

/* ---- RBM ----------------------------------------------------------------------- */
int  bm_rbm_create(bm_ctx* ctx, const bm_rbm_cfg* cfg, bm_rbm** out);   /* BaseRBM._make_tf_model, base_rbm.py:527-531 */
void bm_rbm_destroy(bm_rbm* rbm);
/* variables by name: "W" [V,H], "vb" [V], "hb" [H], "dW", "dvb", "dhb", "q_means" [H]
 * (get_tf_params / Saver.restore, base/tf_model.py:183-202,22-28); element type = cfg.dtype */
int  bm_rbm_set_param(bm_rbm* rbm, const char* name, const void* host, size_t bytes);
int  bm_rbm_get_param(bm_rbm* rbm, const char* name, void* host, size_t bytes);
/* W <- N(0, stddev) with the stream of tf.random_normal(seed=op_seed) (base_rbm.py:277-279) */
int  bm_rbm_init_weights(bm_rbm* rbm, double stddev, uint64_t op_seed);
/* one mini-batch of CD-k: session.run(train_op, feed_dict) (base_rbm.py:415-479, 566).
 * X: host [rows, n_visible] of cfg.dtype.  On a context with an initialised
 * communicator X is this rank's shard: every rank passes the same `rows`, the
 * global batch is rows*nranks, this shard's first global row is rank*rows, and the
 * gradient statistics are sum-allreduced before the (identical) update on every rank.
 * metric_mask != 0: also fill metrics_out[4] (computed with the pre-update weights). */
int  bm_rbm_train_step(bm_rbm* rbm, const void* X, int32_t rows, double lr, double momentum,
                       int32_t n_gibbs_steps, uint64_t seed, uint32_t tick,
                       uint32_t metric_mask, double* metrics_out);
/* dataset-resident variant (SURVEY.md §8f.2): upload once, then step on row ranges */
int  bm_rbm_set_data(bm_rbm* rbm, const void* X, int64_t n_rows);
int  bm_rbm_train_step_at(bm_rbm* rbm, int64_t first_row, int32_t rows, double lr, double momentum,
                          int32_t n_gibbs_steps, uint64_t seed, uint32_t tick,
                          uint32_t metric_mask, double* metrics_out);
/* transform_op: chain-end E[h | v_k] (base_rbm.py:438-440, 687-700); H_out host [rows, n_hidden] */
/* BaseRBM._train_epoch (rbm/base_rbm.py:549-571): the whole mini-batch loop of one epoch over a HOST dataset
 * X[n_rows, n_visible].  Batch i = rows [i*batch, min(n_rows, (i+1)*batch)) runs exactly bm_rbm_train_step(..., tick0 + i);
 * its host->device copy is double-buffered on a copy stream and overlaps batch i-1's compute (full overlap needs X in
 * pinned memory, bm_host_alloc; pageable memory works but serialises).  Metrics selected by `mask` are computed for
 * the batches with (iter0 + i + 1) % metrics_every == 0 (train_metrics_every_iter, base_rbm.py:560-567; 0 = never),
 * read back asynchronously and returned in out[4*i .. 4*i+3] (other rows are zeroed); out may be NULL if mask is 0. */
int  bm_rbm_train_epoch(bm_rbm* rbm, const void* X, int64_t n_rows, int32_t batch, double lr, double momentum,
                        int32_t n_gibbs_steps, uint64_t seed, uint32_t tick0, uint32_t metric_mask,
                        int32_t metrics_every, int64_t iter0, double* out);
/* Same epoch for BYTE-VALUED data (SURVEY.md §8f.2, README.md:462 "optimize input pipeline"): X[n_rows, n_visible] holds
 * one unsigned byte per visible unit -- {0,1} for binarised MNIST -- and is widened exactly on the device, so every
 * result is bit-identical to bm_rbm_train_epoch on float(X) while the host->device copy is 4x (float32) / 8x (float64)
 * smaller.  BaseRBM.fit() takes this path when the training set is exactly representable (rbm/base_rbm.py:549-571
 * feeds the same values as float32 through feed_dict). */
int  bm_rbm_train_epoch_u8(bm_rbm* rbm, const uint8_t* X, int64_t n_rows, int32_t batch, double lr, double momentum,
                           int32_t n_gibbs_steps, uint64_t seed, uint32_t tick0, uint32_t metric_mask,
                           int32_t metrics_every, int64_t iter0, double* out);
/* Same epoch for REAL-VALUED data fed as bfloat16 bit patterns (grey levels: examples/rbm_mnist.py:209): the tensor-core
 * engine rounds its input to bf16 before the first GEMM anyway, so the result is bit-identical to bm_rbm_train_epoch on the
 * float32 rows while the host->device copy is half the size.  Only for float32 models on the bf16 engine without dropout or
 * sigma scaling (BM_EINVAL otherwise); bm_host_pack_bf16 makes X. */
int  bm_rbm_train_epoch_bf16(bm_rbm* rbm, const uint16_t* X, int64_t n_rows, int32_t batch, double lr, double momentum,
                             int32_t n_gibbs_steps, uint64_t seed, uint32_t tick0, uint32_t metric_mask,
                             int32_t metrics_every, int64_t iter0, double* out);
int  bm_rbm_transform(bm_rbm* rbm, const void* X, int32_t rows, int32_t n_gibbs_steps,
                      uint64_t seed, uint32_t tick, void* H_out);
/* msre / pll / l2_loss / free_energy_op on a batch without training (base_rbm.py:573-621) */
int  bm_rbm_metrics(bm_rbm* rbm, const void* X, int32_t rows, int32_t n_gibbs_steps,
                    uint64_t seed, uint32_t tick, uint32_t metric_mask, double* metrics_out);
/* debugging / parity hooks: activations of the last train_step/transform/metrics call.
 * name in {"X","h0_means","h0_states","v_means","v_states","h_means"}; element type float32
 * in BF16 compute mode (widened), cfg.dtype otherwise. */
int  bm_rbm_get_activation(bm_rbm* rbm, const char* name, void* host, size_t bytes);

/* ---- DBM -------------------------------------------------------------------------------------
 * Static configuration: what DBM._make_constants/_make_vars bake into the graph (dbm.py:233-383).
 * Per-layer arrays have n_layers entries (hidden layer 0 is adjacent to the visibles). */
typedef struct bm_dbm_cfg {
    int32_t n_layers, n_visible;
    const int32_t* n_hiddens;
    int32_t v_kind;                  /* BM_UNIT_*                                          */
    const int32_t* h_kinds;
    const double*  h_n_samples;      /* MultinomialLayer.n_samples per layer (nullable)    */
    int32_t dtype, compute;          /* BM_COMPUTE_BF16: tensor-core engine (F32 models, Bernoulli hidden layers) */
    int32_t n_particles, batch_size, max_mf_updates;
    int32_t sample_v;
    const int32_t* sample_h;
    double mf_tol, l2, max_norm, sparsity_damping;
    const double* sparsity_target;
    const double* sparsity_cost;
    const double* sigma;             /* [n_visible] for a gaussian visible layer, else NULL */
} bm_dbm_cfg;

int  bm_dbm_create(bm_ctx* ctx, const bm_dbm_cfg* cfg, bm_dbm** out);      /* DBM._make_tf_model, dbm.py:761-769 */
void bm_dbm_destroy(bm_dbm* dbm);
/* variables by TF-uniquified name (dbm.py:294-383, dbm_mnist.py:367-371): "vb", "W", "W_1", "hb", "hb_1",
 * "dvb", "dW"..., "dhb"..., "mu"... [batch_size,H_i], "q_means"..., "mu_means"..., particles "v" [n_particles,V],
 * "h", "h_1"... [n_particles,H_i] */
int  bm_dbm_set_param(bm_dbm* dbm, const char* name, const void* host, size_t bytes);
int  bm_dbm_get_param(bm_dbm* dbm, const char* name, void* host, size_t bytes);
/* persistent particles <- the layers' own random initialisers (dbm.py:362-383) */
int  bm_dbm_init_particles(bm_dbm* dbm, uint64_t seed);
/* session.run(train_op): mean-field E-step, PCD particle update, parameter update (dbm.py:515-622, 805).
 * want_metrics != 0: out2 = {msre, n_mf_updates} (dbm.py:798-803) */
int  bm_dbm_train_step(bm_dbm* dbm, const void* X, int32_t rows, double lr, double momentum, int32_t n_gibbs_steps,
                       uint64_t seed, uint32_t tick, int32_t want_metrics, double* out2);
/* validation msre / n_mf_updates; like the reference it also advances the persistent chains (dbm.py:523, 810-816) */
int  bm_dbm_val_metrics(bm_dbm* dbm, const void* X, int32_t rows, int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, double* out2);
int  bm_dbm_transform(bm_dbm* dbm, const void* X, int32_t rows, void* out);       /* mu of the last layer, dbm.py:526-528,859-872 */
int  bm_dbm_reconstruct(bm_dbm* dbm, const void* X, int32_t rows, void* out);     /* dbm.py:626-632, 874-885 */
int  bm_dbm_log_proba(bm_dbm* dbm, const void* X, int32_t rows, double* out);     /* variational bound + log Z, dbm.py:738-759 */
int  bm_dbm_sample_v(bm_dbm* dbm, int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, void* out);  /* dbm.py:641-648 */
/* AIS estimates of log Z, one per run (dbm.py:650-736, 899-939).  The runs are independent chains and run r always draws
 * from row r of the AIS sites: on a context with a communicator (bm_ctx_comm_init) the n_runs runs are sharded over the
 * ranks and gathered with one sum-allreduce of n_runs doubles -- every rank calls with the same arguments and receives all
 * n_runs values, identical to a single-GPU call (SURVEY 8e). */
int  bm_dbm_ais(bm_dbm* dbm, int32_t n_runs, int32_t n_betas, int32_t n_gibbs_steps, uint64_t seed, double* logZ);
/* runs [first_run, first_run + n_runs) of the same ladder, no communication: for callers that shard or chunk the runs
 * themselves (one process driving several GPUs; more runs than fit in memory at once) */
int  bm_dbm_ais_rows(bm_dbm* dbm, int32_t n_runs, int32_t n_betas, int32_t n_gibbs_steps, uint64_t seed, uint32_t first_run,
                     double* logZ);

/* ---- test hook: the raw tensor-core GEMM (no counterpart in the reference) -----------------
 * C[M,N] (fp32) = A * B^T (+/- A2 * B2^T), operands given as host fp32 and rounded to bf16.
 * a_t == 0: A is [M,K] row-major, else [K,M];  b_t == 0: B is [N,K] row-major, else [K,N]
 * (the second pair uses the same orientations).  splits > 1 exercises the split-K path;
 * force_bn / force_cluster > 0 override the tile-width / TMA-multicast-cluster heuristic. */
int  bm_debug_tc_gemm(bm_ctx* ctx, int32_t M, int32_t N, int32_t K, const float* A, int32_t a_t,
                      const float* B, int32_t b_t, int32_t K2, const float* A2, const float* B2,
                      int32_t neg2, int32_t splits, int32_t force_bn, int32_t force_cluster, float* C);

/* ---- test hook: ONE fused tensor-core op, every output returned whole --------------------
 * C[M,N] = sum_p (+/-) A_p * B_p^T over n_pairs (1 or 2) operand pairs given as bf16 bit patterns:
 * A_p is [M,K_p] row-major (a_t[p]: [K_p,M]), B_p is [N,K_p] (b_t[p]: [K_p,N]); then the op's epilogue
 *   pre = acc_scale * C * sigma[n] + bias_scale * bias[n],  mean = act(pre),  state = sample(mean)
 * with the draws of element (r, c) taken from Philox (seed, site | t << 8, tick + tick_off, row0 + r) as in the engine.
 * ais_kind 1 / 2 select the AIS epilogues (see csrc/bm_tc_desc.h); logw [logw_len] is added to and returned.
 * Outputs are optional (NULL: not written) and given WHOLE, as the caller filled them: each buffer is copied to the device,
 * the op writes its [M, N] window (split s of a split-K op: f32 + s * f32_rows * f32_ld), and the whole buffer comes back,
 * so that a test sees anything written outside the window.  Each needs a guard row (rows > M) and guard columns
 * (ld > round_up(N, 8)); bf16 leading dimensions are multiples of 8, the fp32 one may be odd.
 * On return mode, bn, cluster, units and ctas describe the launch: the epilogue mode the op ran with, the tile width, the
 * row grouping (1: a CTA per 128-row block, 2: CTA pairs per 256-row group), the number of units and the CTAs of the grid.
 * An op the engine does not run is refused with BM_EINVAL before anything is launched. */
typedef struct bm_tc_op_args {
    int32_t M, N, n_pairs;
    int32_t K[2], a_t[2], b_t[2], neg[2];
    const uint16_t* A[2];
    const uint16_t* B[2];
    int32_t splits, force_bn, force_cluster;
    float acc_scale, bias_scale;
    const float* bias;                     /* [N] or NULL (host) */
    const float* sigma;                    /* [N] or NULL */
    const float* noise_sigma;              /* [N] or NULL */
    int32_t act, sample;                   /* 0 linear, 1 sigmoid, 2 softplus;  0 none, 1 Bernoulli, 2 Gaussian */
    uint64_t seed;
    uint32_t site, t, tick, row0, tick_off;
    int32_t ais_kind;
    float ais_a, ais_b, ais_next, ais_lin;
    double* logw;          int32_t logw_len;
    uint16_t* mean_bf;     int32_t mean_rows, mean_ld;
    uint16_t* state_bf;    int32_t state_rows, state_ld;
    float* f32;            int32_t f32_rows, f32_ld;
    int32_t mode, bn, cluster, units, ctas;          /* out: what was launched */
} bm_tc_op_args;
int  bm_debug_tc_op(bm_ctx* ctx, bm_tc_op_args* args);

/* ---- test hook: how the last tensor-core program of an RBM was planned -----------------------
 * One record per op of the last chain the engine ran (train_step, train_step_at, train_epoch's last batch, transform,
 * metrics), in program order across all the launches a long chain is cut into.  Read-only: decoded from the descriptors
 * the launch uploaded.  *n_ops receives the number of ops; at most `cap` records are written.  BM_EINVAL for an engine
 * that runs no tensor-core program. */
typedef struct bm_tc_op_plan {
    int32_t launch;                        /* 0, 1, ...: which launch of the chain ran this op */
    int32_t mode, bn;                      /* epilogue mode (as bm_tc_op_args), tile width */
    int32_t m_groups, n_tiles, splits;     /* 256-row groups, column tiles, K splits: units = their product */
    int32_t pair_begin, pair_count;        /* the CTA pairs that run the op's units */
    int32_t follows_granules;              /* 1: waits for its producer's 64-column granules one by one */
} bm_tc_op_plan;
int  bm_rbm_debug_tc_plan(bm_rbm* rbm, bm_tc_op_plan* out, int32_t cap, int32_t* n_ops);

#ifdef __cplusplus
}
#endif
#endif  /* BM_H_ */
