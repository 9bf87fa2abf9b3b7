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

/* ---- training groups: many RBMs of one shape trained side by side (no counterpart in the reference) ----------------
 * A group drives the training steps of n ordinary bm_rbm handles.  Step i of a group epoch runs, for every member m, exactly
 * what bm_rbm_train_epoch step i of that member runs: the same ops, tile widths, splits and K orders, the same draws from
 * the member's own seed and tick, the same update -- so every variable and metric is bit-identical to the member's own epoch.
 * The members' chains share the program launches of a step (each member on its own CTA pairs; a step whose ops do not fit
 * one launch is cut between members) and one launch updates all of them.  The members stay ordinary handles: get_param,
 * set_param, metrics, transform and bm_rbm_debug_tc_plan work on them as before (the plan then shows the grouped launch).
 * Members must share the context, n_visible, n_hidden, the unit kinds and max_batch (BM_EINVAL naming the field); seeds,
 * sigma, l2, the sparsity settings, dbm_first / dbm_last and the sampling flags may differ.  BM_EUNSUPPORTED, with the
 * option named: multinomial layers, the fp32 / fp64 engines (only BM_COMPUTE_BF16 members), dropout and a context with a
 * communicator. */
typedef struct bm_rbm_group bm_rbm_group;
int  bm_rbm_group_create(bm_ctx* ctx, bm_rbm* const* members, int32_t n, bm_rbm_group** out);
void bm_rbm_group_destroy(bm_rbm_group* group);
/* One epoch of every member over X[n][n_rows][n_visible] (member m trains on X[m]; cfg.dtype, bytes or bfloat16 bit
 * patterns as in bm_rbm_train_epoch / _u8 / _bf16).  Per member m: lr[m], momentum[m], seeds[m], tick0[m], metric_mask[m],
 * metrics_every[m] and iter0[m] mean what they mean for bm_rbm_train_epoch; n_gibbs_steps is shared and at most 43 (a longer
 * chain needs several launches per member).  out[(m * n_batches + i) * 4 ..] receives member m's metrics of batch i (zeros
 * on batches that do not report); out may be NULL when every mask is 0.  Uploads are double-buffered on the copy stream:
 * one host->device copy and one conversion per step for all members. */
int  bm_rbm_group_train_epoch(bm_rbm_group* group, const void* X, int64_t n_rows, int32_t batch, const double* lr,
                              const double* momentum, int32_t n_gibbs_steps, const uint64_t* seeds, const uint32_t* tick0,
                              const uint32_t* metric_mask, const int32_t* metrics_every, const int64_t* iter0, double* out);
int  bm_rbm_group_train_epoch_u8(bm_rbm_group* group, const uint8_t* X, int64_t n_rows, int32_t batch, const double* lr,
                                 const double* momentum, int32_t n_gibbs_steps, const uint64_t* seeds, const uint32_t* tick0,
                                 const uint32_t* metric_mask, const int32_t* metrics_every, const int64_t* iter0, double* out);
int  bm_rbm_group_train_epoch_bf16(bm_rbm_group* group, const uint16_t* X, int64_t n_rows, int32_t batch, const double* lr,
                                   const double* momentum, int32_t n_gibbs_steps, const uint64_t* seeds, const uint32_t* tick0,
                                   const uint32_t* metric_mask, const int32_t* metrics_every, const int64_t* iter0, double* out);

/* ---- DBM -------------------------------------------------------------------------------------
 * Static configuration: what DBM._make_constants/_make_vars bake into the graph (dbm.py:233-383).
 * Per-layer arrays have n_layers entries (hidden layer 0 is adjacent to the visibles). */
typedef struct bm_dbm_cfg {
    int32_t n_layers, n_visible;
    const int32_t* n_hiddens;
    int32_t v_kind;                  /* BM_UNIT_*                                          */
    const int32_t* h_kinds;
    const double*  h_n_samples;      /* MultinomialLayer.n_samples per layer (nullable)    */
    int32_t dtype, compute;          /* BM_COMPUTE_BF16: tensor-core engine (F32 models, Bernoulli or Gaussian visibles,
                                        Bernoulli and multinomial hidden layers); other models run on the FP32 engine */
    int32_t n_particles, batch_size, max_mf_updates;
    int32_t sample_v;
    const int32_t* sample_h;
    double mf_tol, l2, max_norm, sparsity_damping;
    const double* sparsity_target;
    const double* sparsity_cost;
    const double* sigma;             /* [n_visible] for a gaussian visible layer, else NULL */
    /* Parallel tempering of the persistent chains (Desjardins et al., AISTATS 2010).  0 / NULL: off.  Otherwise n_temps
     * inverse temperatures betas[0] = 1 > betas[1] > ... > betas[n_temps-1] >= 0; slot m holds n_particles chains swept at
     * betas[m] (conditionals sigmoid(beta (x + b))), and every committed particle update ends with one round of swaps
     * between neighbouring slots (DESIGN.md §5.4).  Slot 0 is the chain without tempering: gradients, column sums,
     * sample_v and the names "v" / "h..." read it.  BM_EUNSUPPORTED: the fp32 / fp64 engines, gaussian visibles, multinomial
     * hidden layers, a context with a communicator; BM_EINVAL: a malformed ladder, sample_v == 0 or any sample_h == 0. */
    int32_t n_temps;
    const double* betas;
    /* Classification DBM (DESIGN.md §5.7; no counterpart in the reference).  0: off.  n_classes = C >= 2 adds a one-of-C label
     * y above the top hidden layer h_L: energy = the DBM's - e_y'U h_L - yb'e_y with U [C, H_L], yb [C].  Inside the engine y
     * is hidden layer L + 1, multinomial with n_samples 1 and weight W_{L+1} = U^T.  Labels take values in {-1, 0, .., C-1};
     * -1 marks an unlabelled row.  Training (bm_dbm_train_step_labeled): the mean-field E-step holds a labelled row's label
     * at its one-hot e_t (never updated) and updates an unlabelled row's like any multinomial layer; the particles sweep v,
     * h_1 .. h_L, y, drawing y (one categorical draw at site 16 + L); U takes l2, momentum and max-norm like any W, yb the
     * plain momentum update from sum q(y) / rows - sum y / n_particles, with no sparsity term (sparsity_target / _cost keep
     * their n_layers entries).  A batch labelled -1 throughout equals the plain DBM with a multinomial top layer of C units,
     * n_samples 1, sampled, sparsity cost 0, bit for bit where that DBM runs (C > n_layers).  Queries run with y free:
     * bm_dbm_predict_proba gives softmax(yb + mu_L U^T) from the E-step's final mu_L (a mean-field approximation of
     * p(y|x)), bm_dbm_transform mu_L; bm_dbm_log_proba and AIS are refused (BM_EUNSUPPORTED).  Variables: the DBM's names for
     * layers 0..L-1, plus "U", "dU" [C, H_L], "yb", "dyb" [C], the label particles "y" [n_particles, C] and the E-step's label
     * slot "mu_y" [batch_size, C].  BM_EINVAL: n_classes < 0 or == 1, more than 7 hidden layers; BM_EUNSUPPORTED (the option
     * named): float64, BM_COMPUTE_FP32, n_temps > 1, a context with a communicator. */
    int32_t n_classes;
    /* Centering (Montavon & Mueller 2012; DESIGN.md §5.8; not in the reference).  0: off.  centering != 0 trains the
     * centered DBM E_c(x) = -sum_i (x_i - o_i)'W_i (x_{i+1} - o_{i+1}) - sum_j (x_j - o_j)'a_j with data-mean offsets o_j.
     * The engine keeps storing the plain parameters (W, b) with b_j = a_j - W_{j-1}'o_{j-1} - W_j o_{j+1}, so every
     * query, particle sweep, swap and AIS reads what it reads without centering.  A training step takes the centered
     * gradient G_i - o_i s_{i+1}' - s_i o_{i+1}' + (rows / batch_size - 1) o_i o_{i+1}' (s_j = sum data_j / batch_size -
     * sum particles_j / n_particles), applies l2, sparsity, momentum and max-norm to it and to the a_j where they apply to
     * G and b, re-derives b from the new W, then moves o_j <- (1 - offset_rate) o_j + offset_rate mean_rows(data_j).  The
     * first step of a model sets o_j to the batch's data means.  Variables: "v_offset" [V], "h_offset", "h_offset_1"...
     * [H_i] and "offsets_set" [1] (0 until the first step; 1 afterwards).  BM_EINVAL: offset_rate outside [0, 1];
     * BM_EUNSUPPORTED (the option named): float64, BM_COMPUTE_FP32 or any model DbmTC does not run, n_classes > 0, a
     * context with a communicator. */
    int32_t centering;
    double offset_rate;
} bm_dbm_cfg;

int  bm_dbm_create(bm_ctx* ctx, const bm_dbm_cfg* cfg, bm_dbm** out);      /* DBM._make_tf_model, dbm.py:761-769 */
void bm_dbm_destroy(bm_dbm* dbm);
/* variables by TF-uniquified name (dbm.py:294-383, dbm_mnist.py:367-371): "vb", "W", "W_1", "hb", "hb_1",
 * "dvb", "dW"..., "dhb"..., "mu"... [batch_size,H_i], "q_means"..., "mu_means"..., particles "v" [n_particles,V],
 * "h", "h_1"... [n_particles,H_i]; with parallel tempering also the tempered slots 1..n_temps-1 "v_pt"
 * [n_temps-1,n_particles,V], "h_pt", "h_pt_1"... [n_temps-1,n_particles,H_i] */
int  bm_dbm_set_param(bm_dbm* dbm, const char* name, const void* host, size_t bytes);
int  bm_dbm_get_param(bm_dbm* dbm, const char* name, void* host, size_t bytes);
/* persistent particles <- the layers' own random initialisers (dbm.py:362-383) */
int  bm_dbm_init_particles(bm_dbm* dbm, uint64_t seed);
/* session.run(train_op): mean-field E-step, PCD particle update, parameter update (dbm.py:515-622, 805).
 * want_metrics != 0: out2 = {msre, n_mf_updates} (dbm.py:798-803) */
int  bm_dbm_train_step(bm_dbm* dbm, const void* X, int32_t rows, double lr, double momentum, int32_t n_gibbs_steps,
                       uint64_t seed, uint32_t tick, int32_t want_metrics, double* out2);
/* classification DBM (bm_dbm_cfg.n_classes >= 2): one training step with labels [rows] in [-1, n_classes) (BM_EINVAL before
 * any launch otherwise; -1: unlabelled row); out2 as bm_dbm_train_step.  bm_dbm_train_step on a classification DBM is this
 * call with every label -1.  BM_EINVAL on a DBM without a label layer. */
int  bm_dbm_train_step_labeled(bm_dbm* dbm, const void* X, const int32_t* labels, int32_t rows, double lr, double momentum,
                               int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, int32_t want_metrics, double* out2);
/* classification DBM: q(y|x) = softmax(yb + mu_L U^T) [rows, n_classes] (float32) after the E-step with y free, in chunks
 * of batch_size rows; changes "mu..." like bm_dbm_transform.  BM_EINVAL on a DBM without a label layer. */
int  bm_dbm_predict_proba(bm_dbm* dbm, const void* X, int32_t rows, float* out);
/* validation msre / n_mf_updates; like the reference it also advances the persistent chains (dbm.py:523, 810-816) */
int  bm_dbm_val_metrics(bm_dbm* dbm, const void* X, int32_t rows, int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, double* out2);
int  bm_dbm_transform(bm_dbm* dbm, const void* X, int32_t rows, void* out);       /* mu of the last layer, dbm.py:526-528,859-872 */
int  bm_dbm_reconstruct(bm_dbm* dbm, const void* X, int32_t rows, void* out);     /* dbm.py:626-632, 874-885 */
/* The variational bound without -log Z, per row (dbm.py:738-759).  Two hidden layers: either engine.  Any other number of layers:
 * the tensor-core engine with binary layers only (DESIGN.md §5.4c) -- BM_EUNSUPPORTED for Gaussian visibles or a multinomial
 * layer; the CUDA-core engine (float64 models, BM_COMPUTE_FP32) keeps its BM_EINVAL refusal. */
int  bm_dbm_log_proba(bm_dbm* dbm, const void* X, int32_t rows, double* out);
int  bm_dbm_sample_v(bm_dbm* dbm, int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, void* out);  /* dbm.py:641-648 */
/* AIS estimates of log Z, one per run (dbm.py:650-736, 899-939).  The runs are independent chains and run r always draws
 * from row r of the AIS sites: on a context with a communicator (bm_ctx_comm_init) the n_runs runs are sharded over the
 * ranks and gathered with one sum-allreduce of n_runs doubles -- every rank calls with the same arguments and receives all
 * n_runs values, identical to a single-GPU call (SURVEY 8e).  Binary DBMs with two hidden layers run on either engine.  Any
 * other number of layers runs on the tensor-core engine (DESIGN.md §5.4c: chains over h_1, h_3, ..., with v and the even layers
 * summed out); there BM_EUNSUPPORTED refuses Gaussian visibles, multinomial layers and an odd layer h_1, h_3, ... that is not
 * sampled, before any launch.  The CUDA-core engine (float64 models, BM_COMPUTE_FP32) refuses any depth but 2 (BM_EINVAL),
 * and a classification DBM refuses AIS at every depth (BM_EUNSUPPORTED). */
int  bm_dbm_ais(bm_dbm* dbm, int32_t n_runs, int32_t n_betas, int32_t n_gibbs_steps, uint64_t seed, double* logZ);
/* runs [first_run, first_run + n_runs) of the same ladder, no communication: for callers that shard or chunk the runs
 * themselves (one process driving several GPUs; more runs than fit in memory at once) */
int  bm_dbm_ais_rows(bm_dbm* dbm, int32_t n_runs, int32_t n_betas, int32_t n_gibbs_steps, uint64_t seed, uint32_t first_run,
                     double* logZ);
/* AIS from a base-rate model (DESIGN.md §5.4d; Salakhutdinov & Hinton 2009): the ladder starts from the factorial model
 * p_A(x) ∝ exp(sum_j a_j.x_j) over every unit layer instead of the uniform one, along p_beta ∝ p_A^(1-beta) p^beta (weights
 * scaled by beta, layer j's bias beta b_j + (1 - beta) a_j), and each run's estimate includes
 * log Z_A = sum_j sum_n softplus(a_{j,n}) (float64).  base is NULL or n_hiddens + 1 host pointers (v, h_1 .. h_L), each NULL
 * (a_j = 0) or [width of layer j] floats; a typical base sets a_v to the log-odds of the training data's pixel means and leaves
 * the hidden layers NULL.  NULL or all-NULL is bm_dbm_ais / bm_dbm_ais_rows exactly (those two call these).  With any base the
 * ladder runs over the odd layers at every depth, 2 included, and the run keys are those of bm_dbm_ais, so sharded, sliced and
 * single calls agree.  Refused before any launch: BM_EINVAL for a non-finite base entry; BM_EUNSUPPORTED on the CUDA-core engine
 * (float64 models, BM_COMPUTE_FP32), for Gaussian visibles or multinomial layers, an odd layer h_1, h_3, ... that is not
 * sampled, and for classification DBMs. */
int  bm_dbm_ais_base(bm_dbm* dbm, int32_t n_runs, int32_t n_betas, int32_t n_gibbs_steps, uint64_t seed, const float* const* base,
                     double* logZ);
int  bm_dbm_ais_base_rows(bm_dbm* dbm, int32_t n_runs, int32_t n_betas, int32_t n_gibbs_steps, uint64_t seed, uint32_t first_run,
                          const float* const* base, double* logZ);
/* Exact log Z and log p*(v) of a binary DBM whose odd layers h_1, h_3, ... hold n_odd <= 32 units (DESIGN.md §5.4f): every
 * state x of the odd layers is enumerated on the tensor cores, v and the even layers summed out analytically, for the model
 * as stored (float32 W and biases, not the bf16 shadow the chains read).  X [rows, n_visible] float32 (used as given, so grey
 * rows are allowed); log_p_star [rows] receives log p*(v) = log sum_h exp(-E(v, h)) (without -log Z) and log_Z, if not NULL,
 * log Z -- both from one pass over the states.  X = NULL, rows = 0 computes log Z only.  Every rank of a context with a
 * communicator computes the whole sum and gets the same result.  Refused before any launch: BM_EINVAL for rows < 0, a missing
 * X or log_p_star with rows > 0, X with rows = 0, nothing to compute, or a non-finite entry of X; BM_EUNSUPPORTED (the reason
 * named) for the CUDA-core engine (float64 models, BM_COMPUTE_FP32), Gaussian visibles or multinomial layers, classification
 * DBMs and n_odd > 32. */
int  bm_dbm_exact(bm_dbm* dbm, const void* X, int32_t rows, double* log_p_star, double* log_Z);
/* DESIGN.md §5.4g: AIS over the hidden layers with v clamped to each row of X [rows, n_visible] float32.
 * log_w [rows * n_runs] receives each run's estimate of log p*(v_r) (log Z_0 and b_v.v included).
 * An estimate of the true log p*(v) = log sum_h exp(-E(v, h)) of a binary DBM of any depth, where log_proba gives a lower
 * bound: Salakhutdinov & Hinton (2009) run this ladder on each test vector; the reference has nothing like it.  With v fixed
 * the odd layers h_1, h_3, ... are summed out analytically and the even layers h_2, h_4, ... are the chains' state; every
 * layer drawn is sampled, whatever sample_h says.  Temperatures, sweeps and increments are those of bm_dbm_ais, on the bf16
 * shadow of W; log Z_0 = (sum_i H_i) log 2 and b_v.v are added in float64.  X is used as given: grey rows enter the X W_0
 * product as bf16(X).  Entry c = r * n_runs + k is run k of row r; it draws from Philox row (row0 + r) * n_runs + k, so a
 * row's runs depend only on its global index row0 + r, never on how the caller slices the rows.  At one hidden layer there
 * is nothing to anneal: every run is bm_dbm_log_proba's value, exact there, and the call writes the E-step's means as that
 * call does; otherwise it reads W and the biases only.  No communication: each rank computes the call it was given.
 * Refused before any launch: BM_EUNSUPPORTED (the reason named) on the CUDA-core engine (float64 models, BM_COMPUTE_FP32),
 * for Gaussian visibles or multinomial layers and for classification DBMs; BM_EINVAL for a NULL X or log_w, rows < 1,
 * n_runs < 1, n_betas < 2, n_gibbs_steps < 1, a non-finite entry of X, or (row0 + rows) * n_runs >= 2^32. */
int  bm_dbm_ais_clamped(bm_dbm* dbm, const void* X, int32_t rows, uint32_t row0, int32_t n_runs, int32_t n_betas,
                        int32_t n_gibbs_steps, uint64_t seed, double* log_w);
/* test hook: 2^log2_states states per launch of bm_dbm_exact's enumeration (1..30; 0 restores the default 2^22), so that
 * small models span several launches.  The result does not depend on it beyond float64 rounding. */
int  bm_dbm_debug_exact_chunk(bm_dbm* dbm, int32_t log2_states);
/* parallel tempering: swaps accepted / proposed between slots m and m+1 since create, n_temps-1 entries each (BM_EINVAL
 * without tempering) */
int  bm_dbm_pt_counts(bm_dbm* dbm, int64_t* accepted, int64_t* proposed);
/* Conditional sampling with clamped Gibbs chains (DESIGN.md §5.9; not in the reference): fill in the missing visible units of
 * X [rows, n_visible] (model dtype), mask [rows, n_visible] bytes (1: observed, clamped to X; 0: missing, X ignored).  Per row:
 * v0 = X where observed and act(b) (the visible mean with nothing above) elsewhere; h0 from the mean-field E-step's
 * approximate-inference pass on v0; then n_gibbs_steps >= 1 particle sweeps (h_1 .. h_L bottom-up, then v), drawing at sites
 * 16 + i / 11, sweep index t = 1.., the call's seed and tick and row row0 + r, with v reset to X where observed after every
 * visible update.  out [rows, n_visible] = the visible means p(v | h_1) of the last sweep, X where observed.  A row's result
 * depends on its X, mask, label and global index row0 + r only, so a caller may cut a call into pieces.  Classification DBM:
 * labels [rows] in [-1, n_classes) (NULL: all -1); a row labelled t >= 0 holds its label at e_t throughout (the class-
 * conditional chain), -1 leaves it free.  Reads W and b only: no variable, accumulator, particle, offset or counter changes.
 * BM_EINVAL before any launch: a null pointer, rows outside 1..batch_size, n_gibbs_steps < 1, a mask byte other than 0 / 1,
 * a label outside [-1, n_classes), labels on a DBM without a label layer. */
int  bm_dbm_fill(bm_dbm* dbm, const void* X, const uint8_t* mask, const int32_t* labels, int32_t rows, uint32_t row0,
                 int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, void* out);
/* test hook: one chain state of the last bm_dbm_fill, [rows, n] row-major without padding (rows: that call's).  "v", "h",
 * "h_1", ... (a classification DBM's label layer: "y"): the last sweep; the same names + "_prev": the sweep before it (the start
 * after one sweep); "mean": the visible means before the observed units are put back.  Elements: bf16 bit patterns (uint16) on
 * the tensor-core engine, the model dtype on the CUDA-core engine.  Device-to-host copies only.  BM_EINVAL for an unknown name,
 * a wrong size, or before the first fill. */
int  bm_dbm_debug_last_fill(bm_dbm* dbm, const char* name, void* host, size_t bytes);
/* test hook: one sweep of the uncommitted second half of the last bm_dbm_sample_v, [n_particles, n] row-major without padding
 * (slot 0's particles on a tempered DBM).  "v", "h", "h_1", ...: the visible / hidden means of its last sweep (k); the same
 * names + "_prev": of sweep k - 1 (k >= 2; sweep 0 is the committed particles, read with bm_dbm_get_param).  Elements: bf16 bit
 * patterns (uint16) on the tensor-core engine, the model dtype on the CUDA-core engine.  Reads the scratch the sweeps ran on;
 * a device-to-host copy only, no launch.  BM_EINVAL for an unknown name, a wrong size, after k = 0, or once any particle update
 * has run since. */
int  bm_dbm_debug_last_sample_v(bm_dbm* dbm, const char* name, void* host, size_t bytes);

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
    const float* noise_sigma;              /* [N] or NULL; an AIS op (ais_kind != 0) reads it as its base bias a (DESIGN.md §5.4d) */
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

/* ---- test hook: the multinomial conditional of the tensor-core DBM engine ---------------------
 * From host fp32 pre-activations pre [rows, cols] (x + b of the layer), the engine's fused row kernel writes
 * n_samples * softmax(row) -- or, n_draws > 0, the counts of n_draws categorical draws from Philox (seed, site | t << 8,
 * tick, row r) -- as bf16 bit patterns to out_bf and in fp32 to out_f32 (both [rows, cols]); from the same input the
 * CUDA-core engine's two kernels write their fp32 means to ref_means and their counts to ref_counts (n_draws > 0). */
int  bm_debug_dbm_multinomial_rows(bm_ctx* ctx, const float* pre, int32_t rows, int32_t cols, double n_samples, int32_t n_draws,
                                   uint64_t seed, uint32_t site, uint32_t t, uint32_t tick, uint16_t* out_bf, float* out_f32,
                                   float* ref_means, float* ref_counts);

/* ---- Classification RBM (Larochelle & Bengio, ICML 2008; no counterpart in the reference) -------------
 * Visible x [n_visible] and a one-of-n_classes label beside it, both connected to h [n_hidden]:
 * E = -x'W h - e_y'U h - vb'x - hb'h - yb'e_y.  p(y|x) is exact; training takes the hybrid gradient
 * grad = d/dtheta mean log p(t|x) + alpha * (CD-k on the joint p(x, y)) - l2 * (W, U), then the momentum update
 * d <- lr (momentum d + grad), theta += d.  Runs on the tensor cores only: float32 models, BM_COMPUTE_BF16.
 * BM_EUNSUPPORTED (with the option named) for float64, BM_COMPUTE_FP32, dropout, a sparsity cost, dbm_first /
 * dbm_last and a context with a communicator; BM_EINVAL unless 2 <= n_classes <= 64. */
typedef struct bm_crbm bm_crbm;
typedef struct bm_crbm_cfg {
    int32_t n_visible, n_hidden, n_classes;
    int32_t dtype, compute;          /* BM_DTYPE_F32 / BM_COMPUTE_BF16: anything else is refused */
    int32_t sample_v, sample_h;      /* sample_v_states (x and label draws in the chain) / sample_h_states */
    int32_t max_batch;               /* rows of the largest batch (workspaces are sized once) */
    double  alpha;                   /* weight of the generative gradient; 0: purely discriminative, no chain */
    double  l2;
    double  dropout_keep;            /* < 0 (none); anything else is refused */
    double  sparsity_cost;           /* 0; anything else is refused */
    int32_t dbm_first, dbm_last;     /* 0; anything else is refused */
    double  beta;                    /* weight of beta * CD-k of log p(x) for rows labelled -1 (semi-supervised, Larochelle
                                        et al., JMLR 2012); 0 (the default) refuses -1; negative or non-finite: BM_EINVAL */
} bm_crbm_cfg;
int  bm_crbm_create(bm_ctx* ctx, const bm_crbm_cfg* cfg, bm_crbm** out);
void bm_crbm_destroy(bm_crbm* crbm);
/* variables "W" [V,H], "U" [C,H], "vb" [V], "hb" [H], "yb" [C] and their momenta "dW", "dU", "dvb", "dhb", "dyb" (float32) */
int  bm_crbm_set_param(bm_crbm* crbm, const char* name, const void* host, size_t bytes);
int  bm_crbm_get_param(bm_crbm* crbm, const char* name, void* host, size_t bytes);
/* W <- N(0, stddev) from tf.random_normal's stream of op_seed_w, U [C,H] likewise from op_seed_u */
int  bm_crbm_init_weights(bm_crbm* crbm, double stddev, uint64_t op_seed_w, uint64_t op_seed_u);
/* one hybrid step on X [rows, n_visible] (float32) with labels [rows] in [0, n_classes) (BM_EINVAL before any launch
 * otherwise); 1 <= rows <= max_batch.  With beta > 0 a label of -1 marks an unlabelled row: it adds beta * CD-k of log p(x)
 * (exact positive phase; the chain starts from a label drawn from p(y|x)) and the chain runs even at alpha = 0; with
 * beta = 0, -1 is refused like any label outside [0, n_classes).  A batch without -1 computes what it computes at beta = 0.
 * want_metrics != 0: out2 = {mean -log p(t|x), accuracy} over the labelled rows under the pre-update weights (NaN, NaN
 * when the batch has none) */
int  bm_crbm_train_step(bm_crbm* crbm, const void* X, const int32_t* labels, int32_t rows, double lr, double momentum,
                        int32_t n_gibbs_steps, uint64_t seed, uint32_t tick, int32_t want_metrics, double* out2);
/* test hook: copies one buffer of the last bm_crbm_train_step to the host, [rows, width] row-major without padding, where rows
 * is that step's batch.  Device-to-host copies only: it launches nothing and changes no state.  Names and widths:
 *   "A"   float32 [rows, n_hidden]    X W (bf16 operands, fp32 accumulation, no bias)
 *   "P"   float32 [rows, n_classes]   p(y|x)
 *   "y0"  int32   [rows]              the chain's start label (meaningful for rows labelled -1 only)
 *   "G"   uint16  [rows, n_hidden]    bf16 bits of (1 + alpha) S_t - S^ (beta S^ on unlabelled rows), the dW operand
 * and, when the step's chain ran (alpha > 0 or an unlabelled row), bf16 bits of:
 *   "h0"  [rows, n_hidden]            the chain's start (only after a step with n_gibbs_steps = 1)
 *   "x_k" [rows, n_visible], "y_k" [rows, n_classes], "h_k" [rows, n_hidden]   the last sweep's operands
 *   "aH"  [rows, n_hidden]            w_r h_k (w_r = alpha, or beta on unlabelled rows), the negated dW operand
 * BM_EINVAL for an unknown name, a size other than rows * width * element size, a chain buffer the step did not write, or
 * when no step ran since the engine was created or last called predict_proba / transform. */
int  bm_crbm_debug_last_step(bm_crbm* crbm, const char* name, void* host, size_t bytes);
int  bm_crbm_predict_proba(bm_crbm* crbm, const void* X, int32_t rows, float* out);    /* p(y|x): out [rows, n_classes] */
int  bm_crbm_transform(bm_crbm* crbm, const void* X, int32_t rows, float* out);        /* E[h|x]: out [rows, n_hidden]  */

#ifdef __cplusplus
}
#endif
#endif  /* BM_H_ */
