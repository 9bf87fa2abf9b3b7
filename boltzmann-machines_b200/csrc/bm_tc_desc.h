// Descriptors of the tensor-core program kernel (bm_tc.cu): what the host fills in and the kernel reads.  In a header of
// their own so that test infrastructure which interprets a launch on the CPU (tests/hostsim) reads the SAME definitions.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace bm {

// everything of an op except its tensor maps: copied to shared memory at kernel start so that no
// role ever waits on global memory for a descriptor field
constexpr int MAX_KCHUNKS = 32;     // granule-ordered dataflow covers K <= 2048

struct TcPhaseLite {
    int M, N, BN, m_groups, n_tiles, splits, n_pairs;
    int chunks[2], a_mn[2], b_mn[2], a_neg[2], a_row0[2], a_k0[2], a_batch[2];
    // which CTA pairs execute this op: pair c takes the op's units c - pair_begin, + pair_count, + 2 pair_count ...
    // (chain ops keep a fixed (row block, column block) -> pair map; ops that only feed the end of the step --
    // the positive half of dW -- get the pairs the chain never uses and run beside it)
    int pair_begin, pair_count, n_units;
    unsigned long long split_stride;
    float acc_scale, bias_scale;
    const float* bias;
    const float* sigma;
    union {
        const float* noise_sigma;    // Gaussian draws
        const float* ais_base;       // AIS ops (which never draw Gaussians): per-column base bias a, added after the beta
                                     // scaling -- sigmoid(beta u + a) (DESIGN.md §5.4d); nullable, null is a = 0
    };
    int act, sample, mode;
    uint32_t k0, k1;                 // Philox key of this op's draws (an engine's own programs: the launch key; training groups:
                                     // each member's seed)
    uint32_t rng_c2;                 // site | t << 8
    __nv_bfloat16* out_mean_bf;  int ld_mean_bf;
    __nv_bfloat16* out_state_bf; int ld_state_bf;
    float* out_f32;              int ld_f32;
    int n_deps;
    const int* dep_ctr[3]; int dep_need[3]; int dep_groups[3];   // dep_groups == 0: same row group only
    int* done_ctr;                   // [m_groups] completion counters of this op (nullable)
    // granule-level dataflow (row-block dependencies): the producer op publishes every 64-column
    // granule of a tile (two 32-column epilogue chunks) as soon as it is stored; the consumer walks its
    // K chunks in the order in which the producer's epilogues finish them, so its MMAs overlap the
    // producer's epilogue instead of waiting for the whole row block.
    int* chunk_ctr;                  // [m_groups * n_tiles * gran_per_tile] of this op (nullable)
    int gran_per_tile;               // ceil(BN / 64)
    const int* dep_chunk_ctr;        // the producer's granule counters (nullable: unit-level waits only)
    int dep_gran_row, dep_chunk_need;     // counters per producer row group; arrivals per granule
    unsigned char k_order[MAX_KCHUNKS];   // order in which this op consumes its K chunks
    unsigned char k_dep_a[MAX_KCHUNKS], k_dep_b[MAX_KCHUNKS];   // producer granules K chunk c overlaps
    // AIS (dbm.py:650-736) inside the epilogue.  ais_kind 1 ("units"): the accumulator is the shared pre-activation z of a
    // temperature step; the thread adds  sum_n [softplus(ais_b z) - softplus(ais_a z)]  of its row to ais_logw[row] (fp64 atomics;
    // skipped when ais_logw is null) and, if a state output is given, emits sample(sigmoid(ais_next * z)) -- the unit updates of the
    // next transition.  ais_kind 2 ("state"): an ordinary sigmoid / Bernoulli op whose epilogue also adds
    // ais_lin * sum_n state[n] * (bias_scale * bias[n] * -log2 e)  to ais_logw[row]  (the linear term of log p*, dbm.py:658).
    // With a base (ais_base above) every sigmoid argument gains + a[n]: the units op draws from sigmoid(ais_next z + a) and adds
    // softplus(ais_b z + a) - softplus(ais_a z + a); the state op draws from sigmoid(acc_scale acc + bias_scale bias + a), and
    // its linear term stays without a.
    int ais_kind;
    float ais_a, ais_b, ais_next, ais_lin;
    double* ais_logw;
    uint32_t tick_off;               // added to the launch's tick for this op's draws
    uint32_t row_off;                // added to the launch's first row for this op's draws (tempered particle slots)
};
struct alignas(64) TcPhase {
    CUtensorMap tmA[2], tmB[2];      // read by the TMA unit from global / parameter memory
    CUtensorMap tmOut[2];            // bf16 outputs (0: means, 1: states): TMA stores of 64-column granules
    TcPhaseLite l;
};
struct TcLaunch {
    TcPhase inl;                     // single-op launches carry their descriptor in the parameters
    const TcPhase* phases;           // programs: descriptors in global memory
    int n_phases, total_units;
    uint32_t k0, k1, tick, row0;     // Philox key every op of the launch carries unless it has its own (TcPhaseLite::k0) /
                                     // call tick / first global row of this shard
    int batch_row;
    int stages, stage_bytes;
    unsigned long long* dbg;
    int flags;                       // bit 0: granule polls use acquire loads (no gpu-scope fence afterwards)
    // 0x007FFFFF / 0x3F800000 as RUN-TIME values: (word & mant) | one is then ONE LOP3 (register + constant-bank
    // operand); as literals ptxas emits two LOP3 with immediates -- 16 extra instructions per 16-column chunk
    uint32_t mant_mask, one_bits;
    // dataflow counters are never reset between launches of a program: launch number `epoch` (1, 2, ...) waits for
    // epoch x the per-launch arrival counts (saves a memset per step; the host resets them every 2^20 launches)
    int epoch;
    int poll_ns, epi_ns;             // back-off of the granule polls / of the epilogue's wait for an accumulator
};

// ---- the whole parameter update of a CD step in ONE launch (base_rbm.py:445-474) --------------------------------------
// The statistics arrive as split-K slices written by the step's program:
//   part : `splits` slices of [(srow + 2) x H] fp32: rows 0..V-1 = X^T h0_means - v_k^T h_k_means   (:447-448)
//                                                   row  srow    = sum_rows (h0_means - h_k_means)     (:453)
//                                                   row  srow+1  = - sum_rows h_k_means                (:457, negated)
//          (these two rows come out of the same GEMMs: the batch buffers carry two constant columns at column srow >= V;
//           rows V .. srow-1 are don't-cares)
//   vpart: `vsplits` slices of [V] fp32 whose sum is sum_rows (X - v_k)                               (:451)
// Blocks [0, weight blocks) update W / dW / the bf16 shadow (sparsity penalty recomputed from q_old and row V+1);
// the remaining blocks update vb, hb, their accumulators, q_means (into q_new: q_old is still being read) and `pen`.
struct CdTail {
    int V, H, srow;
    const float* part;  size_t stride;  int splits;
    const float* vpart; size_t vstride; int vsplits;
    float n_div, lr, mom, l2, damp, cost, target;
    float *W, *dW, *vb, *hb, *dvb, *dhb;
    const float* q_old; float* q_new; float* pen;
    __nv_bfloat16* Wb; int ldwb;
};

}  // namespace bm
