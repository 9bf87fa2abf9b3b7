// Fused "layer ops" on the Hopper tensor cores (sm_90a: wgmma + TMA + mbarrier), as a persistent
// multi-phase dataflow kernel.
//
//   C[M,N] = sum_p (+/-) A_p * B_p^T          bf16 operands, fp32 accumulation in registers
//   out    = sample(act(acc_scale * C * sigma + bias_scale * bias))
//
// One such op replaces, per Gibbs half-step, the reference's tf.matmul + 3 element-wise kernels +
// the random_uniform/Less/Cast sampling chain (rbm/base_rbm.py:329-365, layers.py:34-51); the dW op
// replaces the two gradient GEMMs (base_rbm.py:447-448) by ONE GEMM over the concatenated batch
// dimension whose negative phase is subtracted by the MMA's scale-a = -1.  A *program* strings the
// 2k+1 half-steps of a CD-k chain and its dW into one launch: units (op, row-block pair, column
// block) are walked in a fixed global order by all CTA pairs and start as soon as the row blocks they
// read are complete (per-row-block counters in global memory), so nothing waits on a kernel boundary,
// and the epilogue of one half-step overlaps the MMAs of the next.  Activations pass between ops
// through L2-resident bf16 buffers (8 MB at batch 4096, well inside the 50 MB L2).
//
// Per CTA (384 threads, one CTA per SM, 128-row tiles; a "pair" is two CTAs that own the two
// 128-row blocks of a 256-row group -- a scheduling unit of the dataflow, the CTAs share nothing):
//   warps 0-7  two consumer warpgroups: warpgroup g issues wgmma m64n64k16 for tile rows 64g..64g+63
//              (one instruction per 64-column block of the tile and one for a last 16/32/48-column block, accumulators in registers), then runs
//              the epilogue on its accumulators: bias, sigmoid by ex2/rcp, Philox-4x32-10 in registers,
//              bf16 outputs into a 128B-swizzled staging FIFO, fp32 outputs straight to global memory
//   warp 11    TMA producer: 128B-swizzled tiles, mbarrier ring of 3 x 48 KiB (BN = 256) to 6 x 24 KiB (BN = 64) stages
//   warps 9-10 publishers: TMA-store the staged bf16 granules and publish them (fence + atomic)
//              for the ops that read them
// Operand layouts: K-major and MN-major shared-memory descriptors are both used (wgmma's transpose
// bits) so that a single bf16 copy of W serves v->h (W as MN-major B) and h->v (W as K-major B) and no
// activation is ever transposed in memory (dW takes X and h as MN-major A and B).
#include "bm_tc.h"
#include "bm_tc_desc.h"
#include <cuda.h>
#include <map>
#include <tuple>
#include <mutex>
#include <string.h>
#include <stdlib.h>
#include <algorithm>
#include <utility>

namespace bm {

constexpr int BM = 128;            // rows per CTA tile (two warpgroups x 64)
constexpr int BK = 64;             // K per pipeline stage = one 128-byte swizzle atom of bf16
constexpr int MAX_BN = 256;        // accumulator columns per tile: up to 4 x 32 fp32 registers per consumer thread
constexpr int NB_MAX = MAX_BN / 64;
// Register split between the warpgroups (setmaxnreg): the producer warpgroup (TMA, publishers) gives registers to the two
// consumer warpgroups, whose 128 accumulator registers at BN = 256 would not fit the launch's 168.  The CTA keeps the registers
// it was launched with (168 x 384): a split that asks for more leaves setmaxnreg.inc waiting for ever.
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;
constexpr int MAX_STAGES = 10;
constexpr int ACC_STAGES = 2;      // per-unit barriers and bias slices are double-buffered
constexpr int A_BYTES = BM * BK * 2;           // 16 KiB
constexpr int RING_BYTES = 160 * 1024;                // 3 x 48 KiB stages (BN = 256) ... 6 x 24 KiB (BN = 64)
constexpr int N_OUT_BUF = 4;                          // bf16 output staging FIFO: 64-column x 128-row granules
constexpr int OUT_BUF_BYTES = BM * 64 * 2;            // 16 KiB each, 128B-swizzled like the operand tiles
constexpr int OUT_BYTES = N_OUT_BUF * OUT_BUF_BYTES;
constexpr int SMEM_BARRIER_BYTES = 320;   // full/empty ring, tempty, unit/granule barriers
constexpr int GRAN_COLS = 64;             // bf16 outputs leave the SM (and are published) in 64-column granules
constexpr int CONSUMER_THREADS = 256;
constexpr int CONSUMER_WARPS = CONSUMER_THREADS / 32;
constexpr int TC_THREADS = CONSUMER_THREADS + 128;
constexpr int LAUNCH_REGS = 65536 / TC_THREADS / 8 * 8;   // per thread under __launch_bounds__(TC_THREADS, 1): 168
// Warp roles.  The SM's issue arbiter prefers the highest warp id: the single-thread roles whose latency
// is on the critical path (TMA producer, publishers) get the highest ids.  Warp 8 has no role.
constexpr int W_PUB0 = 9, W_PUB1 = 10, W_TMA = 11;

enum : int {
    MODE_GENERIC = 0,                // every combination, flags read at run time
    MODE_SIG_BERN_MEAN_STATE = 1,    // h0: sigmoid, Bernoulli draw, bf16 means + bf16 states
    MODE_SIG_BERN_STATE = 2,         // mid-chain hidden: states only
    MODE_SIG_MEAN = 3,               // probabilities only (visible means, last hidden means)
    MODE_RAW_F32 = 4,                // raw fp32 accumulators (dW partials, linear pre-activations)
    MODE_AIS_UNITS = 5,              // AIS: importance-weight increment of the row + sampled unit updates of the next transition
    MODE_AIS_STATE = 6,              // AIS: sampled transition (sigmoid, Bernoulli, states) + the linear term of log p*
    MODE_AIS_UNITS_S = 7,            // AIS units op without a weight increment (first transition, sweeps > 0)
    MODE_AIS_UNITS_G = 8             // AIS units op, run-time flags (unsampled units, the ladder's last increment, far-apart temperatures)
};

constexpr int MAX_PHASES = 96;
// The series form of the AIS increment (pair_body, MODE_AIS_UNITS) is used for ladders of >= 400 temperatures: with
// t = (b - a) z and d = (next - (a + b) / 2) z its errors are t^2/24 sigma''/sigma (midpoint rule) and d^4/24 sigma''''/sigma
// (third-order series) relative to the term -- < 3e-6 and < 1e-8 for |z| <= 10 at these spacings, and both vanish with
// sigma' for large |z|.  Coarser ladders take the closed form (MODE_AIS_UNITS_G).
constexpr float AIS_MAX_CT = 2.5e-3f, AIS_MAX_CD = 4.0e-3f;
constexpr int SBIAS_BYTES = ACC_STAGES * MAX_BN * (int)sizeof(float);

constexpr int SMEM_BYTES = RING_BYTES + OUT_BYTES + SMEM_BARRIER_BYTES + SBIAS_BYTES;     // 231,744 of 232,448

// The ops of the running launch.  Constant memory on purpose: indexed by warp-uniform values it is read
// through the uniform datapath, so the TMA / MMA issue loops keep their descriptors, coordinates and
// trip counts in uniform registers.
__constant__ TcPhaseLite c_ph[MAX_PHASES];
static_assert(PRODUCER_REGS * 128 + CONSUMER_REGS * CONSUMER_THREADS <= LAUNCH_REGS * TC_THREADS,
              "the setmaxnreg split must fit the registers the CTA is launched with");


// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Every wait of the kernel is bounded: a wait that has not been satisfied after HANG_NS of wall time (a lost
// arrival, stale dataflow counters) traps -- the launch fails with an error instead of holding the GPU for
// ever.  The clock is only read every 4096 failed attempts.
constexpr unsigned long long HANG_NS = 4000000000ull;
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void hang_guard(uint32_t& n, unsigned long long& t0) {
    if ((++n & 0xFFFu) == 0) {
        const unsigned long long t = gtime();
        if (t0 == 0) t0 = t;
        else if (t - t0 > HANG_NS) __trap();
    }
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    uint32_t n = 0; unsigned long long t0 = 0;
    for (;;) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) break;
        hang_guard(n, t0);
    }
}
// for waits that are expected to be long (consumers waiting for a staging buffer): sleep between attempts
// instead of spinning in the issue slots of the busy roles
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, uint32_t ns = 128) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    uint32_t n = 0; unsigned long long t0 = 0;
    for (;;) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) break;
        __nanosleep(ns);
        hang_guard(n, t0);
    }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, uint64_t map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_2d(uint64_t map, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t a) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(a) : "memory");
}
// release: everything this thread has observed (completed bulk stores, barrier-acquired stores of the
// consumer warps) is visible to whoever acquires the counter
__device__ __forceinline__ void red_release_add(int* p, int v) {
    asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}
// One lane of a converged warp (elect.sync): unlike `lane == 0`, ptxas knows that exactly one thread
// executes the guarded code and moves its operands to uniform registers.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .b32 rx;\n\t"
        ".reg .pred px;\n\t"
        "elect.sync rx|px, 0xffffffff;\n\t"
        "@px mov.s32 %0, 1;\n\t"
        "}" : "+r"(pred));
    return pred != 0;
}
#define DBG_MARK(slot) do { if (L.dbg && blockIdx.x == 0) L.dbg[(slot)] = (unsigned long long)clock64(); } while (0)
// per-unit marks of CTA 0: slot 64 + ord * 8 + kind (ord = ordinal of the unit within this CTA, < 24)
#define DBG_UNIT(kind, ord) do { if (L.dbg && blockIdx.x == 0 && (ord) < 24) L.dbg[64 + (ord) * 8 + (kind)] = (unsigned long long)clock64(); } while (0)

// ---- wgmma ---------------------------------------------------------------------------------
// every warp of a warpgroup executes one of them, at the top of its role's branch
__device__ __forceinline__ void regs_to_consumers() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS)); }
__device__ __forceinline__ void regs_from_producers() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS)); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64xN] (+)= (+/-A)[64x16] * B[16xN], N = 16, 32, 48 or 64: bf16 operands from shared memory, fp32 accumulator fragment `d`
// (thread t of the warpgroup holds rows 16 (t/32) + (t%32)/4 (+8) and columns 8 i + 2 (t%4) (+1), registers 4 i .. 4 i + 3).
// TA / TB: the operand is MN-major (wgmma transpose bit); NEG: scale-a = -1.
template <int TA, int TB, int NEG>
__device__ __forceinline__ void wgmma_n16(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, %11, 1, %12, %13;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d), "n"(NEG ? -1 : 1), "n"(TA), "n"(TB));
}
template <int TA, int TB, int NEG>
__device__ __forceinline__ void wgmma_n32(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, %19, 1, %20, %21;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d), "n"(NEG ? -1 : 1), "n"(TA), "n"(TB));
}
template <int TA, int TB, int NEG>
__device__ __forceinline__ void wgmma_n48(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
        "%24, %25, p, %27, 1, %28, %29;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(da), "l"(db), "r"(scale_d), "n"(NEG ? -1 : 1), "n"(TA), "n"(TB));
}
template <int TA, int TB, int NEG>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, %35, 1, %36, %37;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d), "n"(NEG ? -1 : 1), "n"(TA), "n"(TB));
}
template <int N, int TA, int TB, int NEG>
__device__ __forceinline__ void wgmma_m64nk16(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (N == 16) wgmma_n16<TA, TB, NEG>(d, da, db, scale_d);
    else if constexpr (N == 32) wgmma_n32<TA, TB, NEG>(d, da, db, scale_d);
    else if constexpr (N == 48) wgmma_n48<TA, TB, NEG>(d, da, db, scale_d);
    else wgmma_n64<TA, TB, NEG>(d, da, db, scale_d);
}

// Shared-memory matrix descriptor (wgmma): start address [0,14), leading byte offset [16,30), stride byte
// offset [32,46) (all >> 4), layout type SWIZZLE_128B = 1 at bits [62,64).
//   K-major tile  [rows][64 k] : 8-row groups are 1024 B apart (SBO); LBO unused.
//   MN-major tile [64 k][64 mn] boxes of 8 KiB: 64-wide MN blocks are 8192 B apart (LBO),
//                 8-k groups 1024 B apart (SBO).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, int mn_major) {
    const uint64_t lbo = mn_major ? (8192u >> 4) : 1u;
    const uint64_t sbo = 1024u >> 4;
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (lbo << 16) | (sbo << 32) | (1ull << 62);
}

// One K chunk (64) of the warpgroup's 64 x BN accumulator, BN = 16 BN16: 4 K=16 steps x (BN / 64 blocks of 64 columns + a
// last block of BN % 64), as one wgmma group.  The A rows of warpgroup g and the B columns of block j both sit 8 KiB apart in
// either layout (one 64-row / 64-column box each), and a K=16 step advances 32 B (K-major, inside the swizzle atom) or 2 KiB
// (MN-major, two 8-k groups).  Every run-time choice is a template argument: a wgmma on a path ptxas cannot prove
// warpgroup-uniform is serialised.
template <int TA, int TB, int NEG, int BN16>
__device__ __forceinline__ void mma_chunk(float (&acc)[NB_MAX][32], uint32_t sA, uint32_t sB, uint32_t first) {
    constexpr int NB = BN16 / 4, TAIL = 16 * (BN16 % 4);
    const uint32_t a_step = TA ? 2048u : 32u, b_step = TB ? 2048u : 32u;
    wg_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
        const uint64_t da = make_smem_desc(sA + (uint32_t)k * a_step, TA);
        const uint32_t scale_d = (first && k == 0) ? 0u : 1u;
#pragma unroll
        for (int j = 0; j < NB; ++j)
            wgmma_m64nk16<64, TA, TB, NEG>(acc[j], da, make_smem_desc(sB + (uint32_t)j * 8192u + (uint32_t)k * b_step, TB), scale_d);
        if constexpr (TAIL > 0)
            wgmma_m64nk16<(TAIL > 0 ? TAIL : 64), TA, TB, NEG>(acc[NB < NB_MAX ? NB : 0], da,
                                                             make_smem_desc(sB + (uint32_t)NB * 8192u + (uint32_t)k * b_step, TB), scale_d);
    }
    wg_commit();
}
// cfg = (A MN-major) << 2 | (B MN-major) << 1 | negated; BN a multiple of 16 (of 64 when B is MN-major), at most 256
template <int C>
__device__ __forceinline__ void mma_chunk_cfg(int bn16, float (&acc)[NB_MAX][32], uint32_t sA, uint32_t sB, uint32_t first) {
    constexpr int TA = (C >> 2) & 1, TB = (C >> 1) & 1, NEG = C & 1;
    if constexpr (TB) {
        switch (bn16) {
            case 4: mma_chunk<TA, TB, NEG, 4>(acc, sA, sB, first); break;
            case 8: mma_chunk<TA, TB, NEG, 8>(acc, sA, sB, first); break;
            case 12: mma_chunk<TA, TB, NEG, 12>(acc, sA, sB, first); break;
            default: mma_chunk<TA, TB, NEG, 16>(acc, sA, sB, first); break;
        }
    } else {
        switch (bn16) {
#define BM_MMA_CASE(W) case W: mma_chunk<TA, TB, NEG, W>(acc, sA, sB, first); break;
            BM_MMA_CASE(1) BM_MMA_CASE(2) BM_MMA_CASE(3) BM_MMA_CASE(4) BM_MMA_CASE(5) BM_MMA_CASE(6) BM_MMA_CASE(7)
            BM_MMA_CASE(8) BM_MMA_CASE(9) BM_MMA_CASE(10) BM_MMA_CASE(11) BM_MMA_CASE(12) BM_MMA_CASE(13) BM_MMA_CASE(14)
            BM_MMA_CASE(15)
#undef BM_MMA_CASE
            default: mma_chunk<TA, TB, NEG, 16>(acc, sA, sB, first); break;
        }
    }
}
__device__ __forceinline__ void mma_chunk_any(int cfg, int bn16, float (&acc)[NB_MAX][32], uint32_t sA, uint32_t sB, uint32_t first) {
    switch (cfg) {
        case 0: mma_chunk_cfg<0>(bn16, acc, sA, sB, first); break;
        case 1: mma_chunk_cfg<1>(bn16, acc, sA, sB, first); break;
        case 2: mma_chunk_cfg<2>(bn16, acc, sA, sB, first); break;
        case 3: mma_chunk_cfg<3>(bn16, acc, sA, sB, first); break;
        case 4: mma_chunk_cfg<4>(bn16, acc, sA, sB, first); break;
        case 5: mma_chunk_cfg<5>(bn16, acc, sA, sB, first); break;
        case 6: mma_chunk_cfg<6>(bn16, acc, sA, sB, first); break;
        default: mma_chunk_cfg<7>(bn16, acc, sA, sB, first); break;
    }
}

__device__ __forceinline__ float fast_softplus(float x) { return fmaxf(x, 0.f) + __logf(1.0f + __expf(-fabsf(x))); }
// sigmoid(x) = 1 / (1 + 2^(-x log2 e)): ex2.approx + rcp.approx keep the *relative* error of small
// probabilities at ~1e-7 (tanh.approx would not)
__device__ __forceinline__ float sigmoid_from_neg_log2(float t) {   // t = -x * log2(e)
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return r;
}
// asfloat((word & 0x7fffff) | 0x3f800000) in [1, 2): TF's Uint32ToFloat before its "- 1.0f"
__device__ __forceinline__ float u32_to_one_two(uint32_t w, uint32_t mant_mask, uint32_t one_bits) {
    uint32_t bits;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(bits) : "r"(w), "r"(mant_mask), "r"(one_bits));
    return __uint_as_float(bits);
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h2);
}
// Polling uses relaxed loads: an acquire load makes ptxas emit a full L1 invalidation on every iteration,
// which evicted the consumer warps' bias/constant lines for as long as a producer warp was waiting.  One
// acquire fence follows the successful poll.
__device__ __forceinline__ int ld_acquire(const int* p) {
    int v; asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ int ld_relaxed(const int* p) {
    int v; asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}

// ------------------------------------------------------------------------------------------
// epilogue of one tile, specialised per output mode
// ------------------------------------------------------------------------------------------
template <int MODE> struct EpiCfg {
    static constexpr bool fixed = MODE != MODE_GENERIC;
    static constexpr bool ais_units = (MODE == MODE_AIS_UNITS || MODE == MODE_AIS_UNITS_S || MODE == MODE_AIS_UNITS_G);
    static constexpr bool ais = ais_units || MODE == MODE_AIS_STATE;
    static constexpr int act = (MODE == MODE_RAW_F32 || ais_units) ? ACT_LINEAR : ACT_SIGMOID;
    static constexpr int sample = (MODE == MODE_SIG_BERN_MEAN_STATE || MODE == MODE_SIG_BERN_STATE || MODE == MODE_AIS_STATE) ? SMP_BERNOULLI : SMP_NONE;
    static constexpr bool mean_bf = (MODE == MODE_SIG_BERN_MEAN_STATE || MODE == MODE_SIG_MEAN);
    static constexpr bool state_bf = (MODE == MODE_SIG_BERN_MEAN_STATE || MODE == MODE_SIG_BERN_STATE || MODE == MODE_AIS_STATE);
    static constexpr bool f32 = (MODE == MODE_RAW_F32);
};

// the epilogue's view of a phase, copied into registers once per unit
struct EpiPhase {
    int M, N, BN, act, sample;
    float acc_scale, bias_scale;
    const float* __restrict__ sigma;
    const float* __restrict__ noise_sigma;
    __nv_bfloat16* __restrict__ out_mean_bf;
    __nv_bfloat16* __restrict__ out_state_bf;
    float* __restrict__ out_f32;              int ld_f32;
    unsigned long long split_stride;
    float ais_a, ais_b, ais_next, ais_lin;
    float ais_ct, ais_cd;          // (b - a) and (next - (a + b) / 2): z-multipliers of the series form of the increment
    double* ais_logw;
};
struct EpiCtx {
    EpiPhase p;
    RngKey rng;
    int m0;                       // global row of this thread's first accumulator row (the second is m0 + 8)
    int r0;                       // the same row inside the 128-row tile
    int n_blk, split;             // the tile's column block and K split
    int lane;
    const float* sbias;           // shared memory: bias_scale * bias (x -log2 e for sigmoid) of the tile's columns
    uint32_t out_base;            // shared address of the staging FIFO
    uint64_t* out_full;           // [N_OUT_BUF] a staged granule is complete (8 warp arrivals)
    uint64_t* out_free;           // [N_OUT_BUF] its TMA store has read the buffer (publisher)
    uint32_t* seq;                // FIFO position (same sequence in every consumer warp and in the publishers)
    uint32_t mant_mask, one_bits; // TcLaunch::mant_mask / one_bits
};

// softplus(b z) - softplus(a z) = log1p(sigmoid(a z) * expm1((b - a) z)) without cancellation (b - a ~ 1e-3): short series
// where both arguments are small (the common case), the library functions elsewhere
__device__ __forceinline__ float ais_softplus_diff(float a, float b, float z) {
    const float sa = sigmoid_from_neg_log2(a * z * -1.4426950408889634f);
    const float t = (b - a) * z;
    float em;
    if (fabsf(t) < 0.03f) em = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.0f / 120.0f, 1.0f / 24.0f), 1.0f / 6.0f), 0.5f), 1.0f);
    else em = expm1f(t);
    const float y = sa * em;
    if (fabsf(y) < 0.03f) return y * fmaf(y, fmaf(y, fmaf(y, fmaf(y, 0.2f, -0.25f), 1.0f / 3.0f), -0.5f), 1.0f);
    return log1pf(y);
}

// Two adjacent accumulator columns (n, n + 1; n even) of one row m: activation, sampling, packed bf16 mean / state and the
// fp32 store.  wf / ws are the Philox words of the two columns: words 2 (n % 4 / 2) and 2 (n % 4 / 2) + 1 of the row's
// block n / 4 -- the same draws, column for column, as a thread that owns the whole block.
// Returns the pair's contribution to the row's AIS log-weight (AIS modes) or 0.
template <int MODE>
__device__ __forceinline__ float pair_body(const EpiCtx& c, float v0, float v1, uint32_t wf, uint32_t ws, float b0, float b1,
                                           int n, int m, bool row_ok, float* out_f32, bool f32_vec,
                                           uint32_t& mean_pk, uint32_t& state_pk) {
    typedef EpiCfg<MODE> E;
    const EpiPhase& p = c.p;
    float ais_part = 0.f;
    const int act = E::fixed ? E::act : p.act;
    const int smp = (MODE == MODE_AIS_UNITS || MODE == MODE_AIS_UNITS_S) ? SMP_BERNOULLI :
                    (E::fixed && MODE != MODE_AIS_UNITS_G) ? E::sample : p.sample;
    // fold the sigmoid's -log2(e) into the affine map of the accumulator
    const float a_s = (act == ACT_SIGMOID) ? p.acc_scale * -1.4426950408889634f : p.acc_scale;
    const bool has_sigma = !E::fixed && p.sigma != nullptr;
    const bool do_f32 = E::fixed ? E::f32 : (out_f32 != nullptr);
    const float v[2] = {v0, v1};
    const float bq[2] = {b0, b1};
    const uint32_t words[2] = {wf, ws};
    float g[2] = {0.f, 0.f};
    if (!E::fixed && smp == SMP_GAUSSIAN) {
        const float u1 = fmaxf(u32_to_unit_float(wf), 1.0e-7f);
        const float r = sqrtf(-2.0f * __logf(u1));
        float s, co;
        __sincosf(6.2831853071795864769f * u32_to_unit_float(ws), &s, &co);
        g[0] = s * r; g[1] = co * r;
    }
    float mu[2], st[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const bool valid = n + j < p.N;
        float x = a_s * v[j];
        if (has_sigma && valid) x *= p.sigma[n + j];
        x += bq[j];
        float m_ = x;
        float s_;
        if (MODE == MODE_AIS_UNITS || MODE == MODE_AIS_UNITS_S) {
            // x = z (acc_scale = bias_scale = 1).  p = sigmoid(beta_next z) serves the draw AND the weight increment:
            //   softplus(b z) - softplus(a z) = int_a^b z sigmoid(beta z) dbeta = t sigmoid(m z)  (+ t^3 z^-2 ... / 24: < 1e-7 t)
            //   with t = (b - a) z, m = (a + b) / 2, and sigmoid(m z) = sigmoid(beta_next z - d), d = (beta_next - m) z, as its
            //   third-order series in d around p (error terms: AIS_MAX_CT / AIS_MAX_CD above).
            float e_, p_;
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e_) : "f"(x * p.ais_next * -1.4426950408889634f));
            asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(p_) : "f"(1.0f + e_));
            s_ = ((u32_to_one_two(words[j], c.mant_mask, c.one_bits) - 1.0f) < p_) ? 1.0f : 0.0f;
            if (MODE == MODE_AIS_UNITS) {
                const float q_ = fmaf(-p_, p_, p_);                                 // sigma1 = p (1 - p)
                const float d_ = p.ais_cd * x;
                const float s2 = fmaf(-2.0f, p_, 1.0f);                             // sigma2 / sigma1
                const float s3 = fmaf(-6.0f, q_, 1.0f);                             // sigma3 / sigma1
                const float in = fmaf(-d_ * (1.0f / 3.0f), s3, s2);
                const float sm = fmaf(-d_ * q_, fmaf(-0.5f * d_, in, 1.0f), p_);    // sigmoid(m z)
                ais_part = fmaf(valid ? p.ais_ct * x : 0.f, sm, ais_part);
            }
            mu[j] = 0.f; st[j] = s_;
            continue;
        }
        if (MODE == MODE_AIS_UNITS_G) {
            // any temperatures, optional sampling / output: the closed forms
            if (p.ais_logw && valid) ais_part += ais_softplus_diff(p.ais_a, p.ais_b, x);
            float e_;
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e_) : "f"(x * p.ais_next * -1.4426950408889634f));
            const float d_ = 1.0f + e_;
            if (smp == SMP_BERNOULLI) {
                const float u12 = u32_to_one_two(words[j], c.mant_mask, c.one_bits);
                s_ = (fmaf(u12, d_, -d_) < 1.0f) ? 1.0f : 0.0f;
            } else {
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(s_) : "f"(d_));
            }
            mu[j] = 0.f; st[j] = s_;
            continue;
        }
        if (MODE == MODE_SIG_BERN_STATE || MODE == MODE_AIS_STATE) {
            // only the draw is needed: u < 1/(1+e)  <=>  u*(1+e) < 1, with u = u12 - 1 folded into one FMA
            // (no reciprocal, no "- 1.0f"); e = inf (p = 0) gives NaN -> 0, e = 0 (p = 1) gives u < 1 -> 1
            float e_;
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e_) : "f"(x));
            const float d_ = 1.0f + e_;
            const float u12 = u32_to_one_two(words[j], c.mant_mask, c.one_bits);
            s_ = (fmaf(u12, d_, -d_) < 1.0f) ? 1.0f : 0.0f;
            mu[j] = 0.f; st[j] = s_;
            if (MODE == MODE_AIS_STATE && valid) ais_part = fmaf(s_, bq[j], ais_part);
            continue;
        }
        if (act == ACT_SIGMOID) m_ = sigmoid_from_neg_log2(x);
        else if (!E::fixed && act == ACT_SOFTPLUS) m_ = fast_softplus(x);
        s_ = m_;
        if (smp == SMP_BERNOULLI) s_ = ((u32_to_one_two(words[j], c.mant_mask, c.one_bits) - 1.0f) < m_) ? 1.0f : 0.0f;
        else if (!E::fixed && smp == SMP_GAUSSIAN)
            s_ = m_ + ((p.noise_sigma && valid) ? p.noise_sigma[n + j] : 1.0f) * g[j];
        mu[j] = m_; st[j] = s_;
    }
    mean_pk = pack_bf16(mu[0], mu[1]);
    state_pk = pack_bf16(st[0], st[1]);
    if (do_f32 && row_ok) {
        float* dst = out_f32 + (size_t)m * p.ld_f32 + n;
        if (f32_vec && n + 1 < p.N) *reinterpret_cast<float2*>(dst) = make_float2(mu[0], mu[1]);
        else {
            if (n < p.N) dst[0] = mu[0];
            if (n + 1 < p.N) dst[1] = mu[1];
        }
    }
    return ais_part;
}

// The warpgroup's share of a tile, granule (64 columns = one accumulator block) by granule: each granule of each bf16
// output takes the next buffer of the staging FIFO, is written by the 8 consumer warps and announced on the buffer's
// `full` barrier; the publisher warps store it with TMA and publish it to the other SMs.
template <int MODE>
__device__ __forceinline__ void epilogue_tile(const EpiCtx& c, const float (&acc)[NB_MAX][32]) {
    typedef EpiCfg<MODE> E;
    const EpiPhase& p = c.p;
    const int nb = (p.BN + GRAN_COLS - 1) / GRAN_COLS;     // the last block may be 16, 32 or 48 columns wide (fp32 outputs only)
    const bool do_mean = E::fixed ? E::mean_bf : (p.out_mean_bf != nullptr);
    const bool do_state = (MODE == MODE_AIS_UNITS || MODE == MODE_AIS_UNITS_S) ? true :
                          (E::fixed && MODE != MODE_AIS_UNITS_G) ? E::state_bf : (p.out_state_bf != nullptr);
    const int smp = (MODE == MODE_AIS_UNITS || MODE == MODE_AIS_UNITS_S) ? SMP_BERNOULLI :
                    (E::fixed && MODE != MODE_AIS_UNITS_G) ? E::sample : p.sample;
    float* const out_f32 = ((E::fixed && !E::f32) || !p.out_f32) ? nullptr : p.out_f32 + (size_t)c.split * p.split_stride;
    // float2 stores: even row pitch, split stride and 8-byte aligned base
    const bool f32_vec = (p.ld_f32 & 1) == 0 && (p.split_stride & 1) == 0 && (reinterpret_cast<uintptr_t>(p.out_f32) & 7) == 0;
    const int lane = c.lane, q = lane & 3;
    const int m1 = c.m0 + 8;
    const bool ok0 = c.m0 < p.M, ok1 = m1 < p.M;
    const bool odd = (lane & 1) != 0;
    // rows r0 and r0 + 8 share their position inside the 128-byte swizzle pattern (r & 7 = lane / 4)
    const uint32_t swz = (uint32_t)(lane >> 2) & 7u;
    const uint32_t off0 = (uint32_t)c.r0 * 128u + (uint32_t)q * 4u, off1 = off0 + 8u * 128u;
    float ais0 = 0.f, ais1 = 0.f;
    uint32_t seq = *c.seq;
#pragma unroll
    for (int j = 0; j < NB_MAX; ++j) {
        if (j >= nb) break;
        uint32_t smem_mean = 0, smem_state = 0;
        int b_mean = 0, b_state = 0;
        if (do_mean) {
            b_mean = (int)(seq % N_OUT_BUF);
            mbar_wait_relaxed(&c.out_free[b_mean], ((seq / N_OUT_BUF) & 1u) ^ 1u);      // first use of a buffer passes at once
            smem_mean = c.out_base + (uint32_t)b_mean * OUT_BUF_BYTES; ++seq;
        }
        if (do_state) {
            b_state = (int)(seq % N_OUT_BUF);
            mbar_wait_relaxed(&c.out_free[b_state], ((seq / N_OUT_BUF) & 1u) ^ 1u);
            smem_state = c.out_base + (uint32_t)b_state * OUT_BUF_BYTES; ++seq;
        }
        const int col0 = c.n_blk * p.BN + j * GRAN_COLS;
        const int gcols = min(GRAN_COLS, p.BN - j * GRAN_COLS);
        if (col0 < p.N) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (8 * i >= gcols) break;
                const int cl = 8 * i + 2 * q;                    // column inside the granule
                const int n = col0 + cl;
                // Philox: the lane pair (q even, q odd) shares the 4-column block n / 4 of rows m0 and m0 + 8.  The even
                // lane draws the block of m0, the odd lane that of m0 + 8, and they swap the halves the other one needs.
                uint32_t w0f = 0, w0s = 0, w1f = 0, w1s = 0;
                if (smp != SMP_NONE) {
                    const U4 w = site_block(c.rng, (uint32_t)(odd ? m1 : c.m0), (uint32_t)(n >> 2));
                    const uint32_t give_f = odd ? w.x : w.z, give_s = odd ? w.y : w.w;
                    const uint32_t got_f = __shfl_xor_sync(0xffffffffu, give_f, 1);
                    const uint32_t got_s = __shfl_xor_sync(0xffffffffu, give_s, 1);
                    if (!odd) { w0f = w.x; w0s = w.y; w1f = got_f; w1s = got_s; }
                    else { w0f = got_f; w0s = got_s; w1f = w.z; w1s = w.w; }
                }
                const float2 b2 = *reinterpret_cast<const float2*>(c.sbias + j * GRAN_COLS + cl);
                uint32_t mp0, sp0, mp1, sp1;
                ais0 += pair_body<MODE>(c, acc[j][4 * i], acc[j][4 * i + 1], w0f, w0s, b2.x, b2.y, n, c.m0, ok0, out_f32, f32_vec, mp0, sp0);
                ais1 += pair_body<MODE>(c, acc[j][4 * i + 2], acc[j][4 * i + 3], w1f, w1s, b2.x, b2.y, n, m1, ok1, out_f32, f32_vec, mp1, sp1);
                // columns past N and rows past M are written to the staging buffer too: the TMA store clips them
                const uint32_t u = (((uint32_t)i ^ swz) << 4);
                if (do_mean) { sts32(smem_mean + off0 + u, mp0); sts32(smem_mean + off1 + u, mp1); }
                if (do_state) { sts32(smem_state + off0 + u, sp0); sts32(smem_state + off1 + u, sp1); }
            }
        }
        if (do_mean || do_state) {
            fence_proxy_async_smem();                // this thread's staging writes -> visible to the TMA unit
            __syncwarp();
            if (lane == 0) {
                if (do_mean) mbar_arrive(&c.out_full[b_mean]);
                if (do_state) mbar_arrive(&c.out_full[b_state]);
            }
        }
    }
    *c.seq = seq;
    if constexpr (E::ais) {
        // the row's log-weight increment: the four lanes of a row sum their columns, one fp64 atomic per row and tile
        ais0 += __shfl_xor_sync(0xffffffffu, ais0, 1); ais0 += __shfl_xor_sync(0xffffffffu, ais0, 2);
        ais1 += __shfl_xor_sync(0xffffffffu, ais1, 1); ais1 += __shfl_xor_sync(0xffffffffu, ais1, 2);
        if (p.ais_logw && q == 0) {
            const float s = MODE == MODE_AIS_STATE ? p.ais_lin : 1.0f;
            if (ok0) asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p.ais_logw + c.m0), "d"((double)(ais0 * s)) : "memory");
            if (ok1) asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p.ais_logw + m1), "d"((double)(ais1 * s)) : "memory");
        }
    }
}

// ------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------
struct UnitInfo { int split, m_group, n_blk, c_begin, c_end, total_chunks; };

// Next unit of CTA pair `cid`: ops in program order, inside an op the units cid - pair_begin (mod pair_count).
// (pi, l) = current op and local unit; l < 0: before the first unit of op pi.  All values are warp-uniform.
__device__ __forceinline__ bool walk_next(int& pi, int& l, int cid, int n_ops) {
    while (pi < n_ops) {
        const TcPhaseLite* p = &c_ph[pi];
        const int rel = cid - p->pair_begin;
        if (rel >= 0 && rel < p->pair_count) {
            l = (l < 0) ? rel : l + p->pair_count;
            if (l < p->n_units) return true;
        }
        ++pi; l = -1;
    }
    return false;
}
__device__ __forceinline__ UnitInfo decode_unit(const TcPhaseLite* ph, int local) {
    UnitInfo u;
    u.split = local % ph->splits;
    const int tile = local / ph->splits;
    u.m_group = tile / ph->n_tiles;
    u.n_blk = tile % ph->n_tiles;
    u.total_chunks = ph->chunks[0] + (ph->n_pairs > 1 ? ph->chunks[1] : 0);
    u.c_begin = (int)(((long long)u.total_chunks * u.split) / ph->splits);
    u.c_end = (int)(((long long)u.total_chunks * (u.split + 1)) / ph->splits);
    return u;
}

// CL = 2: CTAs 2c and 2c + 1 take row blocks 2g and 2g + 1 of row group g of every unit of pair c; CL = 1: one CTA per
// row block (single-op launches with one row block).
template <int CL>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_program_kernel(const __grid_constant__ TcLaunch L) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw;                      // [operand ring | output staging FIFO | barriers | bias]
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // 128B-swizzle atoms need 1024-byte alignment
    uint8_t* const out_stage = smem + RING_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + RING_BYTES + OUT_BYTES);
    uint64_t* empty = full + MAX_STAGES;
    uint64_t* tempty = empty + MAX_STAGES;                        // [ACC_STAGES] the publishers are done with the unit's stage
    uint64_t* unit_bar = tempty + ACC_STAGES;                     // [ACC_STAGES] all consumer warps stored the unit
    uint64_t* out_full = unit_bar + ACC_STAGES;                   // [N_OUT_BUF] staged granule written by all consumer warps
    uint64_t* out_free = out_full + N_OUT_BUF;                    // [N_OUT_BUF] staged granule read by its TMA store

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { DBG_MARK(0); if (L.dbg && blockIdx.x == 0) L.dbg[6] = gtime(); }
    float* const s_bias = reinterpret_cast<float*>(smem + RING_BYTES + OUT_BYTES + SMEM_BARRIER_BYTES);
    const TcPhase* const gph = L.n_phases ? L.phases : &L.inl;      // tensor maps (global / parameter memory)
    if (warp == W_TMA && lane == 0) {
        tma_prefetch_desc(&gph->tmA[0]); tma_prefetch_desc(&gph->tmB[0]);
        for (int s = 0; s < L.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }   // empty: both consumer warpgroups
        for (int a = 0; a < ACC_STAGES; ++a) { mbar_init(&tempty[a], 2); mbar_init(&unit_bar[a], CONSUMER_WARPS); }
        for (int b = 0; b < N_OUT_BUF; ++b) { mbar_init(&out_full[b], CONSUMER_WARPS); mbar_init(&out_free[b], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) DBG_MARK(1);

    const int n_ops = L.n_phases ? L.n_phases : 1;
    // (kept as expressions of blockIdx so that the compiler knows they are warp-uniform)
    const int crank = CL == 2 ? (int)(blockIdx.x & 1u) : 0;
    const int cid = CL == 2 ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;

    if (warp == W_TMA) {
        // ================================ TMA producer =====================================
        regs_to_consumers();
        int stage = 0; uint32_t phase = 0;
        int pi = 0, ul = -1;
        int ord = -1;
        while (walk_next(pi, ul, cid, n_ops)) {
            ++ord;
            const TcPhaseLite* ph = &c_ph[pi];
            const TcPhase* gp = &gph[pi];
            const UnitInfo u = decode_unit(ph, ul);
            if (lane == 0) DBG_UNIT(0, ord);
            // this op's tensor maps -> descriptor cache while the unit still waits for its inputs
            if ((L.flags & 8) && lane < 2 * ph->n_pairs) tma_prefetch_desc(lane & 1 ? &gp->tmB[lane >> 1] : &gp->tmA[lane >> 1]);
            const int BN = ph->BN;
            const uint32_t tx_bytes = A_BYTES + (uint32_t)BN * BK * 2;
            const int m_blk = u.m_group * CL + crank;
            const int n_col0 = u.n_blk * BN;
            // ---- dataflow: wait until the row blocks this unit reads have been written ----------
            if (ph->n_deps > 0) {
                if (lane == 0) {
                    uint32_t hn = 0; unsigned long long ht0 = 0;
                    for (int d = 0; d < ph->n_deps; ++d) {
                        const int* ctr = ph->dep_ctr[d];
                        const int need = ph->dep_need[d] * L.epoch;
                        if (ph->dep_groups[d] == 0) {
                            if (ph->dep_chunk_ctr) continue;          // handled chunk by chunk below
                            while (ld_relaxed(ctr + u.m_group) < need) { __nanosleep(64); hang_guard(hn, ht0); }
                        } else {
                            for (int gq = 0; gq < ph->dep_groups[d]; ++gq)
                                while (ld_relaxed(ctr + gq) < need) { __nanosleep(64); hang_guard(hn, ht0); }
                        }
                    }
                    // acquire the producers' (generic-proxy) stores, then order them before this unit's
                    // TMA reads, which go through the async proxy
                    asm volatile("fence.acq_rel.gpu;" ::: "memory");
                    asm volatile("fence.proxy.async;" ::: "memory");
                }
                __syncwarp();
            }
            if (lane == 0) DBG_UNIT(1, ord);
            const int* const cdep = ph->dep_chunk_ctr ? ph->dep_chunk_ctr + (size_t)u.m_group * ph->dep_gran_row : nullptr;
            // ---- per-unit setup (warp-uniform: uniform registers): operand-pair configuration -------
            const int chunks0 = ph->chunks[0];
            uint64_t mapA[2], mapB[2];
            int a_c0[2], a_c1[2], b_c0[2], b_c1[2], a_mn[2], b_mn[2];
#pragma unroll
            for (int pr = 0; pr < 2; ++pr) {
                const int shift = ph->a_batch[pr] ? L.batch_row : 0;
                a_mn[pr] = ph->a_mn[pr]; b_mn[pr] = ph->b_mn[pr];
                mapA[pr] = (uint64_t)&gp->tmA[pr]; mapB[pr] = (uint64_t)&gp->tmB[pr];
                // box coordinates at K offset 0: K-major {k, row}; MN-major {mn, k}
                a_c0[pr] = a_mn[pr] ? m_blk * BM : 0;
                a_c1[pr] = a_mn[pr] ? ph->a_k0[pr] + shift : ph->a_row0[pr] + shift + m_blk * BM;
                b_c0[pr] = b_mn[pr] ? n_col0 : 0;
                b_c1[pr] = b_mn[pr] ? 0 : n_col0;
            }
            const int nB_mn = BN >> 6;                // 64-column boxes of an MN-major B tile
            const uint32_t smem_base = smem_u32(smem);
            const bool ordered = cdep != nullptr;
            int fenced_upto = u.c_begin;         // K positions [c_begin, fenced_upto) are known ready and fenced
            for (int ci = u.c_begin; ci < u.c_end; ++ci) {
                int c = ci;
                if (ordered) {
                    c = (int)ph->k_order[ci];
                    if (ci >= fenced_upto) {
                        // every lane polls one K position (ci + lane): one L2 round trip tells how long the
                        // prefix of ready positions is (a serial scan costs a round trip per position)
                        const int need = ph->dep_chunk_need * L.epoch;
                        const int n = ci + lane;
                        int ga = 0, gb = 0;
                        if (n < u.c_end) { const int j = (int)ph->k_order[n]; ga = (int)ph->k_dep_a[j]; gb = (int)ph->k_dep_b[j]; }
                        int ready_prefix = 0;
                        uint32_t hn = 0; unsigned long long ht0 = 0;
                        for (;;) {
                            bool ok;
                            if (L.flags & 1) ok = n < u.c_end && ld_acquire(cdep + ga) >= need && (gb == ga || ld_acquire(cdep + gb) >= need);
                            else ok = n < u.c_end && ld_relaxed(cdep + ga) >= need && (gb == ga || ld_relaxed(cdep + gb) >= need);
                            const uint32_t m = __ballot_sync(0xffffffffu, ok);
                            ready_prefix = __ffs(~m) - 1;              // ~m != 0: lanes past c_end are never ready... (32 positions max)
                            if (m == 0xffffffffu) ready_prefix = 32;
                            if (ready_prefix > 0) break;
                            __nanosleep((uint32_t)L.poll_ns);
                            hang_guard(hn, ht0);
                        }
                        fenced_upto = ci + ready_prefix;
                        // acquire the producers' stores, then order them before this unit's TMA reads (async proxy)
                        if (!(L.flags & 1)) asm volatile("fence.acq_rel.gpu;" ::: "memory");
                        // The producers' data was written by TMA stores and is read here by TMA loads (the same
                        // proxy); only the counter travels through the generic proxy.  flags bit 1 narrows the
                        // cross-proxy fence to the global state space, bit 2 drops it (the TMA issue below is
                        // control-dependent on the acquired counter value) -- a full fence.proxy.async also waits
                        // for this thread's own in-flight bulk copies.
                        if (L.flags & 4) {}
                        else if (L.flags & 2) asm volatile("fence.proxy.async.global;" ::: "memory");
                        else asm volatile("fence.proxy.async;" ::: "memory");
                    }
                }
                const int pr = (c >= chunks0) ? 1 : 0;
                const int kc = (c - (pr ? chunks0 : 0)) * BK;
                const uint32_t sA = smem_base + (uint32_t)stage * (uint32_t)L.stage_bytes;
                const uint32_t sB = sA + (uint32_t)A_BYTES;
                const uint64_t mA = pr ? mapA[1] : mapA[0], mB = pr ? mapB[1] : mapB[0];
                const int amn = pr ? a_mn[1] : a_mn[0], bmn = pr ? b_mn[1] : b_mn[0];
                const int ac0 = pr ? a_c0[1] : a_c0[0], ac1 = pr ? a_c1[1] : a_c1[0];
                const int bc0 = pr ? b_c0[1] : b_c0[0], bc1 = pr ? b_c1[1] : b_c1[0];
                mbar_wait(&empty[stage], phase ^ 1);
                if (elect_one()) {               // one thread issues; every operand above is warp-uniform
                    if (ci - u.c_begin < 24 && (L.n_phases == 0 || ord == 1)) DBG_MARK(8 + (ci - u.c_begin));
                    const uint32_t fbar = smem_u32(&full[stage]);
                    mbar_expect_tx(&full[stage], tx_bytes);
                    if (!amn) tma_load_2d(sA, mA, fbar, kc, ac1);
                    else { tma_load_2d(sA, mA, fbar, ac0, ac1 + kc); tma_load_2d(sA + 8192u, mA, fbar, ac0 + 64, ac1 + kc); }
                    if (!bmn) tma_load_2d(sB, mB, fbar, kc, bc1);
                    else for (int j = 0; j < nB_mn; ++j) tma_load_2d(sB + (uint32_t)j * 8192u, mB, fbar, bc0 + j * 64, kc);
                }
                __syncwarp();
                if (++stage == L.stages) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp == W_PUB0 || warp == W_PUB1) {
        // ================================ publishers ========================================
        // Send every staged 64-column granule of the bf16 outputs to global memory with a TMA store
        // and, once that store has completed (bulk async-group wait: no MEMBAR over the SM's whole store
        // stream), bump the granule's dataflow counter with a release: consumers start on a row block's
        // first columns while its last ones are still in the epilogue.  Two publisher threads take the
        // even / odd granules so that one store's completion latency hides behind the other's.
        // fp32 outputs (dW partials) are stored by the consumer warps directly and published per unit.
        regs_to_consumers();
        if (lane == 0) {
            const int pub = warp - W_PUB0;
            int acc = 0; uint32_t acc_phase = 0;
            uint32_t seq = 0;                               // FIFO position of the unit's first granule
            int pi = 0, ul = -1;
            int ord = -1;
            const uint32_t out_base = smem_u32(out_stage);
            while (walk_next(pi, ul, cid, n_ops)) {
                ++ord;
                const TcPhaseLite* ph = &c_ph[pi];
                const TcPhase* gp = &gph[pi];
                const UnitInfo u = decode_unit(ph, ul);
                const bool has_mean = ph->out_mean_bf != nullptr, has_state = ph->out_state_bf != nullptr;
                const int n_arr = (has_mean ? 1 : 0) + (has_state ? 1 : 0);
                const int gpt = n_arr ? ph->gran_per_tile : 0;
                const int row0 = (u.m_group * CL + crank) * BM;
                int* const ctr = ph->chunk_ctr ? ph->chunk_ctr + ((size_t)u.m_group * ph->n_tiles + u.n_blk) * gpt : nullptr;
                for (int g = pub; g < gpt; g += 2) {
                    const int col0 = u.n_blk * ph->BN + g * GRAN_COLS;
                    uint32_t sq = seq + (uint32_t)(g * n_arr);
                    int bufs[2] = {-1, -1};
                    for (int a = 0; a < 2; ++a) {
                        if (!(a == 0 ? has_mean : has_state)) continue;
                        const int b = (int)(sq % N_OUT_BUF);
                        mbar_wait(&out_full[b], (sq / N_OUT_BUF) & 1u);
                        if (col0 < ph->N) tma_store_2d((uint64_t)&gp->tmOut[a], out_base + (uint32_t)b * OUT_BUF_BYTES, col0, row0);
                        bufs[a] = b; ++sq;
                    }
                    bulk_commit();
                    bulk_wait<0>();                          // stores complete: data is in global memory
                    for (int a = 0; a < 2; ++a) if (bufs[a] >= 0) mbar_arrive(&out_free[bufs[a]]);
                    if (ctr && col0 < ph->N) red_release_add(ctr + g, 1);
                }
                seq += (uint32_t)(gpt * n_arr);
                mbar_wait(&unit_bar[acc], acc_phase);      // every consumer warp has finished the unit (direct fp32 stores included)
                if (ph->done_ctr) red_release_add(ph->done_ctr + u.m_group, 1);
                if (pub == 1) DBG_UNIT(6, ord);
                mbar_arrive(&tempty[acc]);                 // the unit barrier of this stage may be reused
                if (++acc == ACC_STAGES) { acc = 0; acc_phase ^= 1; }
            }
        }
    } else if (warp < CONSUMER_WARPS) {
        // ================================ consumers (2 warpgroups) ==========================
        regs_from_producers();
        const int wg = warp >> 2;
        EpiCtx c;
        c.lane = lane;
        uint32_t out_seq = 0;
        c.seq = &out_seq;
        c.out_base = smem_u32(out_stage); c.out_full = out_full; c.out_free = out_free;
        c.mant_mask = L.mant_mask; c.one_bits = L.one_bits;
        c.r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const uint32_t smem_base = smem_u32(smem);
        const uint32_t wg_off = (uint32_t)wg * 8192u;      // this warpgroup's 64 A rows (either layout)
        int stage = 0; uint32_t phase = 0;
        int acc_st = 0; uint32_t acc_phase = 0;
        int pi = 0, ul = -1;
        int ord = -1;
        const int et = threadIdx.x;                // 0..255
        float acc[NB_MAX][32];
        while (walk_next(pi, ul, cid, n_ops)) {
            ++ord;
            const TcPhaseLite* ph = &c_ph[pi];
            const UnitInfo u = decode_unit(ph, ul);
            // the publishers have finished the unit two back, which used this stage's barrier and bias slice
            mbar_wait(&tempty[acc_st], acc_phase ^ 1);
            {   // this tile's (pre-scaled) bias slice -> shared memory
                const float bsc = (ph->act == ACT_SIGMOID) ? ph->bias_scale * -1.4426950408889634f : ph->bias_scale;
                const int n = u.n_blk * ph->BN + et;
                if (et < MAX_BN) s_bias[acc_st * MAX_BN + et] = (ph->bias && et < ph->BN && n < ph->N) ? bsc * __ldg(ph->bias + n) : 0.f;
                asm volatile("bar.sync 1, 256;" ::: "memory");
                c.sbias = s_bias + acc_st * MAX_BN;
            }
            // ---- mainloop: one wgmma group per K chunk, the previous chunk's stage released once its group retired
            const int bn16 = ph->BN / 16;
            const int chunks0 = ph->chunks[0];
            const int cfg0 = (ph->a_mn[0] << 2) | (ph->b_mn[0] << 1) | ph->a_neg[0];
            const int cfg1 = (ph->a_mn[1] << 2) | (ph->b_mn[1] << 1) | ph->a_neg[1];
            const bool ordered = ph->dep_chunk_ctr != nullptr;
            if (threadIdx.x == 0) DBG_UNIT(2, ord);
            int prev = -1;
            for (int ci = u.c_begin; ci < u.c_end; ++ci) {
                const int cc = ordered ? (int)ph->k_order[ci] : ci;     // same order as the producer warp
                const int cfg = (cc >= chunks0) ? cfg1 : cfg0;
                const uint32_t sA = smem_base + (uint32_t)stage * (uint32_t)L.stage_bytes;
                mbar_wait(&full[stage], phase);
                mma_chunk_any(cfg, bn16, acc, sA + wg_off, sA + (uint32_t)A_BYTES, ci == u.c_begin ? 1u : 0u);
                wg_wait<1>();
                if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == L.stages) { stage = 0; phase ^= 1; }
            }
            wg_wait<0>();
            if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
            if (threadIdx.x == 0) { DBG_MARK(3); DBG_UNIT(3, ord); DBG_UNIT(4, ord); }
            // ---- epilogue
            c.p.M = ph->M; c.p.N = ph->N; c.p.BN = ph->BN; c.p.act = ph->act; c.p.sample = ph->sample;
            c.p.acc_scale = ph->acc_scale; c.p.bias_scale = ph->bias_scale;
            c.p.sigma = ph->sigma; c.p.noise_sigma = ph->noise_sigma;
            c.p.out_mean_bf = ph->out_mean_bf; c.p.out_state_bf = ph->out_state_bf;
            c.p.out_f32 = ph->out_f32; c.p.ld_f32 = ph->ld_f32; c.p.split_stride = ph->split_stride;
            c.p.ais_a = ph->ais_a; c.p.ais_b = ph->ais_b; c.p.ais_next = ph->ais_next; c.p.ais_lin = ph->ais_lin; c.p.ais_logw = ph->ais_logw;
            c.p.ais_ct = ph->ais_b - ph->ais_a; c.p.ais_cd = ph->ais_next - 0.5f * (ph->ais_a + ph->ais_b);
            c.rng.k0 = L.k0; c.rng.k1 = L.k1; c.rng.tick = L.tick + ph->tick_off; c.rng.row0 = L.row0; c.rng.c2 = ph->rng_c2;
            c.m0 = (u.m_group * CL + crank) * BM + c.r0;
            c.n_blk = u.n_blk; c.split = u.split;
            switch (ph->mode) {
                case MODE_SIG_BERN_MEAN_STATE: epilogue_tile<MODE_SIG_BERN_MEAN_STATE>(c, acc); break;
                case MODE_SIG_BERN_STATE: epilogue_tile<MODE_SIG_BERN_STATE>(c, acc); break;
                case MODE_SIG_MEAN: epilogue_tile<MODE_SIG_MEAN>(c, acc); break;
                case MODE_RAW_F32: epilogue_tile<MODE_RAW_F32>(c, acc); break;
                case MODE_AIS_UNITS: epilogue_tile<MODE_AIS_UNITS>(c, acc); break;
                case MODE_AIS_UNITS_S: epilogue_tile<MODE_AIS_UNITS_S>(c, acc); break;
                case MODE_AIS_UNITS_G: epilogue_tile<MODE_AIS_UNITS_G>(c, acc); break;
                case MODE_AIS_STATE: epilogue_tile<MODE_AIS_STATE>(c, acc); break;
                default: epilogue_tile<MODE_GENERIC>(c, acc); break;
            }
            if (threadIdx.x == 0) DBG_UNIT(5, ord);
            // this warp's part of the unit is stored: the publisher warps make it visible to other SMs
            __syncwarp();
            if (lane == 0) mbar_arrive(&unit_bar[acc_st]);
            if (threadIdx.x == 0) DBG_MARK(4);
            if (++acc_st == ACC_STAGES) { acc_st = 0; acc_phase ^= 1; }
        }
    } else {
        regs_to_consumers();         // warp 8: no role
    }

    // no CTA may exit while its bulk stores can still read its shared memory (the publishers waited for them)
    __syncthreads();
    if (threadIdx.x == 0) { DBG_MARK(5); if (L.dbg && blockIdx.x == 0) L.dbg[7] = gtime(); }
}

// ------------------------------------------------------------------------------------------
// host side: tensor maps (driver entry point resolved at run time -> no libcuda link dependency)
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    if (!fn) throw Error(BM_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");
    return fn;
}

// 2-D map over a row-major bf16 matrix: dim0 = columns (contiguous), dim1 = rows; box = box0 x box1;
// 128-byte swizzle; out-of-range elements read as zero (ragged M/N/K need no padding in memory).
static CUtensorMap make_map(const TcMat& m, int box0, int box1) {
    typedef std::tuple<const void*, int, int, int, int, int> Key;
    static std::map<Key, CUtensorMap> cache;
    static std::mutex mu;
    Key key(m.ptr, m.rows, m.cols, m.ld, box0, box1);
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
    BM_REQUIRE(m.ptr != nullptr && (reinterpret_cast<uintptr_t>(m.ptr) & 15) == 0, "tensor-core operand must be 16-byte aligned");
    BM_REQUIRE(m.ld % 8 == 0 && m.ld >= m.cols, "tensor-core operand leading dimension must be a multiple of 8");
    CUtensorMap tm;
    const cuuint64_t gdim[2] = {(cuuint64_t)m.cols, (cuuint64_t)m.rows};
    const cuuint64_t gstride[1] = {(cuuint64_t)m.ld * 2};
    const cuuint32_t box[2] = {(cuuint32_t)box0, (cuuint32_t)box1};
    const cuuint32_t estr[2] = {1, 1};
    CUresult rc = encode_fn()(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<__nv_bfloat16*>(m.ptr), gdim, gstride, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (rc != CUDA_SUCCESS) throw Error(BM_ECUDA, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)rc));
    if (cache.size() > 4096) cache.clear();
    cache[key] = tm;
    return tm;
}

struct TilePick { int bn, cluster; };

static TilePick pick_tile(int N, int m_tiles, int splits, int chunks, int sms, int force_cluster) {
    // Tile width BN (64 or 128: whole 64-column wgmma blocks and TMA-store granules) and row grouping (CTAs
    // taking one 128-row block each, or pairs taking a 256-row group).  Cycle model per CTA:
    // waves * chunks * max(mma, ingest) + epilogue of the last tile, with the tensor cores at ~2048 bf16
    // MACs/clk per SM (989 TFLOP/s dense over 132 SMs) and L2 ingest assumed at ~32 B/clk per SM (not measured).
    TilePick best{64, 1};
    double best_cost = 1e30;
    for (int c = 1; c <= 2; ++c) {
        if (force_cluster && c != force_cluster) continue;
        if (!force_cluster && c == 2 && m_tiles < 2) break;
        const int slots = sms / c * c;                 // CTAs of the grid
        // (192 / 256 and widths of 16-column steps are reachable through force_bn only: a 256-wide tile leaves 3 ring stages)
        for (int bn = 64; bn <= 128; bn += 64) {
            const int nt = (N + bn - 1) / bn;
            const int m_groups = (m_tiles + c - 1) / c;
            const long units = (long)m_groups * c * nt * splits;
            const long waves = (units + slots - 1) / slots;
            const double mma = (double)BM * bn * BK / 2048.0;                     // cycles per K chunk
            const double ingest = (double)(A_BYTES + bn * BK * 2) / 32.0;         // bytes per chunk per SM / (B/clk)
            const double cost = (double)waves * chunks * (mma > ingest ? mma : ingest) + 12.0 * bn;
            if (cost < best_cost - 1e-9) { best_cost = cost; best.bn = bn; best.cluster = c; }
        }
    }
    return best;
}

static int epilogue_mode(const TcGemm& g) {
    if (g.ais_kind == 1) {
        const bool emit = g.out_state_bf != nullptr && g.sample == SMP_BERNOULLI;
        const float ct = fabsf(g.ais_b - g.ais_a), cd = fabsf(g.ais_next - 0.5f * (g.ais_a + g.ais_b));
        const bool close = ct <= AIS_MAX_CT && cd <= AIS_MAX_CD;
        if (emit && !g.ais_logw) return MODE_AIS_UNITS_S;
        if (emit && g.ais_logw && close) return MODE_AIS_UNITS;
        return MODE_AIS_UNITS_G;
    }
    if (g.ais_kind == 2) return MODE_AIS_STATE;
    if (g.sigma || g.noise_sigma) return MODE_GENERIC;
    const bool mb = g.out_mean_bf != nullptr, sb = g.out_state_bf != nullptr, f = g.out_f32 != nullptr;
    if (g.act == ACT_SIGMOID && g.sample == SMP_BERNOULLI && mb && sb && !f) return MODE_SIG_BERN_MEAN_STATE;
    if (g.act == ACT_SIGMOID && g.sample == SMP_BERNOULLI && !mb && sb && !f) return MODE_SIG_BERN_STATE;
    if (g.act == ACT_SIGMOID && g.sample == SMP_NONE && mb && !sb && !f) return MODE_SIG_MEAN;
    if (g.act == ACT_LINEAR && g.sample == SMP_NONE && !mb && !sb && f) return MODE_RAW_F32;
    return MODE_GENERIC;
}

// fills everything of a phase descriptor except the dataflow fields and the unit range
static void fill_phase(Ctx* ctx, const TcGemm& g, int cluster, TcPhase& ph) {
    TcPhaseLite& p = ph.l;
    BM_REQUIRE(g.M > 0 && g.N > 0 && g.n_pairs >= 1 && g.n_pairs <= 2, "bad tensor-core GEMM shape");
    memset(&ph, 0, sizeof(ph));
    p.M = g.M; p.N = g.N; p.n_pairs = g.n_pairs;
    const int m_tiles = (g.M + BM - 1) / BM;
    int chunks_total = 0;
    for (int i = 0; i < g.n_pairs; ++i) chunks_total += (g.K[i] + BK - 1) / BK;
    const int nsplit = g.splits > 0 ? g.splits : 1;
    TilePick tp = pick_tile(g.N, m_tiles, nsplit, (chunks_total + nsplit - 1) / nsplit, ctx->sm_count, cluster);
    if (g.force_bn > 0) tp.bn = g.force_bn;
    BM_REQUIRE(tp.cluster == cluster, "tile picker returned another row grouping");
    bool b_mn = false;
    for (int i = 0; i < g.n_pairs; ++i) b_mn = b_mn || g.b_t[i];
    const bool staged_out = g.out_mean_bf != nullptr || g.out_state_bf != nullptr;
    BM_REQUIRE(tp.bn % 16 == 0 && tp.bn >= 16 && tp.bn <= MAX_BN, "tile width must be a multiple of 16 columns, at most 256");
    BM_REQUIRE(!b_mn || tp.bn % 64 == 0, "an MN-major B operand needs tiles of whole 64-column boxes");
    BM_REQUIRE(!staged_out || tp.bn % 64 == 0, "ops with bf16 outputs need tiles of whole 64-column granules");
    p.BN = tp.bn;
    p.gran_per_tile = (p.BN + GRAN_COLS - 1) / GRAN_COLS;
    p.m_groups = (m_tiles + cluster - 1) / cluster;
    p.n_tiles = (g.N + p.BN - 1) / p.BN;
    p.splits = nsplit;
    p.split_stride = g.split_stride;
    for (int i = 0; i < 2; ++i) {
        const int j = i < g.n_pairs ? i : 0;
        p.chunks[i] = i < g.n_pairs ? (g.K[j] + BK - 1) / BK : 0;
        p.a_mn[i] = g.a_t[j]; p.b_mn[i] = g.b_t[j]; p.a_neg[i] = g.neg[j];
        p.a_row0[i] = g.a_row0[j]; p.a_k0[i] = g.a_k0[j]; p.a_batch[i] = g.a_batch[j];
        // K-major: box = 64 k x (128 | BN) rows; MN-major: box = 64 mn x 64 k
        ph.tmA[i] = g.a_t[j] ? make_map(g.A[j], 64, 64) : make_map(g.A[j], 64, BM);
        ph.tmB[i] = g.b_t[j] ? make_map(g.B[j], 64, 64) : make_map(g.B[j], 64, p.BN);
        BM_REQUIRE(i >= g.n_pairs || g.K[j] > 0, "tensor-core GEMM pair with K == 0");
    }
    BM_REQUIRE(p.splits <= chunks_total, "more K splits than K chunks");
    BM_REQUIRE(p.splits == 1 || (g.out_f32 && !g.out_mean_bf && !g.out_state_bf), "split-K writes fp32 partials only");
    p.acc_scale = g.acc_scale; p.bias_scale = g.bias_scale;
    p.bias = g.bias; p.sigma = g.sigma; p.noise_sigma = g.noise_sigma;
    p.act = g.act; p.sample = g.sample; p.mode = epilogue_mode(g);
    p.rng_c2 = g.rng.c2;
    p.ais_kind = g.ais_kind; p.ais_a = g.ais_a; p.ais_b = g.ais_b; p.ais_next = g.ais_next; p.ais_lin = g.ais_lin;
    p.ais_logw = g.ais_logw; p.tick_off = g.tick_off;
    if (g.ais_kind == 1)
        BM_REQUIRE(!g.sigma && !g.noise_sigma && g.act == ACT_LINEAR && !g.out_mean_bf && !g.out_f32 && g.splits <= 1 &&
                   g.acc_scale == 1.f && g.bias_scale == 1.f && (g.sample == SMP_NONE || g.sample == SMP_BERNOULLI),
                   "AIS unit op: linear accumulator, optional state output only");
    if (g.ais_kind == 2)
        BM_REQUIRE(!g.sigma && !g.noise_sigma && g.act == ACT_SIGMOID && g.sample == SMP_BERNOULLI && g.out_state_bf && !g.out_mean_bf &&
                   !g.out_f32 && g.splits <= 1 && g.bias, "AIS state op: sampled sigmoid states with a bias");
    p.out_mean_bf = g.out_mean_bf; p.ld_mean_bf = g.ld_mean_bf;
    p.out_state_bf = g.out_state_bf; p.ld_state_bf = g.ld_state_bf;
    p.out_f32 = g.out_f32; p.ld_f32 = g.ld_f32;
    // bf16 outputs leave the SM as TMA stores of (64 columns x 128 rows) granules, clipped to [M, N]
    if (g.out_mean_bf) { TcMat o; o.ptr = g.out_mean_bf; o.rows = g.M; o.cols = g.N; o.ld = g.ld_mean_bf; ph.tmOut[0] = make_map(o, GRAN_COLS, BM); }
    if (g.out_state_bf) { TcMat o; o.ptr = g.out_state_bf; o.rows = g.M; o.cols = g.N; o.ld = g.ld_state_bf; ph.tmOut[1] = make_map(o, GRAN_COLS, BM); }
    BM_REQUIRE(!g.out_mean_bf || (g.ld_mean_bf % 8 == 0), "bf16 output leading dimension must be a multiple of 8");
    BM_REQUIRE(!g.out_state_bf || (g.ld_state_bf % 8 == 0), "bf16 output leading dimension must be a multiple of 8");
}

// The ops' descriptors (minus tensor maps) go to constant memory, stream-ordered before the launch;
// skipped when the bank already holds exactly this image (the common case: the same program every step).
static void upload_ops(Ctx* ctx, const TcPhase* ph, int n) {
    struct Bank { std::vector<unsigned char> image; cudaStream_t user = nullptr; };
    static std::map<int, Bank> banks;                             // constant memory is per device
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    Bank& bank = banks[ctx->device];
    // another context of this device (another stream) may still be running a kernel that reads the bank: wait for it
    // before the bank changes hands
    if (bank.user && bank.user != ctx->stream) BM_CUDA(cudaStreamSynchronize(bank.user));
    bank.user = ctx->stream;
    std::vector<unsigned char>& current = bank.image;
    std::vector<unsigned char> img((size_t)n * sizeof(TcPhaseLite));
    for (int i = 0; i < n; ++i) memcpy(img.data() + (size_t)i * sizeof(TcPhaseLite), &ph[i].l, sizeof(TcPhaseLite));
    if (img.size() <= current.size() && memcmp(img.data(), current.data(), img.size()) == 0) return;
    BM_CUDA(cudaMemcpyToSymbolAsync(c_ph, img.data(), img.size(), 0, cudaMemcpyHostToDevice, ctx->stream));
    if (current.size() < img.size()) current.resize(img.size());
    memcpy(current.data(), img.data(), img.size());
}

static void do_launch(Ctx* ctx, TcLaunch& L, int cluster, double flops, int max_bn) {
    static bool attr_set[64] = {false};                         // function attributes are per device
    if (!attr_set[ctx->device & 63]) {
        BM_CUDA(cudaFuncSetAttribute(tc_program_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        BM_CUDA(cudaFuncSetAttribute(tc_program_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        attr_set[ctx->device & 63] = true;
    }
    // ring stages sized for the widest tile of the launch: narrower tiles buy a deeper pipeline
    L.stage_bytes = A_BYTES + max_bn * BK * 2;
    L.stage_bytes = (L.stage_bytes + 1023) & ~1023;           // 128B-swizzle atoms are 1024-byte aligned
    L.stages = RING_BYTES / L.stage_bytes;
    if (L.stages > MAX_STAGES) L.stages = MAX_STAGES;
    { const char* e = getenv("BM_TC_STAGES"); if (e && atoi(e) >= 2 && atoi(e) <= L.stages) L.stages = atoi(e); }
    const int max_groups = ctx->sm_count / cluster;
    // programs address pairs by number (TcPhaseLite::pair_begin/pair_count): launch all of them
    const int n_groups = L.n_phases ? max_groups : (L.total_units < max_groups ? L.total_units : max_groups);
    const int n_ctas = n_groups * cluster;
    // The CTAs of a pair share nothing, so the grid is launched as clusters of one CTA: a pair never has to fit into
    // one GPC, and the residency question below counts single CTAs.
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(n_ctas); lc.blockDim = dim3(TC_THREADS); lc.dynamicSmemBytes = SMEM_BYTES; lc.stream = ctx->stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    lc.attrs = at; lc.numAttrs = 1;
    if (L.n_phases) {
        // a program's CTAs wait for each other through counters in global memory: all of them must be resident at once.  Ask the
        // runtime once per device (a GPU shared through MPS / MIG, or a part with fewer SMs than it reports, would otherwise only
        // show up as the kernel's 4-second trap); BM_TC_SKIP_RESIDENCY_CHECK=1 trusts the device properties instead.
        static int resident[64] = {0};
        int& r = resident[ctx->device & 63];
        if (r == 0) {
            const char* e = getenv("BM_TC_SKIP_RESIDENCY_CHECK");
            int n = 0;
            if (e && atoi(e) == 1) r = -1;
            else if (cudaOccupancyMaxActiveClusters(&n, cluster == 2 ? (const void*)tc_program_kernel<2> : (const void*)tc_program_kernel<1>, &lc) == cudaSuccess) r = n > 0 ? n : -2;
            else { cudaGetLastError(); r = -1; }
            if (getenv("BM_TC_DEBUG_RESIDENCY"))
                fprintf(stderr, "[bm] device %d: cudaOccupancyMaxActiveClusters(tc_program_kernel<%d>) = %d, the program grid has %d CTAs\n",
                        ctx->device, cluster, n, n_ctas);
        }
        BM_REQUIRE(r == -1 || r >= n_ctas,
                   "the device cannot hold all CTA clusters of a dataflow program at once (cudaOccupancyMaxActiveClusters); it would deadlock");
    }
    if (ctx->profile_tc) BM_CUDA(cudaEventRecord(profile_event(ctx), ctx->stream));
    if (cluster == 2) BM_CUDA(cudaLaunchKernelEx(&lc, tc_program_kernel<2>, L));
    else BM_CUDA(cudaLaunchKernelEx(&lc, tc_program_kernel<1>, L));
    if (ctx->profile_tc) {
        BM_CUDA(cudaEventRecord(profile_event(ctx), ctx->stream));
        ctx->prof_flops += flops;       // algorithmic FLOPs (no padding counted)
        ctx->prof_launches++;
    }
    count_launch(ctx);
}

static double gemm_flops(const TcGemm& g) {
    double k_total = 0.0;
    for (int i = 0; i < g.n_pairs; ++i) k_total += g.K[i];
    return 2.0 * g.M * g.N * k_total;
}

void launch_tc_gemm(Ctx* ctx, const TcGemm& g) {
    const int m_tiles = (g.M + BM - 1) / BM;
    int cluster = g.force_cluster > 0 ? g.force_cluster : (m_tiles >= 2 ? 2 : 1);
    BM_REQUIRE(cluster == 1 || cluster == 2, "cluster must be 1 or 2");
    TcLaunch L;
    memset(&L, 0, sizeof(L));
    fill_phase(ctx, g, cluster, L.inl);
    L.inl.l.n_units = L.inl.l.m_groups * L.inl.l.n_tiles * L.inl.l.splits;
    L.total_units = L.inl.l.n_units;
    {   // every CTA pair (or CTA) of the grid takes part
        const int max_clusters = ctx->sm_count / cluster;
        L.inl.l.pair_begin = 0;
        L.inl.l.pair_count = L.total_units < max_clusters ? L.total_units : max_clusters;
    }
    L.k0 = g.rng.k0; L.k1 = g.rng.k1; L.tick = g.rng.tick; L.row0 = g.rng.row0;
    L.dbg = g.dbg;
    L.mant_mask = 0x007FFFFFu; L.one_bits = 0x3F800000u;
    L.epoch = 1; L.poll_ns = 64; L.epi_ns = 128;
    upload_ops(ctx, &L.inl, 1);
    do_launch(ctx, L, cluster, gemm_flops(g), L.inl.l.BN);
}

int tc_plan_units(Ctx* ctx, const TcGemm& g) {
    TcPhase ph;
    fill_phase(ctx, g, 2, ph);
    return ph.l.m_groups * ph.l.n_tiles * ph.l.splits;
}

TcProgram::~TcProgram() {
    if (dev_phases) cudaFree(dev_phases);
    if (dev_counters) cudaFree(dev_counters);
}

void launch_tc_program(Ctx* ctx, TcProgram& prog, RngKey rng, int batch_row) {
    const int n = (int)prog.ops.size();
    BM_REQUIRE(n >= 1 && n <= MAX_PHASES, "a program holds 1..96 ops");
    const int cluster = 2;            // programs always run on CTA pairs (all CTAs walk one unit list)
    std::vector<unsigned char> image((size_t)n * sizeof(TcPhase));
    TcPhase* ph = reinterpret_cast<TcPhase*>(image.data());
    // counters: per op one int per row-block group (unit level) + one per (row-block group, tile, granule)
    size_t n_ctr = 0;
    std::vector<size_t> ctr_off(n), cctr_off(n);
    int unit = 0;
    double flops = 0.0;
    for (int i = 0; i < n; ++i) {
        fill_phase(ctx, prog.ops[i], cluster, ph[i]);
        ph[i].l.n_units = ph[i].l.m_groups * ph[i].l.n_tiles * ph[i].l.splits;
        unit += ph[i].l.n_units;
        ctr_off[i] = n_ctr;
        n_ctr += (size_t)ph[i].l.m_groups;
        cctr_off[i] = n_ctr;
        n_ctr += (size_t)ph[i].l.m_groups * ph[i].l.n_tiles * ph[i].l.gran_per_tile;
        flops += gemm_flops(prog.ops[i]);
    }
    if (n_ctr > prog.n_counters) {
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        if (prog.dev_counters) cudaFree(prog.dev_counters);
        BM_CUDA(cudaMalloc(&prog.dev_counters, n_ctr * sizeof(int)));
        prog.n_counters = n_ctr;
        prog.host_image.clear();
        prog.epoch = 0;
    }
    // pair assignment: chain ops on pairs [0, P), spare-lane ops on [P, total), the rest on all pairs
    {
        const int total = ctx->sm_count / cluster;
        int P = 0;
        for (int i = 0; i < n; ++i) if (prog.ops[i].lane == LANE_CHAIN) P = std::max(P, ph[i].l.n_units);
        if (P > total || P == 0) P = total;
        for (int i = 0; i < n; ++i) {
            int lane = prog.ops[i].lane;
            if (lane == LANE_SPARE && total - P < 1) lane = LANE_ALL;
            ph[i].l.pair_begin = lane == LANE_SPARE ? P : 0;
            ph[i].l.pair_count = lane == LANE_CHAIN ? P : (lane == LANE_SPARE ? total - P : total);
        }
    }
    static int chunk_deps = -1;
    if (chunk_deps < 0) { const char* e = getenv("BM_TC_CHUNK_DEPS"); chunk_deps = e ? atoi(e) : 1; }
    for (int i = 0; i < n; ++i) {
        const TcGemm& g = prog.ops[i];
        ph[i].l.done_ctr = prog.dev_counters + ctr_off[i];
        ph[i].l.n_deps = g.n_deps;
        for (int d = 0; d < g.n_deps; ++d) {
            const int j = g.dep[d];
            BM_REQUIRE(j >= 0 && j < i, "a program op may only depend on earlier ops");
            ph[i].l.dep_ctr[d] = prog.dev_counters + ctr_off[j];
            ph[i].l.dep_need[d] = ph[j].l.n_tiles * ph[j].l.splits * cluster * 2;  // both publishers of every CTA, per unit
            if (g.dep_all[d]) ph[i].l.dep_groups[d] = ph[j].l.m_groups;
            else {
                ph[i].l.dep_groups[d] = 0;
                BM_REQUIRE(ph[i].l.m_groups <= ph[j].l.m_groups, "row-block dependency on an op with fewer row blocks");
                // granule-level dataflow: this op's (K-major) A operand is op j's output (K = its N); only
                // for the first such dependency, single-pair ops without split-K
                const TcPhaseLite& pj = ph[j].l;
                const int kchunks = ph[i].l.chunks[0];
                // (the kernel's wait loop skips the unit-level wait of EVERY same-row-block dependency of an op that follows
                // granules: only an op whose single such dependency is this one may do so)
                int same_row_deps = 0;
                for (int q = 0; q < g.n_deps; ++q) same_row_deps += g.dep_all[q] ? 0 : 1;
                if (chunk_deps && d == 0 && same_row_deps == 1 && g.n_pairs == 1 && !g.a_t[0] && ph[i].l.splits == 1 && pj.splits == 1 &&
                    kchunks <= MAX_KCHUNKS && g.K[0] == pj.N && pj.n_tiles * pj.gran_per_tile <= 255) {
                    ph[j].l.chunk_ctr = prog.dev_counters + cctr_off[j];
                    ph[i].l.dep_chunk_ctr = prog.dev_counters + cctr_off[j];
                    ph[i].l.dep_gran_row = pj.n_tiles * pj.gran_per_tile;
                    ph[i].l.dep_chunk_need = cluster;              // the publisher of each CTA of the producing pair
                    // K chunk c = columns [64c, 64c+64) of the producer's output: the granule(s) holding its
                    // first and last column; consumed in the order the producer's epilogues finish them
                    std::vector<std::pair<int, int>> order;
                    for (int c = 0; c < kchunks; ++c) {
                        const int col_a = 64 * c, col_b = std::min(64 * c + 63, pj.N - 1);
                        const int ta = col_a / pj.BN, tb = col_b / pj.BN;
                        const int ga = (col_a - ta * pj.BN) / GRAN_COLS, gb = (col_b - tb * pj.BN) / GRAN_COLS;
                        ph[i].l.k_dep_a[c] = (unsigned char)(ta * pj.gran_per_tile + ga);
                        ph[i].l.k_dep_b[c] = (unsigned char)(tb * pj.gran_per_tile + gb);
                        order.push_back(std::make_pair(std::max(ga, gb), c));
                    }
                    std::stable_sort(order.begin(), order.end());
                    for (int c = 0; c < kchunks; ++c) ph[i].l.k_order[c] = (unsigned char)order[c].second;
                }
            }
        }
    }
    // descriptors live in device memory; re-uploaded only when they changed (buffers and shapes are
    // stable across steps; the per-step values -- tick, batch cursor -- travel in the kernel parameters)
    if (image.size() != prog.host_image.size() || memcmp(image.data(), prog.host_image.data(), image.size()) != 0) {
        if (image.size() > prog.dev_phases_bytes) {
            BM_CUDA(cudaStreamSynchronize(ctx->stream));   // a running launch may still read the old allocation
            if (prog.dev_phases) cudaFree(prog.dev_phases);
            BM_CUDA(cudaMalloc(&prog.dev_phases, image.size()));
            prog.dev_phases_bytes = image.size();
        }
        // stream-ordered: the copy runs after every earlier launch of this stream has finished reading the descriptors (the
        // pageable source is staged before the call returns) -- no host synchronisation between the launches of a ladder
        BM_CUDA(cudaMemcpyAsync(prog.dev_phases, image.data(), image.size(), cudaMemcpyHostToDevice, ctx->stream));
        prog.host_image = image;
        prog.epoch = 0;                                   // another op list: other arrival counts per launch
    }
    if (prog.epoch == 0 || prog.epoch >= (1 << 20)) {
        BM_CUDA(cudaMemsetAsync(prog.dev_counters, 0, prog.n_counters * sizeof(int), ctx->stream));
        prog.epoch = 0;
    }
    // (the epoch is only advanced once the launch has been accepted: after a refused launch the counters of the
    //  program are re-zeroed before its next launch instead of being waited on one epoch behind)
    TcLaunch L;
    memset(&L, 0, sizeof(L));
    L.phases = reinterpret_cast<const TcPhase*>(prog.dev_phases);
    L.n_phases = n;
    L.total_units = unit;
    L.k0 = rng.k0; L.k1 = rng.k1; L.tick = rng.tick; L.row0 = rng.row0;
    L.batch_row = batch_row;
    L.epoch = prog.epoch + 1;
    { static int pn = -1, en = -1;
      if (pn < 0) { const char* e = getenv("BM_TC_POLL_NS"); pn = e ? atoi(e) : 64; }
      if (en < 0) { const char* e = getenv("BM_TC_EPI_NS"); en = e ? atoi(e) : 128; }
      L.poll_ns = pn; L.epi_ns = en; }
    { static int fl = -1; if (fl < 0) { const char* e = getenv("BM_TC_FLAGS"); fl = e ? atoi(e) : 3; } L.flags = fl; }
    L.mant_mask = 0x007FFFFFu; L.one_bits = 0x3F800000u;
    static unsigned long long* dbg_buf = nullptr;
    static int dbg_left = -1;
    if (dbg_left < 0) { const char* e = getenv("BM_TC_PROGRAM_TIMELINE"); dbg_left = e ? atoi(e) : 0; }
    const bool dbg = dbg_left > 0;
    if (dbg) {
        if (!dbg_buf) BM_CUDA(cudaMalloc(&dbg_buf, 1024 * sizeof(unsigned long long)));
        BM_CUDA(cudaMemsetAsync(dbg_buf, 0, 1024 * sizeof(unsigned long long), ctx->stream));
        L.dbg = dbg_buf;
    }
    int max_bn = 16;
    for (int i = 0; i < n; ++i) max_bn = std::max(max_bn, ph[i].l.BN);
    try {
        upload_ops(ctx, ph, n);
        do_launch(ctx, L, cluster, flops, max_bn);
        ++prog.epoch;
    } catch (...) {
        prog.epoch = 0;
        throw;
    }
    if (dbg) {
        --dbg_left;
        unsigned long long h[1024];
        BM_CUDA(cudaStreamSynchronize(ctx->stream));
        BM_CUDA(cudaMemcpy(h, dbg_buf, sizeof(h), cudaMemcpyDeviceToHost));
        fprintf(stderr, "program timeline (SM cycles, CTA 0): setup=%llu exit=%llu wall=%llu ns, %d units total\n",
                h[1] - h[0], h[5] - h[0], h[7] - h[6], unit);
        fprintf(stderr, "  unit 1 tma_issue:");
        for (int i = 0; i < 24 && h[8 + i]; ++i) fprintf(stderr, " %llu", h[8 + i] - h[0]);
        fprintf(stderr, "\n  ord: start dep_ok mma_first mma_done epi_start epi_done published\n");
        for (int o = 0; o < 24 && h[64 + o * 8]; ++o) {
            fprintf(stderr, "  %2d:", o);
            for (int k = 0; k < 7; ++k) fprintf(stderr, " %7llu", h[64 + o * 8 + k] ? h[64 + o * 8 + k] - h[0] : 0ull);
            fprintf(stderr, "\n");
        }
    }
}

}  // namespace bm
