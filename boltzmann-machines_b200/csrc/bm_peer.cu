// Data-parallel CD step over NVLink peer memory: see bm_peer.h.
#include "bm_peer.h"
#include <string.h>
#include <stdlib.h>
#include <vector>
#include <stdio.h>

namespace bm {

namespace {

constexpr unsigned long long PEER_HANG_NS = 4000000000ull;      // a peer that never arrives: trap instead of spinning for ever

__device__ __forceinline__ int ld_acquire_sys(const int* p) {
    int v; asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release_sys(int* p, int v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long now_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void wait_flag(const int* p, int want) {
    unsigned n = 0; unsigned long long t0 = 0;
    while (ld_acquire_sys(p) < want) {
        __nanosleep(200);
        if ((++n & 0x3FFu) == 0) {
            const unsigned long long t = now_ns();
            if (t0 == 0) t0 = t; else if (t - t0 > PEER_HANG_NS) __trap();
        }
    }
}
// the block that finishes last publishes `flag[rank] = step` on every rank (threadFenceReduction pattern, system scope:
// every block's stores -- local and to peers -- are fenced before its arrival on the counter)
__device__ __forceinline__ void publish_when_all_blocks_done(const DpStep& s, unsigned int* counter, int flag_off) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned old = atomicAdd(counter, 1u);
        if (old == gridDim.x - 1) {
            atomicExch(counter, 0u);
            __threadfence_system();
            for (int q = 0; q < s.nranks; ++q) st_release_sys(s.peer[q].flags + flag_off + s.rank, s.step);
        }
    }
}

__global__ void __launch_bounds__(256) dp_push_kernel(const __grid_constant__ DpStep s) {
    const int V = s.V, H = s.H;
    const size_t n4 = (size_t)V * H / 4;
    for (size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += (size_t)gridDim.x * blockDim.x) {
        const size_t i = i4 * 4;
        float4 a = *reinterpret_cast<const float4*>(s.part + i);
        for (int k = 1; k < s.splits; ++k) {
            const float4 b = *reinterpret_cast<const float4*>(s.part + (size_t)k * s.stride + i);
            a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        const int v = (int)(i / (size_t)H), h = (int)(i % (size_t)H);
        const int owner = v / s.rows_per;
        float* dst = s.peer[owner].inbox + (size_t)s.rank * s.shard_elems + (size_t)(v - owner * s.rows_per) * H + h;
        *reinterpret_cast<float4*>(dst) = a;
    }
    // rows srow and srow + 1 of the slices (2H contiguous values), then sum(X - v_k): to every rank
    const int n_small = 2 * H + V;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_small; j += gridDim.x * blockDim.x) {
        float x = 0.f;
        if (j < 2 * H) { const size_t off = (size_t)s.srow * H + j; for (int k = 0; k < s.splits; ++k) x += s.part[(size_t)k * s.stride + off]; }
        else { for (int k = 0; k < s.vsplits; ++k) x += s.vpart[(size_t)k * s.vstride + (j - 2 * H)]; }
        for (int q = 0; q < s.nranks; ++q) s.peer[q].small[(size_t)s.rank * s.small_len + j] = x;
    }
    publish_when_all_blocks_done(s, s.counter, 0);
}

__global__ void __launch_bounds__(256) dp_update_kernel(const __grid_constant__ DpStep s, unsigned w_blocks, int local_only) {
    if (threadIdx.x < s.nranks) wait_flag(s.peer[s.rank].flags + threadIdx.x, s.step);        // every rank's push has landed here
    __syncthreads();
    const int V = s.V, H = s.H, R = s.nranks;
    const PeerView& me = s.peer[s.rank];
    if (blockIdx.x < w_blocks) {
        const int r0 = s.rank * s.rows_per;
        const int r1 = min(V, r0 + s.rows_per);
        const size_t n = r1 > r0 ? (size_t)(r1 - r0) * H : 0;
        const size_t li = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (li < n) {
            float4 g = *reinterpret_cast<const float4*>(me.inbox + li);
            for (int r = 1; r < R; ++r) {
                const float4 b = *reinterpret_cast<const float4*>(me.inbox + (size_t)r * s.shard_elems + li);
                g.x += b.x; g.y += b.y; g.z += b.z; g.w += b.w;
            }
            const size_t i = (size_t)r0 * H + li;
            const int h = (int)(i % (size_t)H);
            const size_t v = i / (size_t)H;
            float pen[4] = {0.f, 0.f, 0.f, 0.f};
            if (s.cost != 0.f) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float qs = 0.f;
                    for (int r = 0; r < R; ++r) qs += me.small[(size_t)r * s.small_len + H + h + j];
                    const float q = s.damp * s.q_old[h + j] + (1.0f - s.damp) * (-qs);
                    pen[j] = s.cost * (q - s.target);
                }
            }
            const float4 w4 = *reinterpret_cast<const float4*>(me.W + i), d4 = *reinterpret_cast<const float4*>(me.dW + i);
            const float gg[4] = {g.x, g.y, g.z, g.w}, w[4] = {w4.x, w4.y, w4.z, w4.w}, d0[4] = {d4.x, d4.y, d4.z, d4.w};
            float d[4], wn[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                d[j] = s.lr * (s.mom * d0[j] + (gg[j] / s.n_div - s.l2 * w[j] - pen[j]));       // base_rbm.py:449, 462, 467
                wn[j] = w[j] + d[j];                                                             // :468
            }
            __nv_bfloat162 lo = __floats2bfloat162_rn(wn[0], wn[1]), hi = __floats2bfloat162_rn(wn[2], wn[3]);
            uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
            const float4 dv = make_float4(d[0], d[1], d[2], d[3]), wv = make_float4(wn[0], wn[1], wn[2], wn[3]);
            for (int q = 0; q < R; ++q) {                        // the all-gather: one writer per row, every copy
                if (local_only && q != s.rank) continue;         // (split variant: dp_scatter_kernel copies the rows out)
                const PeerView& pq = s.peer[q];
                // what every rank's next program reads is the bf16 shadow; the fp32 master and the momentum rows stay with their
                // owner unless s.replicate_fp32 (peers pull them when something reads them: dp_pull_kernel)
                if (q == s.rank || s.replicate_fp32) {
                    *reinterpret_cast<float4*>(pq.dW + i) = dv;
                    *reinterpret_cast<float4*>(pq.W + i) = wv;
                }
                *reinterpret_cast<uint2*>(pq.Wb + v * (size_t)s.ldwb + h) = pk;
            }
        }
    } else {
        // biases and sparsity statistics: every rank computes the same sums in the same order
        const int i = (int)(blockIdx.x - w_blocks) * blockDim.x + threadIdx.x;
        if (i < H) {
            float ds = 0.f, qs = 0.f;
            for (int r = 0; r < R; ++r) { ds += me.small[(size_t)r * s.small_len + i]; qs += me.small[(size_t)r * s.small_len + H + i]; }
            const float q = s.damp * s.q_old[i] + (1.0f - s.damp) * (-qs);                     // :457-459
            s.q_new[i] = q;
            const float pen = s.cost * (q - s.target);
            s.pen[i] = pen;
            const float dd = s.lr * (s.mom * s.dhb[i] + (ds / s.n_div - pen));                  // :453, :461, :473-474
            s.dhb[i] = dd;
            s.hb[i] += dd;
        }
        if (i < V) {
            float vs = 0.f;
            for (int r = 0; r < R; ++r) vs += me.small[(size_t)r * s.small_len + 2 * H + i];
            const float dd = s.lr * (s.mom * s.dvb[i] + vs / s.n_div);                          // :451, :470-471
            s.dvb[i] = dd;
            s.vb[i] += dd;
        }
    }
    if (!local_only) publish_when_all_blocks_done(s, s.counter + 1, MAX_PEERS);
}

// split variant of the all-gather: every block of the grid copies a piece of this rank's freshly updated rows (fp32 W, momentum,
// bf16 shadow) to ONE peer (blockIdx.y), so that the stores to the 7 peers come from all SMs instead of from the shard's own blocks
__global__ void __launch_bounds__(256) dp_scatter_kernel(const __grid_constant__ DpStep s) {
    const int V = s.V, H = s.H;
    const int q = (int)blockIdx.y >= s.rank ? (int)blockIdx.y + 1 : (int)blockIdx.y;      // the peers other than this rank
    const int r0 = s.rank * s.rows_per;
    const int r1 = min(V, r0 + s.rows_per);
    const size_t n4 = r1 > r0 ? (size_t)(r1 - r0) * H / 4 : 0;
    const PeerView& me = s.peer[s.rank];
    const PeerView& pq = s.peer[q];
    for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < n4; j += (size_t)gridDim.x * blockDim.x) {
        const size_t i = (size_t)r0 * H + j * 4;
        const int h = (int)(i % (size_t)H);
        const size_t v = i / (size_t)H;
        *reinterpret_cast<float4*>(pq.W + i) = *reinterpret_cast<const float4*>(me.W + i);
        *reinterpret_cast<float4*>(pq.dW + i) = *reinterpret_cast<const float4*>(me.dW + i);
        *reinterpret_cast<uint2*>(pq.Wb + v * (size_t)s.ldwb + h) = *reinterpret_cast<const uint2*>(me.Wb + v * (size_t)s.ldwb + h);
    }
    // (gridDim.x * gridDim.y blocks arrive on the counter)
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned old = atomicAdd(s.counter + 1, 1u);
        if (old == gridDim.x * gridDim.y - 1) {
            atomicExch(s.counter + 1, 0u);
            __threadfence_system();
            for (int p = 0; p < s.nranks; ++p) st_release_sys(s.peer[p].flags + MAX_PEERS + s.rank, s.step);
        }
    }
}

// ---- the same two kernels with the transfers as BULK asynchronous copies (shared memory -> peer global memory) -------------
// An alternative (BM_PEER_BULK=1, off by default): a block sums / updates whole rows into shared memory and one thread hands
// them to the copy engine of its SM (cp.async.bulk.global.shared::cta: one transaction of n_hidden * 4 bytes per row and
// destination), the local copy included.  Its speed against the plain stores is not measured on H100s.
__device__ __forceinline__ uint32_t peer_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bulk_store(void* gdst, const void* ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(peer_smem_u32(ssrc)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_smem_to_async_proxy() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__global__ void __launch_bounds__(256) dp_push_bulk_kernel(const __grid_constant__ DpStep s, int rows_per_block) {
    extern __shared__ __align__(128) unsigned char dp_smem[];
    float* buf = reinterpret_cast<float*>(dp_smem);                      // [rows_per_block][H]
    const int V = s.V, H = s.H;
    const int n_chunks = (V + rows_per_block - 1) / rows_per_block;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const int v0 = c * rows_per_block, v1 = min(V, v0 + rows_per_block);
        const int n4 = (v1 - v0) * H / 4;
        for (int j = threadIdx.x; j < n4; j += blockDim.x) {
            const size_t i = (size_t)v0 * H + (size_t)j * 4;
            float4 a = *reinterpret_cast<const float4*>(s.part + i);
            for (int k = 1; k < s.splits; ++k) {
                const float4 b = *reinterpret_cast<const float4*>(s.part + (size_t)k * s.stride + i);
                a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
            }
            *reinterpret_cast<float4*>(buf + (size_t)j * 4) = a;
        }
        fence_smem_to_async_proxy();
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int v = v0; v < v1; ++v) {
                const int owner = v / s.rows_per;
                bulk_store(s.peer[owner].inbox + (size_t)s.rank * s.shard_elems + (size_t)(v - owner * s.rows_per) * H,
                           buf + (size_t)(v - v0) * H, (uint32_t)H * 4u);
            }
            bulk_commit_group();
            bulk_wait_read_all();                                            // the buffer may be rewritten
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) bulk_wait_all();                                   // ... and the rows have arrived
    const int n_small = 2 * H + V;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_small; j += gridDim.x * blockDim.x) {
        float x = 0.f;
        if (j < 2 * H) { const size_t off = (size_t)s.srow * H + j; for (int k = 0; k < s.splits; ++k) x += s.part[(size_t)k * s.stride + off]; }
        else { for (int k = 0; k < s.vsplits; ++k) x += s.vpart[(size_t)k * s.vstride + (j - 2 * H)]; }
        for (int q = 0; q < s.nranks; ++q) s.peer[q].small[(size_t)s.rank * s.small_len + j] = x;
    }
    publish_when_all_blocks_done(s, s.counter, 0);
}

__global__ void __launch_bounds__(256) dp_update_bulk_kernel(const __grid_constant__ DpStep s, unsigned w_blocks, int rows_per_block) {
    extern __shared__ __align__(128) unsigned char dp_smem[];
    if (threadIdx.x < s.nranks) wait_flag(s.peer[s.rank].flags + threadIdx.x, s.step);        // every rank's push has landed here
    __syncthreads();
    const int V = s.V, H = s.H, R = s.nranks;
    const PeerView& me = s.peer[s.rank];
    if (blockIdx.x < w_blocks) {
        float* Ws = reinterpret_cast<float*>(dp_smem);                                   // [rows_per_block][H] new weights
        float* Ds = Ws + (size_t)rows_per_block * H;                                     // new momentum
        __nv_bfloat16* Bs = reinterpret_cast<__nv_bfloat16*>(Ds + (size_t)rows_per_block * H);   // bf16 shadow
        const int r0 = s.rank * s.rows_per;
        const int r1 = min(V, r0 + s.rows_per);
        const int n_chunks = r1 > r0 ? (r1 - r0 + rows_per_block - 1) / rows_per_block : 0;
        for (int c = blockIdx.x; c < n_chunks; c += (int)w_blocks) {
            const int v0 = r0 + c * rows_per_block, v1 = min(r1, v0 + rows_per_block);
            const int n4 = (v1 - v0) * H / 4;
            for (int j = threadIdx.x; j < n4; j += blockDim.x) {
                const size_t i = (size_t)v0 * H + (size_t)j * 4;
                const size_t li = i - (size_t)r0 * H;
                const int h = (int)(i % (size_t)H);
                float4 g = *reinterpret_cast<const float4*>(me.inbox + li);
                for (int r = 1; r < R; ++r) {
                    const float4 b = *reinterpret_cast<const float4*>(me.inbox + (size_t)r * s.shard_elems + li);
                    g.x += b.x; g.y += b.y; g.z += b.z; g.w += b.w;
                }
                float pen[4] = {0.f, 0.f, 0.f, 0.f};
                if (s.cost != 0.f) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float qs = 0.f;
                        for (int r = 0; r < R; ++r) qs += me.small[(size_t)r * s.small_len + H + h + k];
                        const float q = s.damp * s.q_old[h + k] + (1.0f - s.damp) * (-qs);
                        pen[k] = s.cost * (q - s.target);
                    }
                }
                const float4 w4 = *reinterpret_cast<const float4*>(me.W + i), d4 = *reinterpret_cast<const float4*>(me.dW + i);
                const float gg[4] = {g.x, g.y, g.z, g.w}, w[4] = {w4.x, w4.y, w4.z, w4.w}, d0[4] = {d4.x, d4.y, d4.z, d4.w};
                float d[4], wn[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    d[k] = s.lr * (s.mom * d0[k] + (gg[k] / s.n_div - s.l2 * w[k] - pen[k]));       // base_rbm.py:449, 462, 467
                    wn[k] = w[k] + d[k];                                                             // :468
                }
                *reinterpret_cast<float4*>(Ws + (size_t)j * 4) = make_float4(wn[0], wn[1], wn[2], wn[3]);
                *reinterpret_cast<float4*>(Ds + (size_t)j * 4) = make_float4(d[0], d[1], d[2], d[3]);
                __nv_bfloat162 lo = __floats2bfloat162_rn(wn[0], wn[1]), hi = __floats2bfloat162_rn(wn[2], wn[3]);
                uint2 pk; pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
                *reinterpret_cast<uint2*>(Bs + (size_t)j * 4) = pk;
            }
            fence_smem_to_async_proxy();
            __syncthreads();                        // (also: every thread's reads of the old rows precede the copies below)
            if (threadIdx.x == 0) {
                const uint32_t bytes = (uint32_t)(v1 - v0) * (uint32_t)H * 4u;
                for (int q = 0; q < R; ++q) {        // the all-gather, this rank's own copy included: one writer per row
                    const PeerView& pq = s.peer[q];
                    bulk_store(pq.W + (size_t)v0 * H, Ws, bytes);
                    bulk_store(pq.dW + (size_t)v0 * H, Ds, bytes);
                    for (int v = v0; v < v1; ++v) bulk_store(pq.Wb + (size_t)v * s.ldwb, Bs + (size_t)(v - v0) * H, (uint32_t)H * 2u);
                }
                bulk_commit_group();
                bulk_wait_read_all();
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) bulk_wait_all();
    } else {
        // biases and sparsity statistics: every rank computes the same sums in the same order
        const int i = (int)(blockIdx.x - w_blocks) * blockDim.x + threadIdx.x;
        if (i < H) {
            float ds = 0.f, qs = 0.f;
            for (int r = 0; r < R; ++r) { ds += me.small[(size_t)r * s.small_len + i]; qs += me.small[(size_t)r * s.small_len + H + i]; }
            const float q = s.damp * s.q_old[i] + (1.0f - s.damp) * (-qs);                     // :457-459
            s.q_new[i] = q;
            const float pen = s.cost * (q - s.target);
            s.pen[i] = pen;
            const float dd = s.lr * (s.mom * s.dhb[i] + (ds / s.n_div - pen));                  // :453, :461, :473-474
            s.dhb[i] = dd;
            s.hb[i] += dd;
        }
        if (i < V) {
            float vs = 0.f;
            for (int r = 0; r < R; ++r) vs += me.small[(size_t)r * s.small_len + 2 * H + i];
            const float dd = s.lr * (s.mom * s.dvb[i] + vs / s.n_div);                          // :451, :470-471
            s.dvb[i] = dd;
            s.vb[i] += dd;
        }
    }
    publish_when_all_blocks_done(s, s.counter + 1, MAX_PEERS);
}

// the fp32 master and momentum rows of the OTHER ranks' shards, read from their owners (who are not in an update: an update
// needs this rank's push of the same step)
__global__ void __launch_bounds__(256) dp_pull_kernel(const __grid_constant__ DpStep s) {
    const int V = s.V, H = s.H;
    const size_t n4 = (size_t)V * H / 4;
    const PeerView& me = s.peer[s.rank];
    for (size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += (size_t)gridDim.x * blockDim.x) {
        const size_t i = i4 * 4;
        const int owner = (int)(i / (size_t)H) / s.rows_per;
        if (owner == s.rank) continue;
        *reinterpret_cast<float4*>(me.W + i) = *reinterpret_cast<const float4*>(s.peer[owner].W + i);
        *reinterpret_cast<float4*>(me.dW + i) = *reinterpret_cast<const float4*>(s.peer[owner].dW + i);
    }
}

__global__ void dp_wait_kernel(const int* done, int nranks, int step) {
    if ((int)threadIdx.x < nranks) wait_flag(done + threadIdx.x, step);
}

struct Blob {
    cudaIpcMemHandle_t h[4];      // arena, W, dW, Wb
    unsigned int ok;
    unsigned int pad[3];
};
static_assert(sizeof(Blob) % 4 == 0, "blob travels as 32-bit words");

}  // namespace

void PeerExchange::setup(Ctx* c, int V_, int H_, float* W, float* dW, __nv_bfloat16* Wb, int ldwb_) {
    ctx = c; V = V_; H = H_; ldwb = ldwb_;
    active = false;
    const int R = c->nranks;
    { const char* e = getenv("BM_PEER"); if (e && !atoi(e)) return; }
    if (R <= 1 || R > MAX_PEERS || c->nccl_comm == nullptr) return;
    if (H % 4 != 0 || ldwb % 4 != 0) return;                 // (every rank takes the same branch: same model)
    rows_per = (V + R - 1) / R;
    shard_elems = (size_t)rows_per * H;
    small_len = (2 * H + V + 3) & ~3;
    const size_t inbox_b = (size_t)R * shard_elems * sizeof(float);
    const size_t small_b = (size_t)R * small_len * sizeof(float);
    const size_t flags_off = (inbox_b + small_b + 127) & ~(size_t)127;
    const size_t total = flags_off + 2 * MAX_PEERS * sizeof(int) + 4 * sizeof(unsigned int);
    BM_CUDA(cudaMalloc(&arena, total));
    BM_CUDA(cudaMemsetAsync(arena, 0, total, c->stream));
    BM_CUDA(cudaStreamSynchronize(c->stream));

    Blob mine;
    memset(&mine, 0, sizeof(mine));
    void* bases[4] = {arena, W, dW, Wb};
    mine.ok = 1;
    for (int i = 0; i < 4; ++i)
        if (cudaIpcGetMemHandle(&mine.h[i], bases[i]) != cudaSuccess) { (void)cudaGetLastError(); mine.ok = 0; }
    // all-gather of the blobs: a table of zeros with this rank's slot filled in, summed over the ranks
    const size_t words = sizeof(Blob) / 4;
    unsigned int* tab = nullptr;
    BM_CUDA(cudaMalloc(&tab, (size_t)R * words * 4));
    std::vector<Blob> all(R);
    bool everyone = true;
    try {
        BM_CUDA(cudaMemsetAsync(tab, 0, (size_t)R * words * 4, c->stream));
        BM_CUDA(cudaMemcpyAsync(tab + (size_t)c->rank * words, &mine, sizeof(Blob), cudaMemcpyHostToDevice, c->stream));
        allreduce_sum_u32(c, tab, (size_t)R * words);
        BM_CUDA(cudaMemcpyAsync(all.data(), tab, (size_t)R * sizeof(Blob), cudaMemcpyDeviceToHost, c->stream));
        BM_CUDA(cudaStreamSynchronize(c->stream));
        for (int r = 0; r < R; ++r) everyone = everyone && all[r].ok == 1;
        unsigned int opened = 1;
        if (everyone) {
            for (int r = 0; r < R && opened; ++r) {
                if (r == c->rank) continue;
                for (int i = 0; i < 4; ++i)
                    if (cudaIpcOpenMemHandle(&mapped[r][i], all[r].h[i], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                        (void)cudaGetLastError(); mapped[r][i] = nullptr; opened = 0; break;
                    }
            }
        }
        // agreement: one more sum -- R means every rank exported and mapped everything
        unsigned int vote = (everyone && opened) ? 1u : 0u;
        BM_CUDA(cudaMemcpyAsync(tab, &vote, 4, cudaMemcpyHostToDevice, c->stream));
        allreduce_sum_u32(c, tab, 1);
        BM_CUDA(cudaMemcpyAsync(&vote, tab, 4, cudaMemcpyDeviceToHost, c->stream));
        BM_CUDA(cudaStreamSynchronize(c->stream));
        everyone = vote == (unsigned int)R;
    } catch (...) {
        cudaFree(tab);
        release();
        throw;
    }
    cudaFree(tab);
    if (!everyone) { release(); return; }
    for (int r = 0; r < R; ++r) {
        char* base = static_cast<char*>(r == c->rank ? arena : mapped[r][0]);
        PeerView& pv = view[r];
        pv.inbox = reinterpret_cast<float*>(base);
        pv.small = reinterpret_cast<float*>(base + inbox_b);
        pv.flags = reinterpret_cast<int*>(base + flags_off);
        pv.W = r == c->rank ? W : static_cast<float*>(mapped[r][1]);
        pv.dW = r == c->rank ? dW : static_cast<float*>(mapped[r][2]);
        pv.Wb = r == c->rank ? Wb : static_cast<__nv_bfloat16*>(mapped[r][3]);
    }
    step = 0;
    active = true;
}

void PeerExchange::fill(DpStep& s) const {
    s.rank = ctx->rank; s.nranks = ctx->nranks; s.V = V; s.H = H; s.rows_per = rows_per; s.ldwb = ldwb;
    s.small_len = small_len; s.shard_elems = shard_elems;
    for (int r = 0; r < ctx->nranks; ++r) s.peer[r] = view[r];
    s.counter = reinterpret_cast<unsigned int*>(view[ctx->rank].flags + 2 * MAX_PEERS);
}

void PeerExchange::pull_replicas() {
    if (!active || !stale) return;
    DpStep s{};
    fill(s);
    dp_pull_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(s);
    count_launch(ctx);
    stale = false;
}

void PeerExchange::run(DpStep& s) {
    s.step = ++step;
    static const int repl_env = [] { const char* e = getenv("BM_PEER_REPLICATE_FP32"); return e ? atoi(e) : 0; }();
    s.replicate_fp32 = repl_env != 0 ? 1 : 0;
    stale = !s.replicate_fp32;
    const int blocks = ctx->sm_count * 4;
    // BM_PEER_PROFILE=1: CUDA events around the three kernels, averages printed when the exchange is released
    static const bool prof = [] { const char* e = getenv("BM_PEER_PROFILE"); return e && atoi(e) != 0; }();
    if (prof && !ev[0]) for (int i = 0; i < 4; ++i) BM_CUDA(cudaEventCreate(&ev[i]));
    if (prof && prof_pending) {          // fold the previous step's events (they have completed: same stream)
        BM_CUDA(cudaEventSynchronize(ev[3]));
        for (int i = 0; i < 3; ++i) { float ms = 0.f; BM_CUDA(cudaEventElapsedTime(&ms, ev[i], ev[i + 1])); prof_ms[i] += ms; }
        ++prof_n; prof_pending = false;
    }
    if (prof) BM_CUDA(cudaEventRecord(ev[0], ctx->stream));
    // BM_PEER_BULK=1: transfers as bulk asynchronous copies from shared memory (not measured on H100s; off by default).
    static const int bulk_env = [] { const char* e = getenv("BM_PEER_BULK"); return e ? atoi(e) : 0; }();
    const bool bulk = bulk_env != 0 && H % 8 == 0 && (size_t)H * 4 * 2 + (size_t)H * 2 <= 96 * 1024;
    const int r0 = ctx->rank * rows_per;
    const int r1 = V < r0 + rows_per ? V : r0 + rows_per;
    const int nb = V > H ? V : H;
    if (bulk) {
        static bool attr_done = false;
        if (!attr_done) {
            BM_CUDA(cudaFuncSetAttribute(dp_push_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
            BM_CUDA(cudaFuncSetAttribute(dp_update_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
            attr_done = true;
        }
        // push: rows per block so that a block's buffer is <= 32 KB and the grid has about two blocks per SM
        int prb = (int)(32768 / ((size_t)H * 4)); if (prb < 1) prb = 1;
        while (prb > 1 && (V + prb - 1) / prb < 2 * ctx->sm_count) --prb;
        const int pblocks = (V + prb - 1) / prb;
        dp_push_bulk_kernel<<<pblocks < 4 * ctx->sm_count ? pblocks : 4 * ctx->sm_count, 256, (size_t)prb * H * 4, ctx->stream>>>(s, prb);
        count_launch(ctx);
        if (prof) BM_CUDA(cudaEventRecord(ev[1], ctx->stream));
        // update: rows per block so that W + dW + bf16 rows fit in <= 40 KB, about one block per SM
        const int shard_rows = r1 > r0 ? r1 - r0 : 0;
        int urb = (int)(40960 / ((size_t)H * 10)); if (urb < 1) urb = 1;
        while (urb > 1 && (shard_rows + urb - 1) / urb < ctx->sm_count) --urb;
        unsigned w_blocks = (unsigned)((shard_rows + urb - 1) / urb);
        if (w_blocks > (unsigned)(2 * ctx->sm_count)) w_blocks = (unsigned)(2 * ctx->sm_count);
        dp_update_bulk_kernel<<<w_blocks + (unsigned)((nb + 255) / 256), 256, (size_t)urb * H * 10, ctx->stream>>>(s, w_blocks, urb);
        count_launch(ctx);
    } else {
    dp_push_kernel<<<blocks, 256, 0, ctx->stream>>>(s);
    count_launch(ctx);
    if (prof) BM_CUDA(cudaEventRecord(ev[1], ctx->stream));
    const size_t items = r1 > r0 ? (size_t)(r1 - r0) * H / 4 : 0;
    const unsigned w_blocks = (unsigned)((items + 255) / 256);
    // BM_PEER_SPLIT=1: the update writes this rank's copy only and a second, full-width kernel copies the rows out to the peers
    // (off by default; not measured on H100s)
    static const int split_env = [] { const char* e = getenv("BM_PEER_SPLIT"); return e ? atoi(e) : 0; }();
    const bool split = ctx->nranks > 1 && split_env != 0;
    dp_update_kernel<<<w_blocks + (unsigned)((nb + 255) / 256), 256, 0, ctx->stream>>>(s, w_blocks, split ? 1 : 0);
    count_launch(ctx);
    if (split) {
        dp_scatter_kernel<<<dim3((unsigned)(ctx->sm_count * 2 / (ctx->nranks - 1) + 1), (unsigned)(ctx->nranks - 1)), 256, 0, ctx->stream>>>(s);
        count_launch(ctx);
    }
    }
    if (prof) BM_CUDA(cudaEventRecord(ev[2], ctx->stream));
    dp_wait_kernel<<<1, 32, 0, ctx->stream>>>(view[ctx->rank].flags + MAX_PEERS, ctx->nranks, s.step);
    count_launch(ctx);
    if (prof) { BM_CUDA(cudaEventRecord(ev[3], ctx->stream)); prof_pending = true; }
}

void PeerExchange::release() {
    if (prof_n > 0 && ctx)
        fprintf(stderr, "[bm peer] rank %d of %d: %ld steps, mean us: push %.1f  update (incl. wait for the peers' pushes) %.1f  wait for the peers' updates %.1f\n",
                ctx->rank, ctx->nranks, prof_n, 1e3 * prof_ms[0] / prof_n, 1e3 * prof_ms[1] / prof_n, 1e3 * prof_ms[2] / prof_n);
    prof_n = 0;
    if (ctx) {
        cudaSetDevice(ctx->device);
        cudaStreamSynchronize(ctx->stream);
    }
    for (int r = 0; r < MAX_PEERS; ++r)
        for (int i = 0; i < 4; ++i)
            if (mapped[r][i]) { cudaIpcCloseMemHandle(mapped[r][i]); mapped[r][i] = nullptr; }
    if (arena) { cudaFree(arena); arena = nullptr; }
    (void)cudaGetLastError();
    active = false;
}

}  // namespace bm
