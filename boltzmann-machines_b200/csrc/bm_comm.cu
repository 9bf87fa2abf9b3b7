// Context management and the multi-GPU plumbing of libbm.so.
//
// NCCL is resolved at run time (dlopen "libnccl.so.2"): libbm.so itself has no link-time
// dependency on it, so the library loads (and the single-GPU path runs) without NCCL.
// The reference is single-device (SURVEY.md §2a); the sum-allreduce of the gradient
// statistics is this engine's addition for batch-sharded chains.
#include "bm_internal.h"
#include <dlfcn.h>
#include <string.h>
#include <stdlib.h>
#include <mutex>
#include <thread>
#include <atomic>
#include <vector>
#include <nvtx3/nvToolsExt.h>

namespace bm {

thread_local std::string g_last_error;

static bool nvtx_enabled() {
    static const bool on = [] { const char* e = getenv("BM_NVTX"); return e && atoi(e) != 0; }();
    return on;
}
NvtxRange::NvtxRange(const char* name) : on(nvtx_enabled()) { if (on) nvtxRangePushA(name); }
NvtxRange::~NvtxRange() { if (on) nvtxRangePop(); }

struct NcclId { char internal[128]; };
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, struct NcclId, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};

static NcclApi* nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        // BM_NCCL_LIB: explicit path of the NCCL library (a pinned build; the host simulation's stand-in), else the default names
        const char* names[] = {getenv("BM_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n || !*n) continue;
            api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (!api.lib) return;
        api.GetUniqueId = (int (*)(void*))dlsym(api.lib, "ncclGetUniqueId");
        api.CommInitRank = (int (*)(void**, int, NcclId, int))dlsym(api.lib, "ncclCommInitRank");
        api.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(api.lib, "ncclAllReduce");
        api.CommDestroy = (int (*)(void*))dlsym(api.lib, "ncclCommDestroy");
        api.GetErrorString = (const char* (*)(int))dlsym(api.lib, "ncclGetErrorString");
    });
    if (!api.lib || !api.GetUniqueId || !api.CommInitRank || !api.AllReduce)
        throw Error(BM_ENCCL, "NCCL (libnccl.so.2) could not be loaded");
    return &api;
}

static void nccl_check(int rc, const char* what) {
    if (rc != 0) {
        NcclApi* a = nccl_api();
        throw Error(BM_ENCCL, std::string(what) + " failed: " + (a->GetErrorString ? a->GetErrorString(rc) : "?"));
    }
}

// sum-allreduce in place on the context's compute stream (no-op on a single rank)
void allreduce_sum(Ctx* ctx, void* buf, size_t count, bool is_double) {
    if (ctx->nranks <= 1) return;
    NcclApi* a = nccl_api();
    // ncclFloat32 = 7, ncclFloat64 = 8, ncclSum = 0
    nccl_check(a->AllReduce(buf, buf, count, is_double ? 8 : 7, 0, ctx->nccl_comm, ctx->stream), "ncclAllReduce");
    count_launch(ctx);
}

// max-allreduce of unsigned 32-bit words in place (bit patterns of non-negative floats order like the floats):
// the DBM's mean-field convergence test over row-sharded variational parameters
void allreduce_max_u32(Ctx* ctx, unsigned int* buf, size_t count) {
    if (ctx->nranks <= 1) return;
    NcclApi* a = nccl_api();
    // ncclUint32 = 3, ncclMax = 2
    nccl_check(a->AllReduce(buf, buf, count, 3, 2, ctx->nccl_comm, ctx->stream), "ncclAllReduce(max)");
    count_launch(ctx);
}

// sum-allreduce of unsigned 32-bit words (the all-gather of small opaque tables, bm_peer.cu)
void allreduce_sum_u32(Ctx* ctx, unsigned int* buf, size_t count) {
    if (ctx->nranks <= 1) return;
    NcclApi* a = nccl_api();
    nccl_check(a->AllReduce(buf, buf, count, 3, 0, ctx->nccl_comm, ctx->stream), "ncclAllReduce(u32 sum)");
    count_launch(ctx);
}

cudaEvent_t profile_event(Ctx* c) {
    if (c->prof_used == c->prof_events.size()) {
        if (c->prof_events.size() >= 16384) profile_drain(c);
        else {
            cudaEvent_t e;
            BM_CUDA(cudaEventCreate(&e));
            c->prof_events.push_back(e);
        }
    }
    return c->prof_events[c->prof_used++];
}

void profile_drain(Ctx* c) {
    if (c->prof_used == 0) return;
    BM_CUDA(cudaStreamSynchronize(c->stream));
    for (size_t i = 0; i + 1 < c->prof_used; i += 2) {
        float ms = 0.f;
        BM_CUDA(cudaEventElapsedTime(&ms, c->prof_events[i], c->prof_events[i + 1]));
        c->prof_ms += ms;
    }
    c->prof_used = 0;
}

}  // namespace bm

// ---- host-side packing of a training set for the feed path (multi-threaded, one pass) -------------------------------------
namespace {
template <typename F> void parallel_ranges(size_t n, F&& body) {
    unsigned hw = std::thread::hardware_concurrency();
    size_t nt = hw ? hw : 8;
    if (nt > 32) nt = 32;
    if (n < (size_t)1 << 20) nt = 1;
    std::vector<std::thread> th;
    const size_t per = (n + nt - 1) / nt;
    for (size_t t = 0; t < nt; ++t) {
        const size_t lo = t * per, hi = lo + per < n ? lo + per : n;
        if (lo >= hi) break;
        th.emplace_back([&body, lo, hi] { body(lo, hi); });
    }
    for (std::thread& x : th) x.join();
}
template <typename T> bool pack_u8(const T* X, size_t n, uint8_t* out) {
    std::atomic<int> exact(1);
    parallel_ranges(n, [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            const T v = X[i];
            const uint8_t b = (v >= T(0) && v <= T(255)) ? (uint8_t)v : 0;
            if ((T)b != v) { exact.store(0); return; }          // also false for NaN
            out[i] = b;
        }
    });
    return exact.load() != 0;
}
}  // namespace

using namespace bm;

extern "C" {

const char* bm_version(void) { return "bm 0.1 (sm_90a)"; }
const char* bm_last_error(void) { return g_last_error.c_str(); }

int bm_device_count(int* n) {
    BM_API_BEGIN
    BM_REQUIRE(n != nullptr, "bm_device_count: null output");
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) { c = 0; (void)cudaGetLastError(); }
    *n = c;
    BM_API_END
}

int bm_ctx_create(int device, bm_ctx** out) {
    BM_API_BEGIN
    BM_REQUIRE(out != nullptr, "bm_ctx_create: null output");
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        (void)cudaGetLastError();
        throw Error(BM_ENOGPU, "no CUDA device visible: the engine has no CPU fallback");
    }
    BM_REQUIRE(device >= 0 && device < n, "bm_ctx_create: device index out of range");
    BM_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    BM_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        throw Error(BM_ENOGPU, std::string("device is sm_") + std::to_string(prop.major) + std::to_string(prop.minor) +
                                   "; libbm.so is built for sm_90a (H100) only");
    Ctx* c = new Ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    BM_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    BM_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    BM_CUDA(cudaEventCreate(&c->t0));
    BM_CUDA(cudaEventCreate(&c->t1));
    BM_CUDA(cudaEventCreateWithFlags(&c->copy_done, cudaEventDisableTiming));
    *out = reinterpret_cast<bm_ctx*>(c);
    BM_API_END
}

void bm_ctx_destroy(bm_ctx* h) {
    if (!h) return;
    Ctx* c = reinterpret_cast<Ctx*>(h);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (c->nccl_comm) {
        try { NcclApi* a = nccl_api(); if (a->CommDestroy) a->CommDestroy(c->nccl_comm); } catch (...) {}
    }
    for (cudaEvent_t e : c->prof_events) cudaEventDestroy(e);
    if (c->l2_scratch) cudaFree(c->l2_scratch);
    if (c->sqdiff_scratch) cudaFree(c->sqdiff_scratch);
    if (c->reduce_scratch) cudaFree(c->reduce_scratch);
    if (c->colsum_scratch) cudaFree(c->colsum_scratch);
    cudaEventDestroy(c->t0); cudaEventDestroy(c->t1); cudaEventDestroy(c->copy_done);
    cudaStreamDestroy(c->stream); cudaStreamDestroy(c->copy_stream);
    delete c;
}

int bm_ctx_sync(bm_ctx* h) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c, "null context");
    BM_CUDA(cudaStreamSynchronize(c->copy_stream));
    BM_CUDA(cudaStreamSynchronize(c->stream));
    BM_API_END
}

int bm_ctx_timer_start(bm_ctx* h) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c, "null context");
    BM_CUDA(cudaEventRecord(c->t0, c->stream));
    BM_API_END
}

int bm_ctx_timer_stop(bm_ctx* h, float* ms) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c && ms, "null argument");
    BM_CUDA(cudaEventRecord(c->t1, c->stream));
    BM_CUDA(cudaEventSynchronize(c->t1));
    BM_CUDA(cudaEventElapsedTime(ms, c->t0, c->t1));
    BM_API_END
}

int bm_ctx_flush_l2(bm_ctx* h) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c, "null context");
    if (!c->l2_scratch) {
        c->l2_scratch_bytes = (size_t)256 << 20;      // 256 MiB > 50 MB L2
        BM_CUDA(cudaMalloc(&c->l2_scratch, c->l2_scratch_bytes));
    }
    BM_CUDA(cudaMemsetAsync(c->l2_scratch, 0, c->l2_scratch_bytes, c->stream));
    BM_API_END
}

int bm_host_alloc(void** p, size_t bytes) {
    BM_API_BEGIN
    BM_REQUIRE(p, "null output");
    BM_CUDA(cudaMallocHost(p, bytes));
    BM_API_END
}

int bm_host_free(void* p) {
    BM_API_BEGIN
    if (p) BM_CUDA(cudaFreeHost(p));
    BM_API_END
}

int bm_host_pack_u8(const void* X, int32_t dtype, size_t n, uint8_t* out, int32_t* exact) {
    BM_API_BEGIN
    BM_REQUIRE(X && out && exact && (dtype == BM_DTYPE_F32 || dtype == BM_DTYPE_F64), "bad argument");
    *exact = (dtype == BM_DTYPE_F32 ? pack_u8((const float*)X, n, out) : pack_u8((const double*)X, n, out)) ? 1 : 0;
    BM_API_END
}

int bm_host_pack_bf16(const float* X, size_t n, uint16_t* out) {
    BM_API_BEGIN
    BM_REQUIRE(X && out, "bad argument");
    parallel_ranges(n, [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            uint32_t u; memcpy(&u, X + i, 4);
            if ((u & 0x7fffffffu) > 0x7f800000u) u |= 0x00400000u;          // NaN stays NaN (as __float2bfloat16_rn)
            else u += 0x7fffu + ((u >> 16) & 1u);                            // round to nearest even
            out[i] = (uint16_t)(u >> 16);
        }
    });
    BM_API_END
}

int bm_ctx_launch_count(bm_ctx* h, uint64_t* n) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c && n, "null argument");
    *n = c->launches;
    BM_API_END
}

int bm_ctx_profile_tc(bm_ctx* h, int enable) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c, "null context");
    profile_drain(c);
    c->profile_tc = enable != 0;
    if (enable) { c->prof_flops = 0.0; c->prof_ms = 0.0; c->prof_launches = 0; }
    BM_API_END
}

int bm_ctx_profile_read(bm_ctx* h, double* flops, double* ms, uint64_t* launches) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c && flops && ms && launches, "null argument");
    profile_drain(c);
    *flops = c->prof_flops; *ms = c->prof_ms; *launches = c->prof_launches;
    BM_API_END
}

int bm_comm_unique_id(void* id128) {
    BM_API_BEGIN
    BM_REQUIRE(id128, "null output");
    NcclApi* a = nccl_api();
    NcclId id;
    memset(&id, 0, sizeof(id));
    nccl_check(a->GetUniqueId(&id), "ncclGetUniqueId");
    memcpy(id128, &id, sizeof(id));
    BM_API_END
}

int bm_ctx_comm_init(bm_ctx* h, const void* id128, int rank, int nranks) {
    BM_API_BEGIN
    Ctx* c = reinterpret_cast<Ctx*>(h);
    BM_REQUIRE(c && id128, "null argument");
    BM_REQUIRE(nranks >= 1 && rank >= 0 && rank < nranks, "bad rank / nranks");
    BM_REQUIRE(c->nccl_comm == nullptr, "communicator already initialised");
    c->rank = rank;
    c->nranks = nranks;
    if (nranks > 1) {
        NcclApi* a = nccl_api();
        NcclId id;
        memcpy(&id, id128, sizeof(id));
        BM_CUDA(cudaSetDevice(c->device));
        nccl_check(a->CommInitRank(&c->nccl_comm, nranks, id, rank), "ncclCommInitRank");
    }
    BM_API_END
}

}  // extern "C"
