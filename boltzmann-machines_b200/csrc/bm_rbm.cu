// RBM engine behind bm_rbm_* (include/bm.h): owns the device-resident variables of one RBM
// and runs the whole CD-k mini-batch step -- what the reference executes as ONE
// session.run(train_op) (rbm/base_rbm.py:415-479, 566) -- as a fixed sequence of kernels on
// the context's stream, with no host round trip inside the step.
#include "bm_rbm.h"

using namespace bm;

extern "C" {

int bm_rbm_create(bm_ctx* hctx, const bm_rbm_cfg* cfg, bm_rbm** out) {
    BM_API_BEGIN
    Ctx* ctx = reinterpret_cast<Ctx*>(hctx);
    BM_REQUIRE(ctx && cfg && out, "null argument");
    BM_REQUIRE(cfg->n_visible > 0 && cfg->n_hidden > 0, "n_visible and n_hidden must be positive");
    BM_REQUIRE(cfg->v_kind >= 0 && cfg->v_kind <= 2 && cfg->h_kind >= 0 && cfg->h_kind <= 2, "bad unit kind");
    BM_REQUIRE(cfg->h_kind != BM_UNIT_GAUSSIAN, "gaussian hidden units are not supported");
    BM_REQUIRE(cfg->v_kind != BM_UNIT_GAUSSIAN || cfg->sigma != nullptr, "gaussian visible layer needs sigma");
    BM_CUDA(cudaSetDevice(ctx->device));
    RbmBase* r = nullptr;
    if (cfg->compute == BM_COMPUTE_BF16) {
        BM_REQUIRE(cfg->dtype == BM_DTYPE_F32, "bf16 compute needs float32 storage");
        r = make_rbm_tc(ctx, *cfg);
    } else if (cfg->dtype == BM_DTYPE_F64) {
        r = new RbmSimt<double>(ctx, *cfg);
    } else {
        r = new RbmSimt<float>(ctx, *cfg);
    }
    *out = reinterpret_cast<bm_rbm*>(r);
    BM_API_END
}

void bm_rbm_destroy(bm_rbm* h) {
    if (!h) return;
    RbmBase* r = reinterpret_cast<RbmBase*>(h);
    cudaSetDevice(r->ctx->device);
    cudaStreamSynchronize(r->ctx->stream);
    delete r;
}

#define RBM(h) (reinterpret_cast<RbmBase*>(h))
#define RBM_ENTER(h)                                   \
    BM_REQUIRE((h) != nullptr, "null rbm handle");     \
    BM_CUDA(cudaSetDevice(RBM(h)->ctx->device));

int bm_rbm_set_param(bm_rbm* h, const char* name, const void* host, size_t bytes) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(name && host, "null argument");
    RBM(h)->set_param(name, host, bytes);
    BM_API_END
}
int bm_rbm_get_param(bm_rbm* h, const char* name, void* host, size_t bytes) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(name && host, "null argument");
    RBM(h)->get_param(name, host, bytes);
    BM_API_END
}
int bm_rbm_init_weights(bm_rbm* h, double stddev, uint64_t op_seed) {
    BM_API_BEGIN RBM_ENTER(h)
    RBM(h)->init_weights(stddev, op_seed);
    BM_API_END
}
int bm_rbm_train_step(bm_rbm* h, const void* X, int32_t rows, double lr, double momentum, int32_t k,
                      uint64_t seed, uint32_t tick, uint32_t mask, double* out) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(X, "null batch");
    RBM(h)->train_step(X, 0, rows, lr, momentum, k, seed, tick, mask, out);
    BM_API_END
}
int bm_rbm_set_data(bm_rbm* h, const void* X, int64_t n_rows) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(X && n_rows > 0, "bad dataset");
    RBM(h)->set_data(X, n_rows);
    BM_API_END
}
int bm_rbm_train_step_at(bm_rbm* h, int64_t first_row, int32_t rows, double lr, double momentum, int32_t k,
                         uint64_t seed, uint32_t tick, uint32_t mask, double* out) {
    BM_API_BEGIN RBM_ENTER(h)
    RBM(h)->train_step(nullptr, first_row, rows, lr, momentum, k, seed, tick, mask, out);
    BM_API_END
}
int bm_rbm_train_epoch(bm_rbm* h, const void* X, int64_t n_rows, int32_t batch, double lr, double momentum, int32_t k,
                       uint64_t seed, uint32_t tick0, uint32_t mask, int32_t metrics_every, int64_t iter0, double* out) {
    BM_API_BEGIN RBM_ENTER(h)
    RBM(h)->train_epoch(X, n_rows, batch, lr, momentum, k, seed, tick0, mask, metrics_every, iter0, out, SRC_NATIVE);
    BM_API_END
}
int bm_rbm_train_epoch_u8(bm_rbm* h, const uint8_t* X, int64_t n_rows, int32_t batch, double lr, double momentum, int32_t k,
                          uint64_t seed, uint32_t tick0, uint32_t mask, int32_t metrics_every, int64_t iter0, double* out) {
    BM_API_BEGIN RBM_ENTER(h)
    RBM(h)->train_epoch(X, n_rows, batch, lr, momentum, k, seed, tick0, mask, metrics_every, iter0, out, SRC_U8);
    BM_API_END
}
int bm_rbm_train_epoch_bf16(bm_rbm* h, const uint16_t* X, int64_t n_rows, int32_t batch, double lr, double momentum, int32_t k,
                            uint64_t seed, uint32_t tick0, uint32_t mask, int32_t metrics_every, int64_t iter0, double* out) {
    BM_API_BEGIN RBM_ENTER(h)
    RBM(h)->train_epoch(X, n_rows, batch, lr, momentum, k, seed, tick0, mask, metrics_every, iter0, out, SRC_BF16);
    BM_API_END
}
int bm_rbm_transform(bm_rbm* h, const void* X, int32_t rows, int32_t k, uint64_t seed, uint32_t tick, void* H_out) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(X && H_out, "null argument");
    RBM(h)->transform(X, rows, k, seed, tick, H_out);
    BM_API_END
}
int bm_rbm_metrics(bm_rbm* h, const void* X, int32_t rows, int32_t k, uint64_t seed, uint32_t tick,
                   uint32_t mask, double* out) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(X && out, "null argument");
    RBM(h)->metrics(X, rows, k, seed, tick, mask, out);
    BM_API_END
}
int bm_rbm_get_activation(bm_rbm* h, const char* name, void* host, size_t bytes) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(name && host, "null argument");
    RBM(h)->get_activation(name, host, bytes);
    BM_API_END
}
int bm_rbm_debug_tc_plan(bm_rbm* h, bm_tc_op_plan* out, int32_t cap, int32_t* n_ops) {
    BM_API_BEGIN RBM_ENTER(h) BM_REQUIRE(n_ops && (out || cap == 0) && cap >= 0, "bad argument");
    const std::vector<bm_tc_op_plan>& plan = RBM(h)->tc_plan();
    *n_ops = (int32_t)plan.size();
    for (size_t i = 0; i < plan.size() && (int32_t)i < cap; ++i) out[i] = plan[i];
    BM_API_END
}

}  // extern "C"
