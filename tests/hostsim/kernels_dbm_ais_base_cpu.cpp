// TEST INFRASTRUCTURE ONLY -- CPU restatement of what AIS from a base-rate model adds to the tensor-core program kernel
// (csrc/bm_tc.cu, DESIGN.md §5.4d), for the stand-in runtime (fake_cudart.cpp):
//
//   * the base vector of an AIS op (TcPhaseLite::ais_base, nullable): every sigmoid argument of the op gains + a[n] after the
//     beta scaling.  The units op (ais_kind 1) draws from sigmoid(next z + a) and adds softplus(b z + a) - softplus(a' z + a)
//     with z = acc + bias; the state op (ais_kind 2) draws from sigmoid(acc_scale acc + bias_scale bias + a) and adds its
//     linear term without a.
//
// A launch none of whose ops has a base goes to kernels_cpu.cpp's program restatement unchanged.  A launch with one is run
// one op at a time in program order (a topological order of the dependencies), each as a launch of its own: an op without a
// base is handed down as it is; an op with one is handed down as a raw fp32 op (its accumulators, no bias, no outputs) into a
// scratch buffer, and the epilogue above is applied here.  The dataflow of those launches is not checked by the hazard shadow.
//
// build_dbm_ais_base.sh links this file in front of the depth restatement (kernels_dbm_ais_depth_cpu.cpp, dispatcher renamed
// to execute_ais_depth), which falls back to the multinomial restatement and then to kernels_cpu.cpp.
#include <cuda_runtime_api.h>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>
#undef __host__
#undef __device__
#undef __forceinline__
#include "../../boltzmann-machines_b200/csrc/bm_internal.h"   // RngKey, site_block
#include "../../boltzmann-machines_b200/csrc/bm_tc_desc.h"

namespace fakecuda {
bool execute_ais_depth(const std::string& name, dim3 grid, dim3 block, void** args);    // kernels_dbm_ais_depth_cpu.cpp

static inline __nv_bfloat16 f2bf(float f) {           // round to nearest even, as kernels_cpu.cpp
    unsigned u; memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) { u |= 0x00400000u; } else { u += 0x7fffu + ((u >> 16) & 1u); }
    unsigned short b = (unsigned short)(u >> 16); __nv_bfloat16 v; memcpy(&v, &b, 2); return v;
}

static bool has_base(const bm::TcPhaseLite& p) { return p.ais_kind != 0 && p.ais_base != nullptr; }

// one op with a base: its accumulators from kernels_cpu.cpp, then the AIS epilogue with the base
static bool run_based_op(const std::string& name, dim3 grid, dim3 block, const bm::TcPhase& ph, const bm::TcLaunch& L) {
    const bm::TcPhaseLite& p = ph.l;
    std::vector<float> acc((size_t)p.M * p.N);
    bm::TcPhase raw = ph;
    raw.l.ais_kind = 0; raw.l.ais_logw = nullptr; raw.l.noise_sigma = nullptr;
    raw.l.act = bm::ACT_LINEAR; raw.l.sample = bm::SMP_NONE; raw.l.acc_scale = 1.f; raw.l.bias = nullptr; raw.l.sigma = nullptr;
    raw.l.out_mean_bf = nullptr; raw.l.out_state_bf = nullptr;
    raw.l.out_f32 = acc.data(); raw.l.ld_f32 = p.N; raw.l.splits = 1; raw.l.split_stride = 0;
    raw.l.n_deps = 0; raw.l.dep_chunk_ctr = nullptr;
    bm::TcLaunch one = L;
    one.phases = &raw; one.n_phases = 1; one.total_units = raw.l.n_units;
    void* a[1] = {&one};
    if (!execute_ais_depth(name, grid, block, a)) return false;
    bm::RngKey rng; rng.k0 = L.k0; rng.k1 = L.k1; rng.tick = L.tick + p.tick_off; rng.row0 = L.row0; rng.c2 = p.rng_c2;
    for (int m = 0; m < p.M; ++m) {
        double w = 0.0, lin = 0.0;
        for (int nb = 0; nb < p.N; nb += 4) {
            bm::U4 u{0, 0, 0, 0};
            if (p.sample != bm::SMP_NONE) u = bm::site_block(rng, (uint32_t)m, (uint32_t)(nb >> 2));
            const uint32_t words[4] = {u.x, u.y, u.z, u.w};
            for (int j = 0; j < 4 && nb + j < p.N; ++j) {
                const int n = nb + j;
                const float a0 = p.ais_base[n], c = acc[(size_t)m * p.N + n];
                const float b = p.bias ? p.bias[n] : 0.f;
                float pr;
                if (p.ais_kind == 1) {
                    const float z = c + b;
                    const float sa = 1.0f / (1.0f + expf(-(p.ais_a * z + a0)));
                    w += (double)log1pf(sa * expm1f((p.ais_b - p.ais_a) * z));
                    pr = 1.0f / (1.0f + expf(-(p.ais_next * z + a0)));
                } else {
                    pr = 1.0f / (1.0f + expf(-(p.acc_scale * c + p.bias_scale * b + a0)));
                }
                const float st = p.sample == bm::SMP_BERNOULLI ? ((bm::u32_to_unit_float(words[j]) < pr) ? 1.0f : 0.0f) : pr;
                if (p.ais_kind == 2) lin += (double)(st * b);
                if (p.out_state_bf) p.out_state_bf[(size_t)m * p.ld_state_bf + n] = f2bf(st);
            }
        }
        if (p.out_state_bf && (p.N & 7) != 0)               // the clipped TMA store's poison, as kernels_cpu.cpp models it
            for (int c = p.N; c < ((p.N + 7) & ~7) && c < p.ld_state_bf; ++c) p.out_state_bf[(size_t)m * p.ld_state_bf + c] = f2bf(NAN);
        if (p.ais_logw) {
            if (p.ais_kind == 1) p.ais_logw[m] += w;
            else p.ais_logw[m] += (double)p.ais_lin * (double)(p.bias_scale * -1.4426950408889634f) * lin;
        }
    }
    return true;
}

static bool k_tc_program_base(const std::string& name, dim3 grid, dim3 block, void** args) {
    const bm::TcLaunch& L = *reinterpret_cast<const bm::TcLaunch*>(args[0]);
    if (L.n_phases == 0) {
        if (!has_base(L.inl.l)) return false;
        bm::TcLaunch prog = L;
        prog.phases = &L.inl; prog.n_phases = 1; prog.total_units = L.inl.l.n_units;
        return run_based_op(name, grid, block, L.inl, prog);
    }
    bool any = false;
    for (int i = 0; i < L.n_phases; ++i) any = any || has_base(L.phases[i].l);
    if (!any) return false;
    for (int i = 0; i < L.n_phases; ++i) {
        bm::TcPhase ph = L.phases[i];
        ph.l.n_deps = 0;                       // ordered by running the ops one after the other
        ph.l.dep_chunk_ctr = nullptr;
        if (has_base(ph.l)) {
            if (!run_based_op(name, grid, block, ph, L)) return false;
            continue;
        }
        bm::TcLaunch one = L;
        one.phases = &ph; one.n_phases = 1; one.total_units = ph.l.n_units;
        void* a[1] = {&one};
        if (!execute_ais_depth(name, grid, block, a)) return false;
    }
    return true;
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("tc_program_kernel") != std::string::npos && k_tc_program_base(name, grid, block, args)) return true;
    return execute_ais_depth(name, grid, block, args);
}

}  // namespace fakecuda
