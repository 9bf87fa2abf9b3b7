// TEST INFRASTRUCTURE ONLY -- CPU restatement of the training-group kernels (csrc/bm_rbm_group.cu, csrc/bm_tc_util.cu) for the
// stand-in runtime (fake_cudart.cpp).
//
// build_group.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base and links this file in front of it:
// `execute` below interprets
//   - group_input_kernel<S>: the one conversion of every member's batch,
//   - cd_tail_group_kernel<VEC>: member m's slice is cd_tail_kernel's work on tails[m], handed to kernels_cpu.cpp's restatement,
//   - tc_program_kernel launches whose ops carry keys of their own (TcPhaseLite::k0 / k1): the launch is first interpreted as
//     kernels_cpu.cpp does it, which checks its dataflow (and draws with the launch key), then every op is interpreted again, in
//     program order, as a single-op launch with its own key -- program order is a topological order of the dependencies and
//     every op rewrites all of its outputs, so this leaves exactly what the ops compute with their own keys,
// and hands every other launch to kernels_cpu.cpp unchanged.
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
#include "../../boltzmann-machines_b200/csrc/bm_internal.h"
#include "../../boltzmann-machines_b200/csrc/bm_tc_desc.h"

namespace fakecuda {
bool execute_base(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_cpu.cpp's dispatcher

static inline __nv_bfloat16 f2bf(float f) {           // round to nearest even, as __float2bfloat16_rn
    unsigned u; memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) { u |= 0x00400000u; } else { u += 0x7fffu + ((u >> 16) & 1u); }
    unsigned short b = (unsigned short)(u >> 16); __nv_bfloat16 v; memcpy(&v, &b, 2); return v;
}
template <class T> static inline T arg(void** a, int i) { return *reinterpret_cast<T*>(a[i]); }
static inline float widen(uint8_t x) { return (float)x; }
static inline float widen(uint16_t x) { const unsigned u = (unsigned)x << 16; float f; memcpy(&f, &u, 4); return f; }
static inline float widen(float x) { return x; }

// group_input_kernel<S>(src, V, rows, slot, sigma, Xf, Xb, ldb), grid.z = members
template <class S>
static void k_group_input(void** a, dim3 grid) {
    const S* src = arg<const S*>(a, 0); const int V = arg<int>(a, 1), rows = arg<int>(a, 2); const size_t slot = arg<size_t>(a, 3);
    const float* sigma = arg<const float*>(a, 4); float* Xf = arg<float*>(a, 5); __nv_bfloat16* Xb = arg<__nv_bfloat16*>(a, 6);
    const int ldb = arg<int>(a, 7);
    for (unsigned g = 0; g < grid.z; ++g)
        for (int r = 0; r < rows; ++r)
            for (int c = 0; c < V; ++c) {
                const size_t row = (size_t)g * slot + r;
                float x = widen(src[row * V + c]);
                if (sigma) x = x / sigma[(size_t)g * V + c];
                Xf[row * V + c] = x;
                Xb[row * ldb + c] = f2bf(x);
            }
}

static void k_cd_tail_group(void** a, dim3 grid, dim3 block) {
    const bm::CdTail* tails = arg<const bm::CdTail*>(a, 0); unsigned per = arg<unsigned>(a, 1), w_blocks = arg<unsigned>(a, 2);
    for (unsigned m = 0; m < grid.x / per; ++m) {
        bm::CdTail t = tails[m];
        void* one[2] = {&t, &w_blocks};
        execute_base("cd_tail_kernel", dim3(per), block, one);
    }
}

static bool k_tc_program_own_keys(const std::string& name, dim3 grid, dim3 block, void** a) {
    const bm::TcLaunch& L = *reinterpret_cast<const bm::TcLaunch*>(a[0]);
    bool own = false;
    for (int i = 0; i < L.n_phases; ++i) own = own || L.phases[i].l.k0 != L.k0 || L.phases[i].l.k1 != L.k1;
    if (!own) return execute_base(name, grid, block, a);
    execute_base(name, grid, block, a);
    for (int i = 0; i < L.n_phases; ++i) {
        bm::TcLaunch one = L;
        one.n_phases = 0; one.phases = nullptr;
        one.inl = L.phases[i];
        one.k0 = L.phases[i].l.k0; one.k1 = L.phases[i].l.k1;
        void* args[1] = {&one};
        execute_base(name, grid, block, args);
    }
    return true;
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    auto has = [&](const char* s) { return name.find(s) != std::string::npos; };
    if (has("group_input_kernelIhE")) { k_group_input<uint8_t>(args, grid); return true; }
    if (has("group_input_kernelItE")) { k_group_input<uint16_t>(args, grid); return true; }
    if (has("group_input_kernelIfE")) { k_group_input<float>(args, grid); return true; }
    if (has("cd_tail_group_kernel")) { k_cd_tail_group(args, grid, block); return true; }
    if (has("tc_program_kernel")) return k_tc_program_own_keys(name, grid, block, args);
    return execute_base(name, grid, block, args);
}

}  // namespace fakecuda
