// TEST INFRASTRUCTURE ONLY -- CPU restatement of what parallel tempering adds to the tensor-core DBM engine (csrc/bm_dbm_tc.cuh),
// for the stand-in runtime (fake_cudart.cpp):
//
//   * dbm_pt_swap_kernel: the slots' energies, the swap decisions and the row exchanges of one swap round;
//   * the draw row offset of a program op (TcPhaseLite::row_off: slot m of the ladder draws at rows row0 + m M + r).
//     kernels_cpu.cpp's program restatement keys every draw by the launch's row0, so a launch with an op whose row_off is
//     not 0 is handed to it one op at a time, each as a launch of its own with row0 + row_off, in program order (which is a
//     topological order of the dependencies).  The dataflow between those ops is then not checked by the hazard shadow.
//
// build_dbm_pt.sh compiles kernels_cpu.cpp with its dispatcher renamed to execute_base and links this file in front of it.
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
bool execute_base(const std::string& name, dim3 grid, dim3 block, void** args);     // kernels_cpu.cpp's dispatcher

static inline float bf2f(__nv_bfloat16 b) { unsigned short s; memcpy(&s, &b, 2); unsigned u = (unsigned)s << 16; float f; memcpy(&f, &u, 4); return f; }

// csrc/bm_dbm_tc.cuh::PtSwapArgs, field for field
struct PtSwapArgs {
    int L, T, M, V;
    int H[8];
    int ld[9];
    __nv_bfloat16* x[9];
    const float* P[8];
    const float* vb;
    const double* betas;
    int parity;
    bm::RngKey rng;
    unsigned long long* accepted;
};

static void k_dbm_pt_swap(void** args, dim3 grid) {
    const PtSwapArgs& a = *reinterpret_cast<const PtSwapArgs*>(args[0]);
    std::vector<double> E(a.T);
    std::vector<int> acc(a.T, 0);
    for (unsigned p = 0; p < grid.x; ++p) {
        for (int m = 0; m < a.T; ++m) {                       // one warp per slot: lane-strided sums, then the xor tree
            const size_t row = (size_t)m * a.M + p;
            double lane[32] = {0};
            for (int j = 0; j < a.V; ++j)
                lane[j % 32] = std::fma((double)bf2f(a.x[0][row * a.ld[0] + j]), (double)a.vb[j], lane[j % 32]);
            for (int i = 0; i < a.L; ++i)
                for (int j = 0; j < a.H[i]; ++j)
                    lane[j % 32] = std::fma((double)bf2f(a.x[i + 1][row * a.ld[i + 1] + j]), (double)a.P[i][row * a.H[i] + j], lane[j % 32]);
            for (int o = 16; o > 0; o >>= 1) {
                double t[32];
                for (int l = 0; l < 32; ++l) t[l] = lane[l] + lane[l ^ o];
                memcpy(lane, t, sizeof(t));
            }
            E[m] = -lane[0];
        }
        for (int m = 0; m + 1 < a.T; ++m) {
            int ok = 0;
            if ((m & 1) == a.parity) {
                bm::RngKey k = a.rng;
                k.c2 = (14u & 0xFFu) | (((uint32_t)m & 0xFFFFFFu) << 8);          // SITE_DBM_PT, t = m
                const double u = (double)bm::u32_to_unit_float(bm::site_block(k, p, 0).x);
                ok = std::log(u) < (a.betas[m] - a.betas[m + 1]) * (E[m] - E[m + 1]);
                if (ok) a.accepted[m] += 1;
            }
            acc[m] = ok;
        }
        for (int m = 0; m + 1 < a.T; ++m) {
            if (!acc[m]) continue;
            for (int l = 0; l <= a.L; ++l) {
                const int n = l == 0 ? a.V : a.H[l - 1];
                __nv_bfloat16* r0 = a.x[l] + ((size_t)m * a.M + p) * a.ld[l];
                __nv_bfloat16* r1 = a.x[l] + ((size_t)(m + 1) * a.M + p) * a.ld[l];
                for (int j = 0; j < n; ++j) std::swap(r0[j], r1[j]);
            }
        }
    }
}

static bool k_tc_program_rows(const std::string& name, dim3 grid, dim3 block, void** args) {
    const bm::TcLaunch& L = *reinterpret_cast<const bm::TcLaunch*>(args[0]);
    if (L.n_phases == 0) {
        if (L.inl.l.row_off == 0) return false;
        bm::TcLaunch one = L;
        one.row0 = L.row0 + L.inl.l.row_off;
        one.inl.l.row_off = 0;
        void* a[1] = {&one};
        return execute_base(name, grid, block, a);
    }
    bool any = false;
    for (int i = 0; i < L.n_phases; ++i) any = any || L.phases[i].l.row_off != 0;
    if (!any) return false;
    for (int i = 0; i < L.n_phases; ++i) {
        bm::TcPhase ph = L.phases[i];
        ph.l.n_deps = 0;                       // ordered by running the ops one after the other
        ph.l.dep_chunk_ctr = nullptr;
        bm::TcLaunch one = L;
        one.phases = &ph;
        one.n_phases = 1;
        one.total_units = ph.l.n_units;
        one.row0 = L.row0 + ph.l.row_off;
        ph.l.row_off = 0;
        void* a[1] = {&one};
        if (!execute_base(name, grid, block, a)) return false;
    }
    return true;
}

bool execute(const std::string& name, dim3 grid, dim3 block, void** args) {
    if (name.find("dbm_pt_swap_kernel") != std::string::npos) { k_dbm_pt_swap(args, grid); return true; }
    if (name.find("tc_program_kernel") != std::string::npos && k_tc_program_rows(name, grid, block, args)) return true;
    return execute_base(name, grid, block, args);
}

}  // namespace fakecuda
