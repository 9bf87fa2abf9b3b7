// Philox-4x32-10 counter-based RNG, held in registers.  Shared layout with the
// CPU oracle (oracle/philox.py::site_words): element (r, c) of draw site `site` at
// Gibbs index t and call tick uses counter (c/4, row0+r, site | t<<8, tick),
// key (seed_lo, seed_hi), word lane c%4.
//
// The W initialiser reproduces tf.random_normal's stream (TF-1.3 philox_random.h /
// random_distributions.h; /root/reference/boltzmann_machines/rbm/base_rbm.py:277-279).
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

namespace bm {

enum Site : uint32_t {
    SITE_DROPOUT = 0, SITE_H0 = 1, SITE_V = 2, SITE_H = 3, SITE_PLL = 4,
    SITE_MULTINOMIAL_FE = 5, SITE_PARTICLE_INIT = 6, SITE_AIS_INIT = 7,
    SITE_AIS_V = 8, SITE_AIS_H2 = 9, SITE_AIS_H1 = 10, SITE_DBM_V = 11, SITE_CRBM_Y = 12, SITE_CRBM_Y0 = 13,
    SITE_DBM_PT = 14,        // parallel tempering: the swap decision of pair (m, m+1) at t = m, column 0 of the particle's row
    SITE_AIS_CLAMPED = 15,   // AIS with v clamped: layer j's initial state at t = 2 j, its transition draws at t = 2 j + 1
    SITE_DBM_H = 16
};

struct RngKey {
    uint32_t k0, k1;     // seed lo / hi
    uint32_t c2;         // site | t << 8
    uint32_t tick;       // call tick
    uint32_t row0;       // first global row of this shard
};

__host__ __device__ __forceinline__ RngKey make_rng(uint64_t seed, uint32_t site, uint32_t t,
                                                    uint32_t tick, uint32_t row0) {
    RngKey k;
    k.k0 = (uint32_t)seed; k.k1 = (uint32_t)(seed >> 32);
    k.c2 = (site & 0xFFu) | ((t & 0xFFFFFFu) << 8);
    k.tick = tick; k.row0 = row0;
    return k;
}

struct U4 { uint32_t x, y, z, w; };

__host__ __device__ __forceinline__ void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
    // one 32x32->64 multiply (IMAD.WIDE.U32 on the GPU) instead of separate lo / hi products
    const uint64_t p = (uint64_t)a * (uint64_t)b; lo = (uint32_t)p; hi = (uint32_t)(p >> 32);
}

__host__ __device__ __forceinline__ U4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                     uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0, lo0, hi1, lo1;
        mulhilo(0xD2511F53u, c0, hi0, lo0);
        mulhilo(0xCD9E8D57u, c2, hi1, lo1);
        c0 = hi1 ^ c1 ^ k0; c1 = lo1;
        c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    U4 o; o.x = c0; o.y = c1; o.z = c2; o.w = c3;
    return o;
}

// the 4 words of column block `cblk` (= c/4) of local row r
__host__ __device__ __forceinline__ U4 site_block(const RngKey& k, uint32_t r, uint32_t cblk) {
    return philox4x32_10(cblk, k.row0 + r, k.c2, k.tick, k.k0, k.k1);
}

// TF Uint32ToFloat: 23 mantissa bits -> [0, 1)
__host__ __device__ __forceinline__ float u32_to_unit_float(uint32_t x) {
    uint32_t bits = (x & 0x7FFFFFu) | 0x3F800000u;
#ifdef __CUDA_ARCH__
    return __uint_as_float(bits) - 1.0f;
#else
    union { uint32_t u; float f; } cv; cv.u = bits; return cv.f - 1.0f;
#endif
}

// TF Uint64ToDouble
__host__ __device__ __forceinline__ double u64_to_unit_double(uint32_t x0, uint32_t x1) {
    uint64_t bits = ((uint64_t)(x0 & 0xFFFFFu) << 32) | (uint64_t)x1 | ((uint64_t)1023 << 52);
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)bits) - 1.0;
#else
    union { uint64_t u; double f; } cv; cv.u = bits; return cv.f - 1.0;
#endif
}

}  // namespace bm
