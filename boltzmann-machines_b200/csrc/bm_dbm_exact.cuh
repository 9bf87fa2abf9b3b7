// Exact log Z and log p*(v) of binary DBMs with at most 32 odd-layer units (DESIGN.md §5.4f): included by bm_dbm.cu after DbmTC.
//
// Unit layer j = 0..L is v (j = 0) or h_j; the odd layers h_1, h_3, ... form the state x (n_odd bits, x_1 in the lowest bits),
// v and the even layers are summed out analytically:
//   log p*(x) = c.x + sum_{even j} sum_n softplus(z_{j,n}(x)),   z_j(x) = b_j + x_{j-1} W_{j-1} + x_{j+1} W_j^T
//   log Z     = LSE_x log p*(x)
//   log p*(v) = b_v.v + LSE_x [x_1.(v W_0) + g(x)],              g(x) = log p*(x) - sum_n softplus(z_{0,n}(x))
// Every z_j is linear in x: z(x) = b + x M with M [n_odd, N] the weights of the even layers' columns (N = their widths).  The
// state index s IS x, so both GEMMs take their 0/1 operand straight from the bits of s (0 and 1 are exact in bf16): nothing is
// stored per state but g.
//   dbm_exact_states_kernel  z = s M on the tensor cores (mma.sync m16n8k16, bf16 in, fp32 accumulators), M split as
//                            bf16(M) + bf16(M - bf16(M)) along K; the softplus row sums in float64; per CTA the pair
//                            (max, sum exp(. - max)) of log p*, and g of every state when rows are asked for.
//   dbm_exact_rows_kernel    t = q_r.x_1 + g(x) for query rows q_r = v_r W_0 (split in three bf16 terms) against the keys x_1
//                            of a CTA's states, on the tensor cores; per row a running (max, sum) -- the attention normaliser.
//   dbm_exact_merge_kernel   the CTAs' pairs of one row, merged in a fixed order into the row's running pair.
//   dbm_exact_query_kernel   q_r = v_r W_0 and b_v.v_r in float64 on the CUDA cores (rows x V x n_1 products, not the hot path).
#pragma once

namespace bm {

constexpr int EXACT_STATES_PER_CTA = 512;      // 8 warps x 4 m16 tiles
constexpr int EXACT_ROW_STATES = 8192;         // states per CTA of the rows kernel
constexpr int EXACT_ROW_GROUP = 4096;          // rows per rows-kernel launch (bounds its pairs to 4096 x 512 per chunk)

// two bf16 values 0 / 1: bits k and k + 1 of s (low half: bit k)
__device__ __forceinline__ uint32_t exact_bit_pair(uint32_t s, int k) {
    return (((s >> k) & 1u) * 0x3F80u) | ((((s >> (k + 1)) & 1u) * 0x3F80u) << 16);
}
__device__ __forceinline__ void exact_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// softplus(z) = max(z, 0) + log1p(exp(-|z|)): finite and accurate for every finite z; 0 at z = -inf (the padding columns).
// (The AIS epilogues' log1p(sigmoid(a z) expm1((b - a) z)) at (a, b) = (0, 1) overflows to inf for z > 88.7.)
__device__ __forceinline__ float exact_softplus(float z) { return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z))); }
// (m, s) <- (m, s) (+) (m2, s2), the log-sum-exp pair m + log s; (-inf, 0) is empty.  Symmetric in its two operands.
__device__ __forceinline__ void exact_lse_merge(double& m, double& s, double m2, double s2) {
    const double M = fmax(m, m2);
    if (M == -INFINITY) return;
    s = s * exp(m - M) + s2 * exp(m2 - M);
    m = M;
}

struct ExactStatesArgs {
    const uint32_t* B;              // [n_pad][16 ks] words: column n's 32 ks bf16 operand values, bf16(M) rows then the residual's
    const float* bias;              // [n_pad]; -inf on padding columns
    const double* c;                // [32] the odd-layer bias of each state bit (0 past n_odd)
    int ks;                         // 16-bit steps of the state: 1 (n_odd <= 16) or 2
    int n_pad, n_rest;              // columns [0, n_rest): the even layers above v; [n_rest, n_pad): v (both multiples of 8)
    int n_bits;                     // n_odd
    uint32_t s0, n;                 // the launch's states s0 .. s0 + n - 1
    double* g;                      // nullable, [n]: g(s0 + i)
    double2* part;                  // [gridDim.x] (max, sum exp(log p* - max)) of each CTA's states
};

// 256 threads; warp w of CTA b takes the 64 states s0 + 512 b + 64 w + [0, 64) as four m16 tiles of A (rows = states,
// K = the state's bits, hi then lo).  Each n8 tile of columns is four k16 steps (ks = 2) on every m tile; lane (g, t) keeps the
// fp32 pair sum of its two columns for states g and g + 8 of each tile and adds it to a float64 row sum.
template <int KS>
__global__ void __launch_bounds__(256) dbm_exact_states_kernel(ExactStatesArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
    const uint32_t wofs = (uint32_t)blockIdx.x * EXACT_STATES_PER_CTA + (uint32_t)warp * 64u;
    uint32_t A[4][KS][4];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
        const uint32_t s = a.s0 + wofs + mt * 16 + gq;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int k = ks * 16 + 2 * tq;
            A[mt][ks][0] = exact_bit_pair(s, k);     A[mt][ks][1] = exact_bit_pair(s + 8, k);
            A[mt][ks][2] = exact_bit_pair(s, k + 8); A[mt][ks][3] = exact_bit_pair(s + 8, k + 8);
        }
    }
    double tot[4][2], rest[4][2];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) tot[mt][0] = tot[mt][1] = rest[mt][0] = rest[mt][1] = 0.0;
    for (int n0 = 0; n0 < a.n_pad; n0 += 8) {
        if (n0 == a.n_rest) {
#pragma unroll
            for (int mt = 0; mt < 4; ++mt) { rest[mt][0] = tot[mt][0]; rest[mt][1] = tot[mt][1]; }
        }
        const uint32_t* bc = a.B + (size_t)(n0 + gq) * (16 * KS);
        uint32_t bh[KS][2], bl[KS][2];
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            bh[ks][0] = __ldg(bc + ks * 8 + tq);          bh[ks][1] = __ldg(bc + ks * 8 + 4 + tq);
            bl[ks][0] = __ldg(bc + 8 * KS + ks * 8 + tq); bl[ks][1] = __ldg(bc + 8 * KS + ks * 8 + 4 + tq);
        }
        const float b0 = __ldg(a.bias + n0 + 2 * tq), b1 = __ldg(a.bias + n0 + 2 * tq + 1);
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
            float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) exact_mma(c, A[mt][ks], bh[ks][0], bh[ks][1]);
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) exact_mma(c, A[mt][ks], bl[ks][0], bl[ks][1]);
            tot[mt][0] += (double)(exact_softplus(c[0] + b0) + exact_softplus(c[1] + b1));
            tot[mt][1] += (double)(exact_softplus(c[2] + b0) + exact_softplus(c[3] + b1));
        }
    }
    // the quad's four column partials of each state, then log p* = c.x + tot and g = c.x + rest on lane t = 0
    double lp[4][2];
    double mx = -INFINITY;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            double t = tot[mt][i], r = rest[mt][i];
            t += __shfl_xor_sync(0xffffffffu, t, 1); t += __shfl_xor_sync(0xffffffffu, t, 2);
            r += __shfl_xor_sync(0xffffffffu, r, 1); r += __shfl_xor_sync(0xffffffffu, r, 2);
            const uint32_t off = wofs + mt * 16 + gq + 8 * i;
            lp[mt][i] = -INFINITY;
            if (tq == 0 && off < a.n) {
                const uint32_t s = a.s0 + off;
                double lin = 0.0;
                for (int k = 0; k < a.n_bits; ++k)
                    if ((s >> k) & 1u) lin += __ldg(a.c + k);
                lp[mt][i] = lin + t;
                if (a.g) a.g[off] = lin + r;
                mx = fmax(mx, lp[mt][i]);
            }
        }
    __shared__ double red[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    double M = red[0];
    for (int w = 1; w < 8; ++w) M = fmax(M, red[w]);
    __syncthreads();
    double s = 0.0;
    if (M != -INFINITY) {
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
            for (int i = 0; i < 2; ++i)
                if (lp[mt][i] != -INFINITY) s += exp(lp[mt][i] - M);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double S = 0.0;
        for (int w = 0; w < 8; ++w) S += red[w];
        a.part[blockIdx.x] = make_double2(M, S);
    }
}

struct ExactRowsArgs {
    const uint32_t* Q;              // [rows_pad][24 ks1] words: row r's 3 x 16 ks1 bf16 values, hi, mid and lo of q_r on x_1's bits
    const double* g;                // [n] g of the chunk's states
    int ks1;                        // 16-bit steps of x_1: 1 (n_1 <= 16) or 2
    int rows;
    uint32_t s0, n;                 // the chunk's states s0 .. s0 + n - 1 (g is indexed from s0)
    double2* part;                  // [rows][gridDim.x]
};

// 128 threads; warp w of CTA (x, y) takes rows 64 y + 16 w + [0, 16) (one m16 tile of queries, loaded once) against the states
// [8192 x, 8192 (x + 1)) of the chunk in n8 tiles of keys (B = the bits of each state, three k16 steps per 16 bits).  Lane (g, t)
// keeps a running (max, sum) for rows g and g + 8; the quad merges its four, lane t = 0 writes them.
template <int KS1>
__global__ void __launch_bounds__(128) dbm_exact_rows_kernel(ExactRowsArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
    const int r0 = (blockIdx.y * 4 + warp) * 16;
    if (r0 >= a.rows) return;
    constexpr int W = 24 * KS1;                                   // words per query row
    uint32_t A[3 * KS1][4];
#pragma unroll
    for (int ks = 0; ks < 3 * KS1; ++ks) {
        const uint32_t* q0 = a.Q + (size_t)(r0 + gq) * W + ks * 8;
        const uint32_t* q8 = q0 + (size_t)8 * W;
        A[ks][0] = __ldg(q0 + tq); A[ks][1] = __ldg(q8 + tq); A[ks][2] = __ldg(q0 + 4 + tq); A[ks][3] = __ldg(q8 + 4 + tq);
    }
    double m[2] = {-INFINITY, -INFINITY}, s[2] = {0.0, 0.0};
    const uint32_t lo = blockIdx.x * (uint32_t)EXACT_ROW_STATES, hi = min(lo + (uint32_t)EXACT_ROW_STATES, a.n);
    for (uint32_t t0 = lo; t0 < hi; t0 += 8) {
        const uint32_t key = a.s0 + t0 + gq;                      // column gq of the tile: this lane's B values
        uint32_t b[KS1][2];
#pragma unroll
        for (int ks = 0; ks < KS1; ++ks) { b[ks][0] = exact_bit_pair(key, ks * 16 + 2 * tq); b[ks][1] = exact_bit_pair(key, ks * 16 + 2 * tq + 8); }
        float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int p = 0; p < 3; ++p)
#pragma unroll
            for (int ks = 0; ks < KS1; ++ks) exact_mma(c, A[p * KS1 + ks], b[ks][0], b[ks][1]);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const uint32_t st = t0 + 2 * tq + j;
            if (st >= hi) continue;
            const double gv = __ldg(a.g + st);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const double v = (double)c[2 * i + j] + gv;
                if (v > m[i]) { s[i] = s[i] * (double)expf((float)(m[i] - v)) + 1.0; m[i] = v; }
                else s[i] += (double)expf((float)(v - m[i]));
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            const double m2 = __shfl_xor_sync(0xffffffffu, m[i], o), s2 = __shfl_xor_sync(0xffffffffu, s[i], o);
            exact_lse_merge(m[i], s[i], m2, s2);
        }
    if (tq == 0)
        for (int i = 0; i < 2; ++i) {
            const int r = r0 + gq + 8 * i;
            if (r < a.rows) a.part[(size_t)r * gridDim.x + blockIdx.x] = make_double2(m[i], s[i]);
        }
}

// acc[r] <- acc[r] (+) the n pairs part[r n .. r n + n): thread i merges parts i, i + 256, ... in order, then a fixed tree.
__global__ void __launch_bounds__(256) dbm_exact_merge_kernel(const double2* __restrict__ part, int n, double2* __restrict__ acc) {
    __shared__ double sm[256], ss[256];
    const int r = blockIdx.x, tid = threadIdx.x;
    double m = -INFINITY, s = 0.0;
    for (int i = tid; i < n; i += 256) { const double2 p = part[(size_t)r * n + i]; exact_lse_merge(m, s, p.x, p.y); }
    sm[tid] = m; ss[tid] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (tid < o) { m = sm[tid]; s = ss[tid]; exact_lse_merge(m, s, sm[tid + o], ss[tid + o]); sm[tid] = m; ss[tid] = s; }
        __syncthreads();
    }
    if (tid == 0) { double2 t = acc[r]; exact_lse_merge(t.x, t.y, sm[0], ss[0]); acc[r] = t; }
}

// One warp per row: q = v W_0 (n_1 <= 32 values, lane i sums column i over v in float64), written as three bf16 terms
// hi = bf16(q), mid = bf16(q - hi), lo = bf16(q - hi - mid) into Q's row (16 ks1 values each, zero past n_1); bv[r] = b_v.v.
__global__ void __launch_bounds__(32) dbm_exact_query_kernel(const float* __restrict__ X, int V, const float* __restrict__ W0, int n1,
                                                             const float* __restrict__ vb, int kb1, bf16_t* __restrict__ Q,
                                                             double* __restrict__ bv) {
    const int r = blockIdx.x, lane = threadIdx.x;
    const float* x = X + (size_t)r * V;
    double q = 0.0;
    if (lane < n1)
        for (int v = 0; v < V; ++v) q += (double)x[v] * (double)W0[(size_t)v * n1 + lane];
    const bf16_t h = __float2bfloat16_rn((float)q);
    const double r1 = q - (double)__bfloat162float(h);
    const bf16_t md = __float2bfloat16_rn((float)r1);
    const bf16_t l = __float2bfloat16_rn((float)(r1 - (double)__bfloat162float(md)));
    if (lane < kb1) {
        bf16_t* row = Q + (size_t)r * 3 * kb1;
        row[lane] = h; row[kb1 + lane] = md; row[2 * kb1 + lane] = l;
    }
    double b = 0.0;
    for (int v = lane; v < V; v += 32) b += (double)x[v] * (double)vb[v];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
    if (lane == 0) bv[r] = b;
}

// ---- the engine ------------------------------------------------------------------------------------------------------------
void DbmTC::exact(const void* Xh, int rows, double* log_p_star, double* log_Z) {
    if (v_kind != BM_UNIT_BERNOULLI)
        throw Error(BM_EUNSUPPORTED, "exact log Z and log p(v) are defined for binary layers (Bernoulli visible and hidden units)");
    for (int i = 0; i < L; ++i)
        if (h_kinds[i] != BM_UNIT_BERNOULLI)
            throw Error(BM_EUNSUPPORTED, "exact log Z and log p(v) are defined for binary layers (Bernoulli visible and hidden units)");
    const int NL = L + 1;
    auto width = [&](int j) { return j == 0 ? V : Hs[j - 1]; };
    std::vector<int> bit0(NL, 0);                     // first state bit of each odd layer
    int n_odd = 0;
    for (int j = 1; j < NL; j += 2) { bit0[j] = n_odd; n_odd += width(j); }
    if (n_odd > 32)
        throw Error(BM_EUNSUPPORTED, "exact log Z enumerates the odd layers h_1, h_3, ...: n_odd = " + std::to_string(n_odd) +
                                     " units, at most 32");
    BM_REQUIRE(rows >= 0, "exact: rows must be >= 0");
    BM_REQUIRE(rows == 0 || (Xh && log_p_star), "exact: rows > 0 needs X and log_p_star");
    BM_REQUIRE(rows > 0 || !Xh, "exact: X given with rows = 0");
    BM_REQUIRE(rows > 0 || log_Z, "exact: nothing to compute (rows = 0 and log_Z NULL)");
    const float* X = static_cast<const float*>(Xh);
    for (size_t i = 0; i < (size_t)rows * V; ++i)
        BM_REQUIRE(std::isfinite(X[i]), "exact: X has a non-finite entry");

    // the model as stored (float32 W and biases)
    std::vector<std::vector<float>> Wh(L), bh(NL);
    for (int i = 0; i < L; ++i) {
        Wh[i].resize((size_t)width(i) * width(i + 1));
        BM_CUDA(cudaMemcpyAsync(Wh[i].data(), W[i].p, Wh[i].size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    }
    for (int j = 0; j < NL; ++j) {
        bh[j].resize(width(j));
        BM_CUDA(cudaMemcpyAsync(bh[j].data(), j == 0 ? vb.p : hb[j - 1].p, bh[j].size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    }
    BM_CUDA(cudaStreamSynchronize(ctx->stream));
    // columns: the even layers above v (j = 2, 4, ...), padded to 8, then v, padded to 8
    std::vector<std::pair<int, int>> cols;            // (layer, unit); layer -1: padding
    for (int j = 2; j < NL; j += 2)
        for (int u = 0; u < width(j); ++u) cols.push_back({j, u});
    while (cols.size() % 8) cols.push_back({-1, 0});
    const int n_rest = (int)cols.size();
    for (int u = 0; u < V; ++u) cols.push_back({0, u});
    while (cols.size() % 8) cols.push_back({-1, 0});
    const int n_pad = (int)cols.size();
    const int KS = n_odd <= 16 ? 1 : 2, KB = 16 * KS;
    std::vector<bf16_t> Bop((size_t)n_pad * 2 * KB, __float2bfloat16_rn(0.f));
    std::vector<float> bias(n_pad, -INFINITY);
    std::vector<double> cbit(32, 0.0);
    for (int j = 1; j < NL; j += 2)
        for (int u = 0; u < width(j); ++u) cbit[bit0[j] + u] = (double)bh[j][u];
    for (int n = 0; n < n_pad; ++n) {
        const int e = cols[n].first, c = cols[n].second;
        if (e < 0) continue;
        bias[n] = bh[e][c];
        for (int j = 1; j < NL; j += 2) {             // M[k][n] for the bits k of the odd neighbours of layer e
            if (j != e - 1 && j != e + 1) continue;
            for (int u = 0; u < width(j); ++u) {
                // W_{j}[u][c] (j = e - 1: weights between j and e, [n_j, n_e]) or W_{e}[c][u] (j = e + 1: [n_e, n_j])
                const float w = j == e - 1 ? Wh[j][(size_t)u * width(e) + c] : Wh[e][(size_t)c * width(j) + u];
                const bf16_t whi = __float2bfloat16_rn(w);
                const int k = bit0[j] + u;
                Bop[(size_t)n * 2 * KB + k] = whi;
                Bop[(size_t)n * 2 * KB + KB + k] = __float2bfloat16_rn(w - __bfloat162float(whi));
            }
        }
    }
    DevBuf<bf16_t> Bd; DevBuf<float> biasd; DevBuf<double> cd;
    Bd.ensure(Bop.size()); biasd.ensure(n_pad); cd.ensure(32);
    BM_CUDA(cudaMemcpyAsync(Bd.p, Bop.data(), Bop.size() * sizeof(bf16_t), cudaMemcpyHostToDevice, ctx->stream));
    BM_CUDA(cudaMemcpyAsync(biasd.p, bias.data(), (size_t)n_pad * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    BM_CUDA(cudaMemcpyAsync(cd.p, cbit.data(), 32 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));

    const uint64_t total = 1ull << n_odd;
    const uint32_t chunk = (uint32_t)std::min<uint64_t>(total, 1ull << exact_chunk_bits);
    const int n_cta = (int)((chunk + EXACT_STATES_PER_CTA - 1) / EXACT_STATES_PER_CTA);
    const double2 empty = make_double2(-INFINITY, 0.0);
    DevBuf<double2> spart, accZ;
    spart.ensure(n_cta); accZ.ensure(1);
    BM_CUDA(cudaMemcpyAsync(accZ.p, &empty, sizeof(double2), cudaMemcpyHostToDevice, ctx->stream));
    // the rows: queries, the chunk's g and the rows kernel's pairs
    const int n1 = Hs[0], KS1 = n1 <= 16 ? 1 : 2, KB1 = 16 * KS1;
    const int group = std::min(rows, EXACT_ROW_GROUP);
    const int n_rcta = (int)((chunk + EXACT_ROW_STATES - 1) / EXACT_ROW_STATES);
    DevBuf<float> Xd; DevBuf<bf16_t> Qd; DevBuf<double> bvd, gd; DevBuf<double2> rpart, accR;
    if (rows > 0) {
        const int rows_pad = dbm_round_up(rows, 64);
        Xd.ensure((size_t)rows * V); Qd.ensure((size_t)rows_pad * 3 * KB1); bvd.ensure(rows); gd.ensure(chunk);
        rpart.ensure((size_t)group * n_rcta); accR.ensure(rows);
        Qd.zero(ctx->stream);
        BM_CUDA(cudaMemcpyAsync(Xd.p, X, (size_t)rows * V * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        std::vector<double2> init(rows, empty);
        BM_CUDA(cudaMemcpyAsync(accR.p, init.data(), (size_t)rows * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream));
        dbm_exact_query_kernel<<<rows, 32, 0, ctx->stream>>>(Xd.p, V, W[0].p, n1, vb.p, KB1, Qd.p, bvd.p);
        count_launch(ctx);
        BM_CUDA(cudaStreamSynchronize(ctx->stream));  // `init` is released on leaving this block
    }
    for (uint64_t s0 = 0; s0 < total; s0 += chunk) {
        ExactStatesArgs sa;
        sa.B = reinterpret_cast<const uint32_t*>(Bd.p); sa.bias = biasd.p; sa.c = cd.p; sa.ks = KS;
        sa.n_pad = n_pad; sa.n_rest = n_rest; sa.n_bits = n_odd;
        sa.s0 = (uint32_t)s0; sa.n = chunk; sa.g = rows > 0 ? gd.p : nullptr; sa.part = spart.p;
        if (KS == 1) dbm_exact_states_kernel<1><<<n_cta, 256, 0, ctx->stream>>>(sa);
        else dbm_exact_states_kernel<2><<<n_cta, 256, 0, ctx->stream>>>(sa);
        count_launch(ctx);
        dbm_exact_merge_kernel<<<1, 256, 0, ctx->stream>>>(spart.p, n_cta, accZ.p);
        count_launch(ctx);
        for (int r0 = 0; r0 < rows; r0 += group) {
            const int nr = std::min(group, rows - r0);
            ExactRowsArgs ra;
            ra.Q = reinterpret_cast<const uint32_t*>(Qd.p + (size_t)r0 * 3 * KB1); ra.g = gd.p; ra.ks1 = KS1; ra.rows = nr;
            ra.s0 = (uint32_t)s0; ra.n = chunk; ra.part = rpart.p;
            const dim3 grid(n_rcta, (nr + 63) / 64);
            if (KS1 == 1) dbm_exact_rows_kernel<1><<<grid, 128, 0, ctx->stream>>>(ra);
            else dbm_exact_rows_kernel<2><<<grid, 128, 0, ctx->stream>>>(ra);
            count_launch(ctx);
            dbm_exact_merge_kernel<<<nr, 256, 0, ctx->stream>>>(rpart.p, n_rcta, accR.p + r0);
            count_launch(ctx);
        }
    }
    double2 z;
    BM_CUDA(cudaMemcpyAsync(&z, accZ.p, sizeof(double2), cudaMemcpyDeviceToHost, ctx->stream));
    std::vector<double2> acc(rows);
    std::vector<double> bvh(rows);
    if (rows > 0) {
        BM_CUDA(cudaMemcpyAsync(acc.data(), accR.p, (size_t)rows * sizeof(double2), cudaMemcpyDeviceToHost, ctx->stream));
        BM_CUDA(cudaMemcpyAsync(bvh.data(), bvd.p, (size_t)rows * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    }
    BM_CUDA(cudaStreamSynchronize(ctx->stream));
    if (log_Z) *log_Z = z.x + std::log(z.y);
    for (int r = 0; r < rows; ++r) log_p_star[r] = bvh[r] + acc[r].x + std::log(acc[r].y);
}

}  // namespace bm
