// Tensor-core (wgmma) kernels of the large-state family (d = 16 / 32 / 64): the mean recursions of the shared-model
// LGSSM sweep on the Hopper tensor cores, hand-written PTX (rxg_umma.cuh).
//
//   umma_selftest_kernel<N, K> : D[128 x N] = A[128 x K] * B[N x K]' with the 3xTF32 split -- validates the
//                                descriptors / fragment plumbing of every shape the sweep uses against an fp64 product.
//   umma_ky_kernel<D>          : u_t = K_t y_t for all (t, chain): no dependency along t, so it is a plain batched
//                                GEMM, parallel over time and chain tiles (off the recursion's critical path).
//   lgssm_umma_sweep<D, SMOOTH>: the dependent chain  x_t = F_t x_{t-1} + u_t  (forward) and
//                                mu_s[t] = v_t + G_t mu_s[t+1],  v_t = E_t x_t  (backward).  One CTA = 64 chains =
//                                the M rows of the A operand X[64 x D] (K-major); the forward B operand is the
//                                stacked block [F_t ; E_{t-1}] (N = 2D), so one MMA group yields both x_t and the
//                                backward pass's v_{t-1} from the same A operand.
// A CTA has D / 16 warpgroups; each issues the wgmmas of one N slice of the product and owns that slice's
// accumulator fragments, so the epilogue (fragment + u -> global store, split hi / lo -> next A operand) is
// element-wise in the fragment layout.  The A operand is ping-ponged between two shared-memory buffers: one
// barrier per step separates every warpgroup's reads of step t from the writes of step t + 1.
// Operands are split tf32 hi / lo and combined as hi*hi + hi*lo + lo*hi (3xTF32), accumulated in several register
// accumulators (at most four K = 8 MMAs each) that are summed in fp32 (see DESIGN.md 3.6).
// lgssm_umma_sweep<64, true> is at the 128-register cap of 512 threads and spills 88 bytes (ptxas, sm_90a).
// Per-step gain records are pre-arranged in the canonical K-major layout by large_gain_tables and arrive with one
// TMA bulk copy (cp.async.bulk ... mbarrier::complete_tx) per step, double buffered.
#include "rxg_internal.h"
#include "rxg_umma.cuh"

namespace rxg {

template <int D>
struct US {
    static constexpr int KS = D / 8;                       // MMAs (K = 8) per pass over the K axis
    static constexpr int NHH = (KS + 3) / 4;               // hi*hi accumulators: at most 4 MMAs each
    static constexpr int NACC = NHH + 1;                   // + one for the two cross terms
    static constexpr int ROWS = 64;                        // chains per CTA = M of one wgmma
    static constexpr uint32_t X_BYTES = ROWS * D * 4u;     // one part (hi or lo) of the A operand
    static constexpr uint32_t G_BYTES = (uint32_t)D * D * 4u;       // one part of a D x D gain block
    static constexpr uint32_t FE_BYTES = 2u * G_BYTES;              // one part of [F ; E] (2D x D)
    static constexpr uint32_t SBO = umma::sbo_bytes(D);
    static constexpr int NWG = D / 16;                     // warpgroups per CTA
    static constexpr int NT = 128 * NWG;                   // threads per CTA
};

// this thread's place in the accumulator fragment: rows frow, frow + 8 of the tile; columns n0 + 8 j + fcol + {0, 1}
struct Frag {
    int wg, frow, fcol;
    __device__ Frag() {
        const int tid = threadIdx.x;
        wg = tid >> 7;
        frow = ((tid & 127) >> 5) * 16 + ((tid & 31) >> 2);
        fcol = 2 * (tid & 3);
    }
};

// ------------------------------------------------------------------------------------------------ shared pieces
// one warpgroup: acc = X * W'  (W = the warpgroup's N slice, starting at b_hi / b_lo) as hi*hi (NHH accumulators,
// <= 4 MMAs each) + hi*lo + lo*hi (one accumulator)
template <int D, int NW>
__device__ __forceinline__ void issue_3xtf32(float (&acc)[US<D>::NACC][NW / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                             uint32_t b_lo) {
    using S = US<D>;
    umma::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < S::KS; ++kk)
        umma::mma_tf32<NW>(acc[kk / 4], umma::smem_desc(a_hi + kk * 2 * umma::LBO, umma::LBO, S::SBO),
                           umma::smem_desc(b_hi + kk * 2 * umma::LBO, umma::LBO, S::SBO), (kk % 4) != 0);
#pragma unroll
    for (int kk = 0; kk < S::KS; ++kk)
        umma::mma_tf32<NW>(acc[S::NHH], umma::smem_desc(a_hi + kk * 2 * umma::LBO, umma::LBO, S::SBO),
                           umma::smem_desc(b_lo + kk * 2 * umma::LBO, umma::LBO, S::SBO), kk != 0);
#pragma unroll
    for (int kk = 0; kk < S::KS; ++kk)
        umma::mma_tf32<NW>(acc[S::NHH], umma::smem_desc(a_lo + kk * 2 * umma::LBO, umma::LBO, S::SBO),
                           umma::smem_desc(b_hi + kk * 2 * umma::LBO, umma::LBO, S::SBO), 1u);
    umma::wgmma_commit();
}
// wait for this warpgroup's MMAs and sum the accumulators in fp32 registers (cross terms first: smallest)
template <int D, int NW>
__device__ __forceinline__ void finish_acc(float (&acc)[US<D>::NACC][NW / 2], float* out) {
    using S = US<D>;
    umma::wgmma_wait_all();
#pragma unroll
    for (int a = 0; a < S::NACC; ++a)
#pragma unroll
        for (int i = 0; i < NW / 2; ++i) umma::fence_reg(acc[a][i]);
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) {
        float s = acc[S::NHH][i];
#pragma unroll
        for (int a = 0; a < S::NHH; ++a) s += acc[a][i];
        out[i] = s;
    }
}
// elements (row, col), (row, col + 1) of an A operand with K = D columns: split hi / lo
template <int D>
__device__ __forceinline__ void put_pair(uint8_t* sHi, uint8_t* sLo, int row, int col, float v0, float v1) {
    float2 hi, lo;
    umma::split_tf32(v0, hi.x, lo.x);
    umma::split_tf32(v1, hi.y, lo.y);
    const uint32_t off = umma::elem_off(row, col, D);
    *reinterpret_cast<float2*>(sHi + off) = hi;
    *reinterpret_cast<float2*>(sLo + off) = lo;
}

// ------------------------------------------------------------------------------------------------ self-test
// one warpgroup, both 64-row halves of A, N in slices of 32 (16 when N = 16: both wgmma widths the sweeps issue);
// one accumulator over the three passes
template <int N, int K>
__global__ void __launch_bounds__(128, 1)
umma_selftest_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ Dout) {
    constexpr uint32_t A_BYTES = 128u * K * 4u, B_BYTES = (uint32_t)N * K * 4u;
    extern __shared__ __align__(1024) uint8_t sm[];
    uint8_t* sAhi = sm;
    uint8_t* sAlo = sAhi + A_BYTES;
    uint8_t* sBhi = sAlo + A_BYTES;
    uint8_t* sBlo = sBhi + B_BYTES;
    const int tid = threadIdx.x;
    for (int idx = tid; idx < 128 * K; idx += 128) {
        const int r = idx / K, k = idx % K;
        float hi, lo;
        umma::split_tf32(A[idx], hi, lo);
        *reinterpret_cast<float*>(sAhi + umma::elem_off(r, k, K)) = hi;
        *reinterpret_cast<float*>(sAlo + umma::elem_off(r, k, K)) = lo;
    }
    for (int idx = tid; idx < N * K; idx += 128) {
        const int r = idx / K, k = idx % K;
        float hi, lo;
        umma::split_tf32(B[idx], hi, lo);
        *reinterpret_cast<float*>(sBhi + umma::elem_off(r, k, K)) = hi;
        *reinterpret_cast<float*>(sBlo + umma::elem_off(r, k, K)) = lo;
    }
    umma::fence_async_smem();          // generic-proxy smem writes -> visible to the async (tensor) proxy
    __syncthreads();
    const Frag f;
    const uint32_t sbo = umma::sbo_bytes(K);
    const uint32_t a_hi = (uint32_t)__cvta_generic_to_shared(sAhi), a_lo = (uint32_t)__cvta_generic_to_shared(sAlo);
    const uint32_t b_hi = (uint32_t)__cvta_generic_to_shared(sBhi), b_lo = (uint32_t)__cvta_generic_to_shared(sBlo);
    constexpr int NS = N % 32 == 0 ? 32 : 16;
    for (int h = 0; h < 2; ++h) {
        for (int c = 0; c < N / NS; ++c) {
            float acc[NS / 2];
            umma::wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < 3; ++pass) {
                const uint32_t a0 = (pass == 2 ? a_lo : a_hi) + (uint32_t)h * 8u * sbo;
                const uint32_t bb = (pass == 1 ? b_lo : b_hi) + (uint32_t)c * (NS / 8) * sbo;
#pragma unroll
                for (int kk = 0; kk < K / 8; ++kk)
                    umma::mma_tf32<NS>(acc, umma::smem_desc(a0 + kk * 2 * umma::LBO, umma::LBO, sbo),
                                       umma::smem_desc(bb + kk * 2 * umma::LBO, umma::LBO, sbo), (pass | kk) != 0);
            }
            umma::wgmma_commit();
            umma::wgmma_wait_all();
#pragma unroll
            for (int i = 0; i < NS / 2; ++i) umma::fence_reg(acc[i]);
#pragma unroll
            for (int i = 0; i < NS / 2; ++i) {
                const int row = h * 64 + f.frow + 8 * ((i >> 1) & 1), col = c * NS + 8 * (i >> 2) + f.fcol + (i & 1);
                Dout[row * N + col] = acc[i];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ u_t = K_t y_t
// grid = (chain tiles, time slices); CTA = 64 chains, warpgroup w computes output columns [16 w, 16 w + 16).
// recK[t] = K_t (D x D) hi | lo in the canonical layout.  u is written in the [T][D][batch] layout of the posterior
// means (the sweep consumes u_t from mean[t] before it overwrites that row).
template <int D>
__global__ void __launch_bounds__(US<D>::NT, 1)
umma_ky_kernel(const float* __restrict__ recK, const float* __restrict__ y, float* __restrict__ u, int T, int64_t batch) {
    using S = US<D>;
    constexpr int NW = D / S::NWG, E = NW / 2;
    constexpr uint32_t REC_BYTES = 2 * S::G_BYTES;
    constexpr size_t REC = (size_t)2 * D * D;
    extern __shared__ __align__(1024) uint8_t sm[];
    uint8_t* sY = sm;                              // [2 ping-pong][hi | lo]
    uint8_t* sK0 = sY + 4 * S::X_BYTES;            // two records
    uint64_t* full = reinterpret_cast<uint64_t*>(sK0 + 2 * REC_BYTES);   // [2]
    const int tid = threadIdx.x;
    const Frag f;
    const int n0 = f.wg * NW;
    const int64_t b0 = (int64_t)blockIdx.x * S::ROWS;
    bool act[2];
    int64_t bc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t b = b0 + f.frow + 8 * h;
        act[h] = b < batch;
        bc[h] = act[h] ? b : b0;                   // inactive rows shadow the tile's first chain (never stored)
    }
    const int t_lo = (int)(((int64_t)T * blockIdx.y) / gridDim.y), t_hi = (int)(((int64_t)T * (blockIdx.y + 1)) / gridDim.y);
    if (t_lo >= t_hi) return;
    if (tid == 0) {
        umma::mbar_init(full, 1); umma::mbar_init(full + 1, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // element i = 4 j + 2 h + e: row frow + 8 h, column n0 + 8 j + fcol + e
    auto off = [&](int t, int i) {
        return ((int64_t)t * D + n0 + 8 * (i >> 2) + f.fcol + (i & 1)) * batch + bc[(i >> 1) & 1];
    };
    float yv[E], yn[E];
#pragma unroll
    for (int i = 0; i < E; ++i) yv[i] = __ldg(y + off(t_lo, i));
    __syncthreads();
    const uint32_t y_base = (uint32_t)__cvta_generic_to_shared(sY);
    const uint32_t k_base = (uint32_t)__cvta_generic_to_shared(sK0);
    if (tid == 0) {
        for (int j = 0; j < 2; ++j)
            if (t_lo + j < t_hi) {
                umma::mbar_expect_tx(full + j, REC_BYTES);
                umma::bulk_g2s(sK0 + j * REC_BYTES, recK + (size_t)(t_lo + j) * REC, REC_BYTES, full + j);
            }
    }
    uint32_t use0 = 0, use1 = 0;
    for (int t = t_lo; t < t_hi; ++t) {
        const int i = t - t_lo, p = i & 1, buf = i & 1;
        uint8_t* yhi = sY + 2 * p * S::X_BYTES;
#pragma unroll
        for (int e = 0; e < E; e += 2)
            put_pair<D>(yhi, yhi + S::X_BYTES, f.frow + 8 * ((e >> 1) & 1), n0 + 8 * (e >> 2) + f.fcol, yv[e], yv[e + 1]);
        umma::fence_async_smem();
        __syncthreads();
        if (tid == 0 && i >= 1 && t + 1 < t_hi) {   // every warpgroup is past step t - 1: its K buffer is free
            const int nb = (i + 1) & 1;
            umma::mbar_expect_tx(full + nb, REC_BYTES);
            umma::bulk_g2s(sK0 + nb * REC_BYTES, recK + (size_t)(t + 1) * REC, REC_BYTES, full + nb);
        }
        umma::mbar_wait_bounded(full + buf, buf ? (use1++ & 1) : (use0++ & 1));
        float acc[S::NACC][E];
        const uint32_t a_hi = y_base + 2 * p * S::X_BYTES;
        const uint32_t b_hi = k_base + buf * REC_BYTES + (uint32_t)(n0 / 8) * S::SBO;
        issue_3xtf32<D, NW>(acc, a_hi, a_hi + S::X_BYTES, b_hi, b_hi + S::G_BYTES);
        if (t + 1 < t_hi) {
#pragma unroll
            for (int e = 0; e < E; ++e) yn[e] = __ldg(y + off(t + 1, e));
        }
        float out[E];
        finish_acc<D, NW>(acc, out);
#pragma unroll
        for (int e = 0; e < E; ++e)
            if (act[(e >> 1) & 1]) u[off(t, e)] = out[e];
#pragma unroll
        for (int e = 0; e < E; ++e) yv[e] = yn[e];
    }
}

// ------------------------------------------------------------------------------------------------ the recursion
// mean[t] holds u_t on entry.  Forward step t: D = X_{t-1} [F_t ; E_{t-1}]'  ->  x_t = D[:, :D] + u_t (next A
// operand; stored as the filtered mean when !SMOOTH), v_{t-1} = D[:, D:] (stored into mean[t-1]).  Backward step t:
// mu_s[t] = v_t + mu_s[t+1] G_t' (stored into mean[t]; next A operand).  mu_s[T-1] = x_{T-1}.
// Forward: warpgroup w owns columns [NWF w, NWF (w + 1)) of the 64 x NF product (x columns below D, v columns
// above); backward: columns [NWB w, NWB (w + 1)) of mu_s.
template <int D, bool SMOOTH>
__global__ void __launch_bounds__(US<D>::NT, 1)
lgssm_umma_sweep(const float* __restrict__ recFE, const float* __restrict__ recG, const float* __restrict__ m0,
                 const float* __restrict__ m0c, float* mean, int T, int64_t batch) {
    using S = US<D>;
    constexpr int NF = SMOOTH ? 2 * D : D;                       // forward N
    constexpr int NWF = NF / S::NWG, NWB = D / S::NWG;           // N slice of one warpgroup, forward / backward
    constexpr int EF = NWF / 2, EB = NWB / 2;                    // fragment elements per thread
    constexpr uint32_t FE_REC_BYTES = 2 * S::FE_BYTES, G_REC_BYTES = 2 * S::G_BYTES;
    constexpr size_t FE_REC = (size_t)4 * D * D, G_REC = (size_t)2 * D * D;   // floats per record
    extern __shared__ __align__(1024) uint8_t sm[];
    uint8_t* sX = sm;                              // [2 ping-pong][hi | lo]
    uint8_t* sB0 = sX + 4 * S::X_BYTES;            // two buffers of FE_REC_BYTES
    uint64_t* full = reinterpret_cast<uint64_t*>(sB0 + 2 * FE_REC_BYTES);   // [2]
    const int tid = threadIdx.x;
    const Frag f;
    const int64_t b0 = (int64_t)blockIdx.x * S::ROWS;
    bool act[2];
    int64_t bc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t b = b0 + f.frow + 8 * h;
        act[h] = b < batch;
        bc[h] = act[h] ? b : b0;                   // inactive rows shadow the tile's first chain (never stored)
    }
    const int64_t tstride = (int64_t)D * batch;
    // element i = 4 j + 2 h + e of a slice starting at column n0: row frow + 8 h, column n0 + 8 j + fcol + e
    auto col_of = [&](int n0, int i) { return n0 + 8 * (i >> 2) + f.fcol + (i & 1); };
    // element i of the slice at n0 in mean[t]: one 64-bit column product per 8-column block (fewer live registers)
    auto at = [&](int t, int n0, int i) {
        return mean + t * tstride + bc[(i >> 1) & 1] + (int64_t)(n0 + 8 * (i >> 2) + f.fcol) * batch + ((i & 1) ? batch : 0);
    };
    auto row_of = [&](int i) { return f.frow + 8 * ((i >> 1) & 1); };
    auto xbuf = [&](int p) { return sX + 2 * p * S::X_BYTES; };
    const uint32_t x_base = (uint32_t)__cvta_generic_to_shared(sX);
    const uint32_t b_base = (uint32_t)__cvta_generic_to_shared(sB0);
    if (tid == 0) {
        umma::mbar_init(full, 1); umma::mbar_init(full + 1, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const int n0f = f.wg * NWF;
    // block j of the forward slice holds x columns (n0f + 8 j < D) or v columns; uniform over the warpgroup
    auto is_x = [&](int i) { return !SMOOTH || n0f + 8 * (i >> 2) < D; };
    float cur[EF], nxt[EF];
#pragma unroll
    for (int i = 0; i < EF; i += 2) {
        if (!is_x(i)) continue;
        const int c = col_of(n0f, i);
        float x0, x1;
        if (m0c) {
            x0 = __ldg(m0c + (int64_t)c * batch + bc[(i >> 1) & 1]);
            x1 = __ldg(m0c + (int64_t)(c + 1) * batch + bc[(i >> 1) & 1]);
        } else {
            x0 = m0[c]; x1 = m0[c + 1];
        }
        put_pair<D>(xbuf(0), xbuf(0) + S::X_BYTES, row_of(i), c, x0, x1);
        cur[i] = *at(0, n0f, i);                                // u_0
        cur[i + 1] = *at(0, n0f, i + 1);
    }
    umma::fence_async_smem();
    __syncthreads();
    if (tid == 0) {
        for (int j = 0; j < 2; ++j)
            if (j < T) {
                umma::mbar_expect_tx(full + j, FE_REC_BYTES);
                umma::bulk_g2s(sB0 + j * FE_REC_BYTES, recFE + (size_t)j * FE_REC, FE_REC_BYTES, full + j);
            }
    }
    uint32_t use0 = 0, use1 = 0;
    // ---------------------------------------------------------------- forward
    for (int t = 0; t < T; ++t) {
        const int p = t & 1, buf = t & 1;
        if (t > 0) {
            umma::fence_async_smem();              // this thread's A-operand pieces -> visible to the tensor (async) proxy
            __syncthreads();
            if (tid == 0 && t + 1 < T) {           // every warpgroup is past step t - 1: its B buffer is free
                const int nb = (t + 1) & 1;
                umma::mbar_expect_tx(full + nb, FE_REC_BYTES);
                umma::bulk_g2s(sB0 + nb * FE_REC_BYTES, recFE + (size_t)(t + 1) * FE_REC, FE_REC_BYTES, full + nb);
            }
        }
        umma::mbar_wait_bounded(full + buf, buf ? (use1++ & 1) : (use0++ & 1));
        float acc[S::NACC][EF];
        const uint32_t a_hi = x_base + 2 * p * S::X_BYTES;
        const uint32_t b_hi = b_base + buf * FE_REC_BYTES + (uint32_t)(n0f / 8) * S::SBO;
        issue_3xtf32<D, NWF>(acc, a_hi, a_hi + S::X_BYTES, b_hi, b_hi + S::FE_BYTES);
        if (t + 1 < T) {
#pragma unroll
            for (int i = 0; i < EF; ++i)
                if (is_x(i)) nxt[i] = *at(t + 1, n0f, i);     // u_{t+1}
        }
        float out[EF];
        finish_acc<D, NWF>(acc, out);
        uint8_t* xn = xbuf(p ^ 1);                 // next step's A operand (and the backward pass's first one)
#pragma unroll
        for (int i = 0; i < EF; i += 2) {
            const int c = col_of(n0f, i);
            if (is_x(i)) {
                const float x0 = out[i] + cur[i], x1 = out[i + 1] + cur[i + 1];
                put_pair<D>(xn, xn + S::X_BYTES, row_of(i), c, x0, x1);
                if (act[(i >> 1) & 1] && (!SMOOTH || t == T - 1)) {      // filtered mean, or mu_s[T-1] = x_{T-1}
                    *at(t, n0f, i) = x0;
                    *at(t, n0f, i + 1) = x1;
                }
            } else if (t >= 1 && act[(i >> 1) & 1]) {                    // v_{t-1} = E_{t-1} x_{t-1}
                *at(t - 1, n0f - D, i) = out[i];
                *at(t - 1, n0f - D, i + 1) = out[i + 1];
            }
        }
#pragma unroll
        for (int i = 0; i < EF; ++i) cur[i] = nxt[i];
    }
    if (SMOOTH) {
        // ------------------------------------------------------------ backward
        const int n0b = f.wg * NWB;
        float curb[EB], nxtb[EB];
        umma::fence_async_smem();
        __syncthreads();                           // forward MMAs complete, v_{T-2} stored
        if (tid == 0) {
            for (int j = 0; j < 2; ++j)
                if (T - 2 - j >= 0) {
                    umma::mbar_expect_tx(full + j, G_REC_BYTES);
                    umma::bulk_g2s(sB0 + j * FE_REC_BYTES, recG + (size_t)(T - 2 - j) * G_REC, G_REC_BYTES, full + j);
                }
        }
        if (T >= 2) {
#pragma unroll
            for (int i = 0; i < EB; ++i) curb[i] = *at(T - 2, n0b, i);                    // v_{T-2}
        }
        for (int r = 0; T - 2 - r >= 0; ++r) {
            const int t = T - 2 - r, p = (T + r) & 1, buf = r & 1;
            if (r > 0) {
                umma::fence_async_smem();
                __syncthreads();
                if (tid == 0 && t - 1 >= 0) {
                    const int nb = (r + 1) & 1;
                    umma::mbar_expect_tx(full + nb, G_REC_BYTES);
                    umma::bulk_g2s(sB0 + nb * FE_REC_BYTES, recG + (size_t)(t - 1) * G_REC, G_REC_BYTES, full + nb);
                }
            }
            umma::mbar_wait_bounded(full + buf, buf ? (use1++ & 1) : (use0++ & 1));
            float acc[S::NACC][EB];
            const uint32_t a_hi = x_base + 2 * p * S::X_BYTES;
            const uint32_t b_hi = b_base + buf * FE_REC_BYTES + (uint32_t)(n0b / 8) * S::SBO;
            issue_3xtf32<D, NWB>(acc, a_hi, a_hi + S::X_BYTES, b_hi, b_hi + S::G_BYTES);
            if (t - 1 >= 0) {
#pragma unroll
                for (int i = 0; i < EB; ++i) nxtb[i] = *at(t - 1, n0b, i);               // v_{t-1}
            }
            float out[EB];
            finish_acc<D, NWB>(acc, out);
            uint8_t* xn = xbuf(p ^ 1);
#pragma unroll
            for (int i = 0; i < EB; i += 2) {
                const int c = col_of(n0b, i);
                const float x0 = out[i] + curb[i], x1 = out[i + 1] + curb[i + 1];
                if (t > 0) put_pair<D>(xn, xn + S::X_BYTES, row_of(i), c, x0, x1);
                if (act[(i >> 1) & 1]) {
                    *at(t, n0b, i) = x0;
                    *at(t, n0b, i + 1) = x1;
                }
            }
#pragma unroll
            for (int i = 0; i < EB; ++i) curb[i] = nxtb[i];
        }
    }
}

template <int D>
static int launch_umma_sweep_d(rxg_ctx* ctx, bool smooth, const float* recFE, const float* recG, const float* recK,
                               const float* m0, const float* m0c, const float* y, float* mean, int T, int64_t batch) {
    using S = US<D>;
    const size_t smem_ky = 4 * S::X_BYTES + 4 * S::G_BYTES + 16;
    const size_t smem_sw = 4 * S::X_BYTES + 4 * S::FE_BYTES + 16;
    {   // per-device attributes: set on every call
        RXG_CUDA(ctx, cudaFuncSetAttribute(umma_ky_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ky));
        RXG_CUDA(ctx, cudaFuncSetAttribute(lgssm_umma_sweep<D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sw));
        RXG_CUDA(ctx, cudaFuncSetAttribute(lgssm_umma_sweep<D, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sw));
    }
    const unsigned tiles = (unsigned)((batch + S::ROWS - 1) / S::ROWS);
    // time slices of the K y pre-pass: about two CTAs per SM in flight overall
    int tsplit = (int)((2 * (unsigned)ctx->sm_count + tiles - 1) / tiles);
    if (tsplit < 1) tsplit = 1;
    if (tsplit > T) tsplit = T;
    umma_ky_kernel<D><<<dim3(tiles, (unsigned)tsplit), S::NT, smem_ky, ctx->stream>>>(recK, y, mean, T, batch);
    if (smooth) lgssm_umma_sweep<D, true><<<tiles, S::NT, smem_sw, ctx->stream>>>(recFE, recG, m0, m0c, mean, T, batch);
    else        lgssm_umma_sweep<D, false><<<tiles, S::NT, smem_sw, ctx->stream>>>(recFE, recG, m0, m0c, mean, T, batch);
    ctx->launches += 2;
    return check_cuda(ctx, cudaGetLastError(), "lgssm_umma_sweep");
}

int launch_umma_sweep(rxg_ctx* ctx, int d, bool smooth, const float* recFE, const float* recG, const float* recK,
                      const float* m0, const float* m0c, const float* y, float* mean, int T, int64_t batch) {
    switch (d) {
        case 16: return launch_umma_sweep_d<16>(ctx, smooth, recFE, recG, recK, m0, m0c, y, mean, T, batch);
        case 32: return launch_umma_sweep_d<32>(ctx, smooth, recFE, recG, recK, m0, m0c, y, mean, T, batch);
        case 64: return launch_umma_sweep_d<64>(ctx, smooth, recFE, recG, recK, m0, m0c, y, mean, T, batch);
        default: return fail(ctx, RXG_ERR_UNSUPPORTED, "umma sweep: d=%d", d);
    }
}

template <int N, int K>
static int run_selftest(rxg_ctx* ctx, const float* A, const float* B, float* D) {
    const size_t smem = 2 * (size_t)128 * K * 4 + 2 * (size_t)N * K * 4;
    RXG_CUDA(ctx, cudaFuncSetAttribute(umma_selftest_kernel<N, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    umma_selftest_kernel<N, K><<<1, 128, smem, ctx->stream>>>(A, B, D);
    ctx->launches += 1;
    int rc = check_cuda(ctx, cudaGetLastError(), "umma_selftest_kernel");
    if (rc != RXG_OK) return rc;
    RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

}  // namespace rxg

using namespace rxg;

extern "C" int rxg_selftest_umma_shape_f32(rxg_ctx* ctx, int n, int k, const float* A, const float* B, float* D,
                                           unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE) || !A || !B || !D) return fail(ctx, RXG_ERR_BAD_ARG, "selftest_umma: device pointers required");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    switch (n * 1000 + k) {
        case 64 * 1000 + 128: return run_selftest<64, 128>(ctx, A, B, D);
        case 128 * 1000 + 64: return run_selftest<128, 64>(ctx, A, B, D);
        case 64 * 1000 + 64: return run_selftest<64, 64>(ctx, A, B, D);
        case 64 * 1000 + 32: return run_selftest<64, 32>(ctx, A, B, D);
        case 32 * 1000 + 32: return run_selftest<32, 32>(ctx, A, B, D);
        case 32 * 1000 + 16: return run_selftest<32, 16>(ctx, A, B, D);
        case 16 * 1000 + 16: return run_selftest<16, 16>(ctx, A, B, D);
        default: return fail(ctx, RXG_ERR_UNSUPPORTED, "selftest_umma: shape (N=%d, K=%d) is not one the sweeps use", n, k);
    }
}

extern "C" int rxg_selftest_umma_f32(rxg_ctx* ctx, const float* A, const float* B, float* D, unsigned flags) {
    return rxg_selftest_umma_shape_f32(ctx, 64, 128, A, B, D, flags);
}
