// lgssm_cluster_sweep_kernel: the shared-model smoothing sweep with y read from HBM exactly once.
//
// The mean recursions of the gain-table path are affine in the state with data-independent matrices,
//     forward   x_t      = F_t x_{t-1} + K_t y_t                 (rules #1-#4 + product at x_t)
//     backward  mu_s[t]  = E_t x_t + G_t mu_s[t+1]               (rules #3', #4 + 3-way marginal; G_{T-1} = 0)
// so a sub-segment [a, e] of L steps maps its incoming carry affinely:
//     x_e     = Phi x_{a-1} + c ,       Phi = F_e ... F_a ,   c = the forward recursion from a zero carry
//     mu_s[a] = Psi mu_s[e+1] + b ,     Psi = G_a ... G_e ,   b = the backward recursion from a zero carry
// Phi and Psi depend on the model only (cluster_tables_kernel, once per call).
//
// One thread-block cluster of CL_CTAS CTAs owns 32 consecutive chains (lane = chain) for all T steps; CTA r owns the
// time slice [r S, (r + 1) S), S = SPC L, and its CL_WARPS warps take its SPC sub-segments round robin.  Per CTA:
//   load     y of the slice (S x m x 32 floats) and the slice's F, K, E, G records into shared memory with cp.async:
//            the only read of y.  While those copies are in flight the CTA writes its span of the per-chain
//            covariances (store_cov_span; PEER: in pass D instead).
//   pass A   the zero-carry forward recursion of every sub-segment                           -> c
//   scan     forward carries in two levels: inside the CTA through shared memory, across the cluster through
//            distributed shared memory (each CTA's slice offset, read by the later CTAs between two cluster barriers)
//   pass B   the forward recursion from the true carry; mu_f[t] overwrites y_t in shared memory (m >= d)
//   pass C   the zero-carry backward recursion of every sub-segment over the stored mu_f    -> b
//   scan     backward carries, the same two levels in the other direction
//   pass D   the backward recursion from the true carry; stores the smoothed means (streaming stores)
// The covariances are chain independent (every cov[t][i][j][.] is Sigma_s[t][i][j]), so they need not follow the chain
// tiles: CTA k writes the k-th contiguous span of the flattened buffer as 16-byte streaming stores.  Written per tile in
// pass D instead, they were 128-byte pieces 256 KiB apart from CTAs that drift apart in time (the pattern of
// rxg_lgssm_seg.cuh's header, DESIGN 3.8), two thirds of the kernel's bytes.
// HBM traffic per (chain, step) is 4 (m + d + d^2) bytes, the algorithmic 96 B at d = m = 4 (lgssm_shared_kernel's
// checkpoint variant: ~115 B, it reads y twice and writes / reads a checkpoint per 12 steps).  The only synchronisation
// is __syncthreads and the cluster barrier; the hardware co-schedules the CTAs of a cluster.
#pragma once
#include <cooperative_groups.h>

#include "rxg_lgssm_common.cuh"
#include "rxg_lgssm_shared.cuh"

namespace rxg {

constexpr int CL_CTAS = 8;      // CTAs per cluster (portable cluster size)
constexpr int CL_WARPS = 8;     // warps per CTA
constexpr int CL_L = 16;        // steps per sub-segment

template <int D, int M>
struct ClusterTab {
    static constexpr int FK = pad4(D * D) + pad4(D * M);     // staged prefix of a forward record: F_t, K_t
    static constexpr int EG = 2 * pad4(D * D);               // staged prefix of a backward record: E_t, G_t
    static constexpr int REC = 2 * pad4(D * D);              // scan record (per sub-segment and per slice): Phi, Psi
    static constexpr int PSI_OFF = pad4(D * D);
    static_assert(Tab<D, M>::F_OFF == 0 && Tab<D, M>::K_OFF == pad4(D * D) && Tab<D, M>::E_OFF == 0 &&
                      Tab<D, M>::G_OFF == pad4(D * D),
                  "the staged prefixes are the first FK / EG floats of the gain records");

    // geometry of a call: sub-segments per CTA slice
    static __host__ __device__ int spc(int T) { return ((T + CL_L - 1) / CL_L + CL_CTAS - 1) / CL_CTAS; }
    // scan records: CL_CTAS * spc per sub-segment, then CL_CTAS per slice
    static size_t table_floats(int T) { return (size_t)(CL_CTAS * spc(T) + CL_CTAS) * REC; }
    // dynamic shared memory of one CTA
    static size_t smem_bytes(int T) {
        const size_t S = (size_t)spc(T) * CL_L;
        return 4 * (S * (M * 32 + FK + EG) + (size_t)(spc(T) + CL_CTAS) * REC + (size_t)spc(T) * D * 32 + 2 * D * 32);
    }
};

// Phi / Psi of every sub-segment and of every CTA slice, fp64 products of the fp32 records the sweep runs on.  One
// CTA; sub-segments past T are empty (Phi = Psi = I).
template <int D, int M>
__global__ void __launch_bounds__(256) cluster_tables_kernel(GainWs ws, float* __restrict__ tab, int T, int spc) {
    using TB = Tab<D, M>;
    using CT = ClusterTab<D, M>;
    const int nsub = CL_CTAS * spc;
    for (int j = threadIdx.x; j < nsub; j += blockDim.x) {
        const int a = j * CL_L, e = min(a + CL_L, T);
        Mat<double, D, D> Phi = identity<double, D>(), Psi = identity<double, D>();
        for (int t = a; t < e; ++t) {
            Phi = mul(load_const<double, D, D>(ws.fwd + (size_t)t * TB::FWD_REC + TB::F_OFF), Phi);
            Psi = mul(Psi, load_const<double, D, D>(ws.bwd + (size_t)t * TB::BWD_REC + TB::G_OFF));
        }
        store_f(tab + (size_t)j * CT::REC, Phi);
        store_f(tab + (size_t)j * CT::REC + CT::PSI_OFF, Psi);
    }
    __syncthreads();
    for (int r = threadIdx.x; r < CL_CTAS; r += blockDim.x) {
        Mat<double, D, D> Phi = identity<double, D>(), Psi = identity<double, D>();
        for (int j = r * spc; j < (r + 1) * spc; ++j) {
            Phi = mul(load_const<double, D, D>(tab + (size_t)j * CT::REC), Phi);
            Psi = mul(Psi, load_const<double, D, D>(tab + (size_t)j * CT::REC + CT::PSI_OFF));
        }
        store_f(tab + (size_t)(nsub + r) * CT::REC, Phi);
        store_f(tab + (size_t)(nsub + r) * CT::REC + CT::PSI_OFF, Psi);
    }
}

// v = Mx v + w   (Mx: D x D row-major in shared memory, broadcast reads)
template <int D>
__device__ __forceinline__ void affine_step(const float* Mx, float (&v)[D], const float (&w)[D]) {
    float Mr[pad4(D * D)];
    load_smem<pad4(D * D)>(Mx, Mr);
    float n[D];
#pragma unroll
    for (int i = 0; i < D; ++i) {
        float a = w[i];
#pragma unroll
        for (int j = 0; j < D; ++j) a = __fmaf_rn(Mr[i * D + j], v[j], a);
        n[i] = a;
    }
#pragma unroll
    for (int i = 0; i < D; ++i) v[i] = n[i];
}

// This CTA's span of the per-chain covariances.  Every chain's copy of cov[t][i][j][.] is the table entry
// Sigma_s[t][i][j] (the SS record of bwd_tab), so the bytes may be written in any order: CTA k owns the contiguous
// float4s [k D^2 T, (k + 1) D^2 T) of the flattened cov[T][D][D][batch] (the grid has batch / 32 * CL_CTAS CTAs, so the
// spans tile the buffer; batch % 32 == 0, so a float4 never straddles a row).  Thread-strided 16-byte streaming stores;
// each thread tracks its row incrementally (one 64-bit division per thread) and reloads the entry only when its row
// changes: at most twice at 65 536 chains, where a span covers at most two 256 KiB rows.
template <int D, int M>
__device__ __forceinline__ void store_cov_span(const float* __restrict__ bwd_tab, float* __restrict__ cov, int64_t batch,
                                               int T) {
    using TB = Tab<D, M>;
    constexpr int NT = 32 * CL_WARPS;
    const int n4 = (int)(batch / 4);                       // float4s per row
    const int span = D * D * T;                            // float4s per CTA
    const int64_t base = (int64_t)blockIdx.x * span;
    float4* out = reinterpret_cast<float4*>(cov) + base;
    const int step_rows = NT / n4, step_cols = NT % n4;
    int i = (int)threadIdx.x;
    const int64_t q = base + i;
    int row = (int)(q / n4), col = (int)(q - (int64_t)row * n4);
    int cur = -1;
    float4 v = {};
    for (; i < span; i += NT) {
        if (row != cur) {
            cur = row;
            const float s = bwd_tab[(size_t)(row / (D * D)) * TB::BWD_REC + TB::SS_OFF + row % (D * D)];
            v = make_float4(s, s, s, s);
        }
        __stcs(out + i, v);
        row += step_rows;
        col += step_cols;
        if (col >= n4) { col -= n4; ++row; }
    }
}

// PEER: the smoothed posteriors are also stored to the peer ranks' gathered buffers (fused all-gather, rxg_peer.cu),
// so that a fused gather returns the bits of the plain sweep.
template <int D, int M, bool PEER>
__global__ void __launch_bounds__(32 * CL_WARPS, 2)
lgssm_cluster_sweep_kernel(const float* __restrict__ fwd_tab, const float* __restrict__ bwd_tab,
                           const float* __restrict__ cl_tab, const float* __restrict__ y, float* __restrict__ mean,
                           float* __restrict__ cov, int T, int64_t batch, int write_cov,
                           const __grid_constant__ ModelF<D, M> mdl, const __grid_constant__ PeerOut po) {
    static_assert(M >= D, "pass B stores mu_f[t] over y_t");
    using TB = Tab<D, M>;
    using CT = ClusterTab<D, M>;
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const int r = (int)cluster.block_rank();
    const int spc = CT::spc(T);
    const int S = spc * CL_L;
    const int t0 = r * S;                                  // first step of this CTA's slice
    const int nt = max(0, min(S, T - t0));                 // steps of the slice inside [0, T)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t b = ((int64_t)blockIdx.x / CL_CTAS) * 32 + lane;

    extern __shared__ __align__(16) float smem[];
    float* s_y = smem;                                     // [S][M][32]: y_t, then mu_f[t] in rows 0..D-1
    float* s_fk = s_y + (size_t)S * M * 32;                // [S][FK]
    float* s_eg = s_fk + (size_t)S * CT::FK;               // [S][EG]
    float* s_sub = s_eg + (size_t)S * CT::EG;              // [spc][REC]: this slice's sub-segments
    float* s_slice = s_sub + (size_t)spc * CT::REC;        // [CL_CTAS][REC]: every slice of the cluster
    float* s_car = s_slice + CL_CTAS * CT::REC;            // [spc][D][32]: sub-segment offsets, then carries
    float* s_off = s_car + (size_t)spc * D * 32;           // [2][D][32]: slice offsets (read by the other CTAs)

    // ---------------------------------------------------------------- load (the only read of y)
    {
        const int tid = threadIdx.x;
        for (int p = tid; p < nt * M * 8; p += 32 * CL_WARPS) {          // 8 pieces of 16 B per (t, k) row
            const int row = p >> 3, part = p & 7;
            cp_async16(s_y + row * 32 + part * 4, y + ((int64_t)t0 * M + row) * batch + (b - lane) + part * 4);
        }
        for (int p = tid; p < nt * (CT::FK / 4); p += 32 * CL_WARPS) {
            const int s = p / (CT::FK / 4), part = p % (CT::FK / 4);
            cp_async16(s_fk + s * CT::FK + part * 4, fwd_tab + (size_t)(t0 + s) * TB::FWD_REC + part * 4);
        }
        for (int p = tid; p < nt * (CT::EG / 4); p += 32 * CL_WARPS) {
            const int s = p / (CT::EG / 4), part = p % (CT::EG / 4);
            cp_async16(s_eg + s * CT::EG + part * 4, bwd_tab + (size_t)(t0 + s) * TB::BWD_REC + part * 4);
        }
        for (int p = tid; p < spc * (CT::REC / 4); p += 32 * CL_WARPS)
            cp_async16(s_sub + p * 4, cl_tab + (size_t)r * spc * CT::REC + p * 4);
        for (int p = tid; p < CL_CTAS * (CT::REC / 4); p += 32 * CL_WARPS)
            cp_async16(s_slice + p * 4, cl_tab + (size_t)CL_CTAS * spc * CT::REC + p * 4);
        cp_async_commit();
        if (!PEER && write_cov) store_cov_span<D, M>(bwd_tab, cov, batch, T);
        cp_async_wait<0>();
    }
    __syncthreads();

    auto car = [&](int j, int i) -> float& { return s_car[((size_t)j * D + i) * 32 + lane]; };
    auto off = [&](float* base, int dir, int i) -> float& { return base[(dir * D + i) * 32 + lane]; };

    // ---------------------------------------------------------------- pass A: zero-carry forward offsets
    for (int j = warp; j < spc; j += CL_WARPS) {
        float x[D];
#pragma unroll
        for (int i = 0; i < D; ++i) x[i] = 0.f;
#pragma unroll
        for (int q = 0; q < CL_L; ++q) {
            const int s = j * CL_L + q;
            if (s < nt) {
                float Ft[pad4(D * D)], Kt[pad4(D * M)];
                load_smem<pad4(D * D)>(s_fk + s * CT::FK, Ft);
                load_smem<pad4(D * M)>(s_fk + s * CT::FK + pad4(D * D), Kt);
                float nx[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    float a = Ft[i * D] * x[0];
#pragma unroll
                    for (int jj = 1; jj < D; ++jj) a = __fmaf_rn(Ft[i * D + jj], x[jj], a);
#pragma unroll
                    for (int k = 0; k < M; ++k) a = __fmaf_rn(Kt[i * M + k], s_y[(s * M + k) * 32 + lane], a);
                    nx[i] = a;
                }
#pragma unroll
                for (int i = 0; i < D; ++i) x[i] = nx[i];
            }
        }
#pragma unroll
        for (int i = 0; i < D; ++i) car(j, i) = x[i];
    }
    __syncthreads();

    // ---------------------------------------------------------------- forward carries
    if (warp == 0) {
        float z[D];
#pragma unroll
        for (int i = 0; i < D; ++i) z[i] = 0.f;
        for (int j = 0; j < spc; ++j) {
            float c[D];
#pragma unroll
            for (int i = 0; i < D; ++i) c[i] = car(j, i);
            affine_step<D>(s_sub + j * CT::REC, z, c);
        }
#pragma unroll
        for (int i = 0; i < D; ++i) off(s_off, 0, i) = z[i];
    }
    cluster.sync();
    if (warp == 0) {
        float x[D];                                        // filtered mean before the slice: the prior, then slices 0..r-1
#pragma unroll
        for (int i = 0; i < D; ++i) x[i] = mdl.m0[i];
        for (int q = 0; q < r; ++q) {
            float* rem = cluster.map_shared_rank(s_off, q);
            float c[D];
#pragma unroll
            for (int i = 0; i < D; ++i) c[i] = off(rem, 0, i);
            affine_step<D>(s_slice + q * CT::REC, x, c);
        }
        for (int j = 0; j < spc; ++j) {
            float c[D];
#pragma unroll
            for (int i = 0; i < D; ++i) { c[i] = car(j, i); car(j, i) = x[i]; }
            affine_step<D>(s_sub + j * CT::REC, x, c);
        }
    }
    __syncthreads();

    // ---------------------------------------------------------------- pass B (filtered means over y) + pass C
    for (int j = warp; j < spc; j += CL_WARPS) {
        float x[D];
#pragma unroll
        for (int i = 0; i < D; ++i) x[i] = car(j, i);
#pragma unroll
        for (int q = 0; q < CL_L; ++q) {
            const int s = j * CL_L + q;
            if (s < nt) {
                float Ft[pad4(D * D)], Kt[pad4(D * M)], yt[M];
                load_smem<pad4(D * D)>(s_fk + s * CT::FK, Ft);
                load_smem<pad4(D * M)>(s_fk + s * CT::FK + pad4(D * D), Kt);
#pragma unroll
                for (int k = 0; k < M; ++k) yt[k] = s_y[(s * M + k) * 32 + lane];
                float nx[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    float a = Ft[i * D] * x[0];
#pragma unroll
                    for (int jj = 1; jj < D; ++jj) a = __fmaf_rn(Ft[i * D + jj], x[jj], a);
#pragma unroll
                    for (int k = 0; k < M; ++k) a = __fmaf_rn(Kt[i * M + k], yt[k], a);
                    nx[i] = a;
                }
#pragma unroll
                for (int i = 0; i < D; ++i) { x[i] = nx[i]; s_y[(s * M + i) * 32 + lane] = nx[i]; }
            }
        }
        float v[D];
#pragma unroll
        for (int i = 0; i < D; ++i) v[i] = 0.f;
#pragma unroll
        for (int q = CL_L - 1; q >= 0; --q) {
            const int s = j * CL_L + q;
            if (s < nt) {
                float Et[pad4(D * D)], Gt[pad4(D * D)];
                load_smem<pad4(D * D)>(s_eg + s * CT::EG, Et);
                load_smem<pad4(D * D)>(s_eg + s * CT::EG + pad4(D * D), Gt);
                float nv[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    float a = Et[i * D] * s_y[(s * M) * 32 + lane];
#pragma unroll
                    for (int jj = 1; jj < D; ++jj) a = __fmaf_rn(Et[i * D + jj], s_y[(s * M + jj) * 32 + lane], a);
#pragma unroll
                    for (int jj = 0; jj < D; ++jj) a = __fmaf_rn(Gt[i * D + jj], v[jj], a);
                    nv[i] = a;
                }
#pragma unroll
                for (int i = 0; i < D; ++i) v[i] = nv[i];
            }
        }
#pragma unroll
        for (int i = 0; i < D; ++i) car(j, i) = v[i];
    }
    __syncthreads();

    // ---------------------------------------------------------------- backward carries
    if (warp == 0) {
        float z[D];
#pragma unroll
        for (int i = 0; i < D; ++i) z[i] = 0.f;
        for (int j = spc - 1; j >= 0; --j) {
            float c[D];
#pragma unroll
            for (int i = 0; i < D; ++i) c[i] = car(j, i);
            affine_step<D>(s_sub + j * CT::REC + CT::PSI_OFF, z, c);
        }
#pragma unroll
        for (int i = 0; i < D; ++i) off(s_off, 1, i) = z[i];
    }
    cluster.sync();
    if (warp == 0) {
        float v[D];                                        // smoothed mean after the slice: slices CL_CTAS-1 .. r+1
#pragma unroll
        for (int i = 0; i < D; ++i) v[i] = 0.f;
        for (int q = CL_CTAS - 1; q > r; --q) {
            float* rem = cluster.map_shared_rank(s_off, q);
            float c[D];
#pragma unroll
            for (int i = 0; i < D; ++i) c[i] = off(rem, 1, i);
            affine_step<D>(s_slice + q * CT::REC + CT::PSI_OFF, v, c);
        }
        for (int j = spc - 1; j >= 0; --j) {
            float c[D];
#pragma unroll
            for (int i = 0; i < D; ++i) { c[i] = car(j, i); car(j, i) = v[i]; }
            affine_step<D>(s_sub + j * CT::REC + CT::PSI_OFF, v, c);
        }
    }
    // done with the other CTAs' shared memory; the matching wait is the last thing this CTA does
    asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
    __syncthreads();

    // ---------------------------------------------------------------- pass D: smoothed means and covariances
    for (int j = warp; j < spc; j += CL_WARPS) {
        float v[D][1];
#pragma unroll
        for (int i = 0; i < D; ++i) v[i][0] = car(j, i);
#pragma unroll
        for (int q = CL_L - 1; q >= 0; --q) {
            const int s = j * CL_L + q;
            if (s < nt) {
                const int t = t0 + s;
                float Et[pad4(D * D)], Gt[pad4(D * D)];
                load_smem<pad4(D * D)>(s_eg + s * CT::EG, Et);
                load_smem<pad4(D * D)>(s_eg + s * CT::EG + pad4(D * D), Gt);
                float nv[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    float a = Et[i * D] * s_y[(s * M) * 32 + lane];
#pragma unroll
                    for (int jj = 1; jj < D; ++jj) a = __fmaf_rn(Et[i * D + jj], s_y[(s * M + jj) * 32 + lane], a);
#pragma unroll
                    for (int jj = 0; jj < D; ++jj) a = __fmaf_rn(Gt[i * D + jj], v[jj][0], a);
                    nv[i] = a;
                }
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    v[i][0] = nv[i];
                    __stcs(mean + ((int64_t)t * D + i) * batch + b, nv[i]);
                }
                if constexpr (PEER) {
                    float Sst[pad4(D * D)];
                    if (write_cov) {
                        load_uniform<pad4(D * D)>(bwd_tab + (size_t)t * TB::BWD_REC + TB::SS_OFF, Sst);
#pragma unroll
                        for (int i = 0; i < D * D; ++i) __stcs(cov + ((int64_t)t * D * D + i) * batch + b, Sst[i]);
                    }
                    peer_store<D, 1>(po, write_cov, t, batch, b, v, Sst);
                }
            }
        }
    }
    asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

}  // namespace rxg
