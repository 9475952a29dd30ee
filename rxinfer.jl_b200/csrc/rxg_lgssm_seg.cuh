// lgssm_seg_kernel: the shared-model smoothing sweep, parallel in TIME inside each chain tile.
//
// The mean recursions of the gain-table path are affine in the state with data-independent matrices,
//     forward   x_t      = F_t x_{t-1} + K_t y_t + gf_t            (rules #1-#4 + product at x_t)
//     backward  mu_s[t]  = E_t x_t + G_t mu_s[t+1] + gb_t          (rules #3', #4 + 3-way marginal)
// so a time segment [a, e] can be summarised by two vectors that are LINEAR in its own observations,
//     x_e      = Phi_s x_{a-1} + c_s ,                c_s = sum_t Nf_t y_t + cf_s
//     mu_s[a]  = Psi_s mu_s[e+1] + Omega_s x_{a-1} + b_s ,   b_s = sum_t Nb_t y_t + cb_s
// with Phi_s, Psi_s, Omega_s, Nf_t, Nb_t, cf_s, cb_s functions of the model only (seg_tables_kernel, fp64).
// One CTA owns 32 chains for all T and runs, per tile,
//   pass A   every warp takes segments of L = 16 steps: loads the segment's y (64 independent, coalesced 128-byte
//            loads per thread) and reduces it to (c_s, b_s)                                 -> shared memory
//   scan     one warp (lane = chain) runs the two segment-level recursions over the T/L summaries and leaves
//            x_{a-1} and mu_s[e+1] of every segment in place
//   pass B   every warp re-reads the y of its segments, runs the forward recursion of the segment from the true
//            x_{a-1} (the 16 filtered means stay in registers), then the backward recursion from the true
//            mu_s[e+1], and stores the smoothed means and covariances.
// Compared with lgssm_shared_kernel (one thread walks all T steps): no forward->backward stash or checkpoint at
// all, no dependent chain longer than 16 steps, 64 loads in flight per thread instead of 4-8, and the second read of
// y happens ~one tile lifetime after the first, from a working set of (CTAs x 32 chains x T x 4m bytes) = 76 MB at
// the headline config -- more than the H100's 50 MB L2, so the reuse is partial even when the y lines are loaded evict_last in pass A, evict_first in pass B
// and the 80 B/step of posterior stores are evict_first (createpolicy + .L2::cache_hint).  DRAM traffic per
// (chain, step) then is 4 (m + d + d^2) = the algorithmic 96 B at d = m = 4 (checkpoint kernel: ~115 B).
// STATUS: EXPERIMENTAL, not the default (RXG_OPT_SWEEP_VARIANT = 3 selects it; parity tests keep it honest).
// It measured slower than lgssm_shared_kernel at the headline config.
// Two lessons recorded in DESIGN.md: (1) these sweeps are instruction-cache sensitive -- a first version with per-store
// peer loops was 31 K instructions, this one is 5.1 K (lgssm_shared_kernel: 3.4 K; the same effect slowed that kernel by
// two thirds when peer loops grew it to 11 K); (2) with y[T][m][batch] a CTA that owns 32 chains for
// all T gathers 128-byte pieces 256 KB apart, and once the CTAs drift apart in time the DRAM pages and the output rows
// are no longer shared between neighbouring CTAs -- the lock-step walk of lgssm_shared_kernel (all CTAs at the same t)
// is what keeps its accesses row-coherent.  The L2 reuse the design aims at needs chain tiles that are wide in memory
// (>= 4 K chains) AND time-parallel work inside them, i.e. a grouped three-phase schedule; that is the follow-up.
#pragma once
#include "rxg_lgssm_common.cuh"
#include "rxg_lgssm_shared.cuh"

namespace rxg {

template <int D, int M>
struct SegTab {
    static constexpr int L = 16;                                  // steps per segment
    // per-step record of pass B
    static constexpr int F_OFF = 0;
    static constexpr int K_OFF = F_OFF + pad4(D * D);
    static constexpr int E_OFF = K_OFF + pad4(D * M);
    static constexpr int G_OFF = E_OFF + pad4(D * D);
    static constexpr int SS_OFF = G_OFF + pad4(D * D);
    static constexpr int GF_OFF = SS_OFF + pad4(D * D);
    static constexpr int GB_OFF = GF_OFF + pad4(D);
    static constexpr int REC = GB_OFF + pad4(D);
    // per-step record of pass A
    static constexpr int NF_OFF = 0;
    static constexpr int NB_OFF = NF_OFF + pad4(D * M);
    static constexpr int NREC = NB_OFF + pad4(D * M);
    // per-segment record of the scan
    static constexpr int PHI_OFF = 0;
    static constexpr int PSI_OFF = PHI_OFF + pad4(D * D);
    static constexpr int OMG_OFF = PSI_OFF + pad4(D * D);
    static constexpr int CF_OFF = OMG_OFF + pad4(D * D);
    static constexpr int CB_OFF = CF_OFF + pad4(D);
    static constexpr int SREC = CB_OFF + pad4(D);
};

struct SegWs {
    float* rec;    // [T][REC]
    float* nrec;   // [T][NREC]
    float* srec;   // [nseg][SREC]
};

// One thread per segment, fp64 from the fp32-rounded gain records (so that the summaries describe exactly the
// recursion pass B executes).  S_t = sum_{t' >= t} Gamma_t' E_t' Phi_{t' <- t+1} is the sensitivity of mu_s[a] to an
// injection into x_t; Gamma_t = G_a ... G_{t-1}.
template <int D, int M>
__global__ void seg_tables_kernel(GainWs ws, SegWs sw, int T) {
    using TB = Tab<D, M>;
    using ST = SegTab<D, M>;
    constexpr int L = ST::L;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    const int nseg = (T + L - 1) / L;
    if (s >= nseg) return;
    const int a = s * L, e = min(a + L, T) - 1;
    auto ldF = [&](int t) { return load_const<double, D, D>(ws.fwd + (size_t)t * TB::FWD_REC + TB::F_OFF); };
    auto ldK = [&](int t) { return load_const<double, D, M>(ws.fwd + (size_t)t * TB::FWD_REC + TB::K_OFF); };
    auto ldE = [&](int t) { return load_const<double, D, D>(ws.bwd + (size_t)t * TB::BWD_REC + TB::E_OFF); };
    auto ldG = [&](int t) { return load_const<double, D, D>(ws.bwd + (size_t)t * TB::BWD_REC + TB::G_OFF); };
    auto ldv = [&](const float* p) { Vec<double, D> v; for (int i = 0; i < D; ++i) v(i) = (double)p[i]; return v; };
    // repack the per-step records of pass B
    for (int t = a; t <= e; ++t) {
        const float* fr = ws.fwd + (size_t)t * TB::FWD_REC;
        const float* br = ws.bwd + (size_t)t * TB::BWD_REC;
        float* r = sw.rec + (size_t)t * ST::REC;
        for (int i = 0; i < D * D; ++i) { r[ST::F_OFF + i] = fr[TB::F_OFF + i]; r[ST::E_OFF + i] = br[TB::E_OFF + i];
                                          r[ST::G_OFF + i] = br[TB::G_OFF + i]; r[ST::SS_OFF + i] = br[TB::SS_OFF + i]; }
        for (int i = 0; i < D * M; ++i) r[ST::K_OFF + i] = fr[TB::K_OFF + i];
        for (int i = 0; i < D; ++i) { r[ST::GF_OFF + i] = fr[TB::GF_OFF + i]; r[ST::GB_OFF + i] = br[TB::GB_OFF + i]; }
    }
    // forward: P = F_e ... F_{t+1};  Nf_t = P K_t;  cf = sum P gf_t;  Phi = F_e ... F_a
    Mat<double, D, D> Pm = identity<double, D>();
    Vec<double, D> cf;
    for (int i = 0; i < D; ++i) cf(i) = 0.0;
    for (int t = e; t >= a; --t) {
        const Mat<double, D, M> Nf = mul(Pm, ldK(t));
        store_f(sw.nrec + (size_t)t * ST::NREC + ST::NF_OFF, Nf);
        const Vec<double, D> pg = mulv(Pm, ldv(ws.fwd + (size_t)t * TB::FWD_REC + TB::GF_OFF));
        for (int i = 0; i < D; ++i) cf(i) += pg(i);
        Pm = mul(Pm, ldF(t));
    }
    float* sr = sw.srec + (size_t)s * ST::SREC;
    store_f(sr + ST::PHI_OFF, Pm);
    store_fv(sr + ST::CF_OFF, cf);
    // Gamma_t, t = a..e  (Gamma_a = I), Psi = Gamma_e G_e
    Mat<double, D, D> Gam[L];
    Gam[0] = identity<double, D>();
    for (int t = a; t < e; ++t) Gam[t - a + 1] = mul(Gam[t - a], ldG(t));
    store_f(sr + ST::PSI_OFF, mul(Gam[e - a], ldG(e)));
    // backward: S_e = Gamma_e E_e;  S_t = Gamma_t E_t + S_{t+1} F_{t+1};  Nb_t = S_t K_t;  Omega = S_a F_a
    Mat<double, D, D> S;
    Vec<double, D> cb;
    for (int i = 0; i < D; ++i) cb(i) = 0.0;
    for (int t = e; t >= a; --t) {
        Mat<double, D, D> GE = mul(Gam[t - a], ldE(t));
        if (t < e) {
            const Mat<double, D, D> SF = mul(S, ldF(t + 1));
            for (int i = 0; i < D * D; ++i) GE.a[i] += SF.a[i];
        }
        S = GE;
        store_f(sw.nrec + (size_t)t * ST::NREC + ST::NB_OFF, mul(S, ldK(t)));
        const Vec<double, D> sg = mulv(S, ldv(ws.fwd + (size_t)t * TB::FWD_REC + TB::GF_OFF));
        const Vec<double, D> gg = mulv(Gam[t - a], ldv(ws.bwd + (size_t)t * TB::BWD_REC + TB::GB_OFF));
        for (int i = 0; i < D; ++i) cb(i) += sg(i) + gg(i);
    }
    store_f(sr + ST::OMG_OFF, mul(S, ldF(a)));
    store_fv(sr + ST::CB_OFF, cb);
}

__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
    unsigned long long p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ float ldg_hint(const float* p, unsigned long long pol) {
    float v;
    asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void stg_hint(float* p, float v, unsigned long long pol) {
    asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}

// stage `n16` 16-byte pieces from global to shared memory with cp.async (whole warp)
__device__ __forceinline__ void stage_pieces(float* sdst, const float* __restrict__ gsrc, int n16, int lane) {
    for (int p = lane; p < n16; p += 32) cp_async16(sdst + p * 4, gsrc + p * 4);
}

template <int D, int M, int NW, bool OFFSET, int HINTS>
__global__ void __launch_bounds__(32 * NW, 1)
lgssm_seg_kernel(const __grid_constant__ ModelF<D, M> mdl, SegWs sw, const float* __restrict__ y,
                 float* __restrict__ mean, float* __restrict__ cov, int T, int64_t batch, int write_cov,
                 const float* __restrict__ mu0c, const __grid_constant__ PeerOut po, int nseg_cap) {
    using ST = SegTab<D, M>;
    constexpr int L = ST::L;
    extern __shared__ __align__(16) float smem[];
    // layout: [nseg_cap][2 D][32] summaries | per warp: 2 x (L REC) pass-B records (pass A reuses the front: 2 x L NREC)
    float* s_sum = smem;
    float* s_tab = smem + (size_t)nseg_cap * 2 * D * 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* my_tab = s_tab + (size_t)warp * 2 * L * ST::REC;
    const int nseg = (T + L - 1) / L;
    const int64_t ntiles = (batch + 31) / 32;
    unsigned long long pol_keep = 0, pol_stream = 0;
    if (HINTS) { pol_keep = l2_policy_evict_last(); pol_stream = l2_policy_evict_first(); }

    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t b0 = tile * 32 + lane;
        const bool active = b0 < batch;
        const int64_t b = active ? b0 : (batch - 1);            // inactive lanes shadow the last chain (loads only)
        const float* yb = y + b;

        // ------------------------------------------------------------ pass A: segment summaries
        {
            int buf = 0;
            if (warp < nseg) {
                const int t0 = warp * L, n = min(L, T - t0);
                stage_pieces(my_tab, sw.nrec + (size_t)t0 * ST::NREC, n * ST::NREC / 4, lane);
            }
            cp_async_commit();
            for (int s = warp; s < nseg; s += NW) {
                const int a = s * L;
                float yv[L][M];
#pragma unroll
                for (int q = 0; q < L; ++q)
#pragma unroll
                    for (int k = 0; k < M; ++k) {
                        const int t = a + q;
                        const float* p = yb + ((int64_t)(t < T ? t : T - 1) * M + k) * batch;
                        yv[q][k] = HINTS ? ldg_hint(p, pol_keep) : __ldg(p);
                    }
                const int sn = s + NW;
                if (sn < nseg) {
                    const int t0 = sn * L, n = min(L, T - t0);
                    stage_pieces(my_tab + (buf ^ 1) * L * ST::NREC, sw.nrec + (size_t)t0 * ST::NREC, n * ST::NREC / 4, lane);
                }
                cp_async_commit();
                cp_async_wait<1>();
                __syncwarp();
                const float* nt = my_tab + buf * L * ST::NREC;
                float c[D], bt[D];
#pragma unroll
                for (int i = 0; i < D; ++i) { c[i] = 0.f; bt[i] = 0.f; }
#pragma unroll
                for (int q = 0; q < L; ++q) {
                    if (a + q < T) {
                        float Nf[pad4(D * M)], Nb[pad4(D * M)];
                        load_smem<pad4(D * M)>(nt + q * ST::NREC + ST::NF_OFF, Nf);
                        load_smem<pad4(D * M)>(nt + q * ST::NREC + ST::NB_OFF, Nb);
#pragma unroll
                        for (int i = 0; i < D; ++i)
#pragma unroll
                            for (int k = 0; k < M; ++k) {
                                c[i] = __fmaf_rn(Nf[i * M + k], yv[q][k], c[i]);
                                bt[i] = __fmaf_rn(Nb[i * M + k], yv[q][k], bt[i]);
                            }
                    }
                }
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    s_sum[((size_t)s * 2 * D + i) * 32 + lane] = c[i];
                    s_sum[((size_t)s * 2 * D + D + i) * 32 + lane] = bt[i];
                }
                __syncwarp();
                buf ^= 1;
            }
            cp_async_wait<0>();
        }
        __syncthreads();
        // ------------------------------------------------------------ scan over the segment summaries (lane = chain)
        if (warp == 0) {
            float x[D];
#pragma unroll
            for (int i = 0; i < D; ++i) x[i] = mu0c ? __ldg(mu0c + (int64_t)i * batch + b) : mdl.m0[i];
            for (int s = 0; s < nseg; ++s) {
                const float* sr = sw.srec + (size_t)s * ST::SREC;
                float Phi[pad4(D * D)], cfv[pad4(D)];
                load_uniform<pad4(D * D)>(sr + ST::PHI_OFF, Phi);
                if (OFFSET) load_uniform<pad4(D)>(sr + ST::CF_OFF, cfv);
                float nx[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    float acc = s_sum[((size_t)s * 2 * D + i) * 32 + lane];
                    if (OFFSET) acc += cfv[i];
#pragma unroll
                    for (int j = 0; j < D; ++j) acc = __fmaf_rn(Phi[i * D + j], x[j], acc);
                    nx[i] = acc;
                }
#pragma unroll
                for (int i = 0; i < D; ++i) { s_sum[((size_t)s * 2 * D + i) * 32 + lane] = x[i]; x[i] = nx[i]; }
            }
            float sv[D];
#pragma unroll
            for (int i = 0; i < D; ++i) sv[i] = 0.f;
            for (int s = nseg - 1; s >= 0; --s) {
                const float* sr = sw.srec + (size_t)s * ST::SREC;
                float Psi[pad4(D * D)], Omg[pad4(D * D)], cbv[pad4(D)];
                load_uniform<pad4(D * D)>(sr + ST::PSI_OFF, Psi);
                load_uniform<pad4(D * D)>(sr + ST::OMG_OFF, Omg);
                if (OFFSET) load_uniform<pad4(D)>(sr + ST::CB_OFF, cbv);
                float xin[D], nv[D];
#pragma unroll
                for (int i = 0; i < D; ++i) xin[i] = s_sum[((size_t)s * 2 * D + i) * 32 + lane];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    float acc = s_sum[((size_t)s * 2 * D + D + i) * 32 + lane];
                    if (OFFSET) acc += cbv[i];
#pragma unroll
                    for (int j = 0; j < D; ++j) acc = __fmaf_rn(Psi[i * D + j], sv[j], acc);
#pragma unroll
                    for (int j = 0; j < D; ++j) acc = __fmaf_rn(Omg[i * D + j], xin[j], acc);
                    nv[i] = acc;
                }
#pragma unroll
                for (int i = 0; i < D; ++i) { s_sum[((size_t)s * 2 * D + D + i) * 32 + lane] = sv[i]; sv[i] = nv[i]; }
            }
        }
        __syncthreads();
        // ------------------------------------------------------------ pass B: the segment's recursions from the true carries
        {
            int buf = 0;
            if (warp < nseg) {
                const int t0 = warp * L, n = min(L, T - t0);
                stage_pieces(my_tab, sw.rec + (size_t)t0 * ST::REC, n * ST::REC / 4, lane);
            }
            cp_async_commit();
            for (int s = warp; s < nseg; s += NW) {
                const int a = s * L;
                float yv[L][M];
#pragma unroll
                for (int q = 0; q < L; ++q)
#pragma unroll
                    for (int k = 0; k < M; ++k) {
                        const int t = a + q;
                        const float* p = yb + ((int64_t)(t < T ? t : T - 1) * M + k) * batch;
                        yv[q][k] = HINTS ? ldg_hint(p, pol_stream) : __ldg(p);
                    }
                const int sn = s + NW;
                if (sn < nseg) {
                    const int t0 = sn * L, n = min(L, T - t0);
                    stage_pieces(my_tab + (buf ^ 1) * L * ST::REC, sw.rec + (size_t)t0 * ST::REC, n * ST::REC / 4, lane);
                }
                cp_async_commit();
                cp_async_wait<1>();
                __syncwarp();
                const float* rt = my_tab + buf * L * ST::REC;
                float x[D], sv[D];
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    x[i] = s_sum[((size_t)s * 2 * D + i) * 32 + lane];
                    sv[i] = s_sum[((size_t)s * 2 * D + D + i) * 32 + lane];
                }
                float xs[L][D];
#pragma unroll
                for (int q = 0; q < L; ++q) {
                    if (a + q < T) {
                        const float* rec = rt + q * ST::REC;
                        float Ft[pad4(D * D)], Kt[pad4(D * M)], gf[pad4(D)];
                        load_smem<pad4(D * D)>(rec + ST::F_OFF, Ft);
                        load_smem<pad4(D * M)>(rec + ST::K_OFF, Kt);
                        if (OFFSET) load_smem<pad4(D)>(rec + ST::GF_OFF, gf);
                        float nx[D];
#pragma unroll
                        for (int i = 0; i < D; ++i) {
                            float acc = OFFSET ? __fmaf_rn(Ft[i * D], x[0], gf[i]) : Ft[i * D] * x[0];
#pragma unroll
                            for (int j = 1; j < D; ++j) acc = __fmaf_rn(Ft[i * D + j], x[j], acc);
#pragma unroll
                            for (int k = 0; k < M; ++k) acc = __fmaf_rn(Kt[i * M + k], yv[q][k], acc);
                            nx[i] = acc;
                        }
#pragma unroll
                        for (int i = 0; i < D; ++i) { x[i] = nx[i]; xs[q][i] = nx[i]; }
                    }
                }
#pragma unroll
                for (int q = L - 1; q >= 0; --q) {
                    const int t = a + q;
                    if (t < T) {
                        const float* rec = rt + q * ST::REC;
                        float Et[pad4(D * D)], Gt[pad4(D * D)], gb[pad4(D)];
                        load_smem<pad4(D * D)>(rec + ST::E_OFF, Et);
                        load_smem<pad4(D * D)>(rec + ST::G_OFF, Gt);
                        if (OFFSET) load_smem<pad4(D)>(rec + ST::GB_OFF, gb);
                        float nv[D];
#pragma unroll
                        for (int i = 0; i < D; ++i) {
                            float acc = OFFSET ? __fmaf_rn(Et[i * D], xs[q][0], gb[i]) : Et[i * D] * xs[q][0];
#pragma unroll
                            for (int j = 1; j < D; ++j) acc = __fmaf_rn(Et[i * D + j], xs[q][j], acc);
#pragma unroll
                            for (int j = 0; j < D; ++j) acc = __fmaf_rn(Gt[i * D + j], sv[j], acc);
                            nv[i] = acc;
                        }
#pragma unroll
                        for (int i = 0; i < D; ++i) sv[i] = nv[i];
                        if (active) {
#pragma unroll
                            for (int i = 0; i < D; ++i) {
                                const int64_t off = ((int64_t)t * D + i) * batch + b;
                                if (HINTS) stg_hint(mean + off, sv[i], pol_stream); else mean[off] = sv[i];
                            }
                            if (write_cov) {
                                float Ss[pad4(D * D)];
                                load_smem<pad4(D * D)>(rec + ST::SS_OFF, Ss);
#pragma unroll
                                for (int i = 0; i < D * D; ++i) {
                                    const int64_t off = ((int64_t)t * D * D + i) * batch + b;
                                    if (HINTS) stg_hint(cov + off, Ss[i], pol_stream); else cov[off] = Ss[i];
                                }
                            }
                        }
                    }
                }
                __syncwarp();
                buf ^= 1;
            }
            cp_async_wait<0>();
        }
        // the next tile's pass A overwrites only summary slots this warp has already consumed; the scan of the next
        // tile is separated from this pass B by the __syncthreads after pass A
    }
}

}  // namespace rxg
