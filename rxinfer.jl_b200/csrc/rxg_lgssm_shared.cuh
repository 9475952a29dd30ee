// lgssm_shared_kernel: the mean-only forward/backward sweep of the shared-model path.
//
// One warp = one CTA = 32 x CPT chains, so CTAs spread over the 132 SMs to within one warp and no
// block-wide barrier is ever needed.  Per (chain, step) the sweep moves
//     forward : read y_t (m)            write filtered mean (d)      [stash, in post_mean]
//     backward: read filtered mean (d)  write smoothed mean (d) + smoothed covariance (d*d)
// = 4 (m + 3 d + d^2) bytes (128 B at d = m = 4; 96 B of it is the contract's algorithmic I/O).
//
// Latency hiding (the kernel is HBM-latency bound, ~3.5 warps per SM sub-partition):
//   * the data-independent gain tables (F_t, K_t / E_t, G_t, Sigma_s,t) are staged through shared
//     memory TC steps at a time with cp.async (double buffered), so the per-step table reads are
//     29-cycle broadcast LDS instead of ~300-cycle L2 hits on the dependent chain;
//   * the per-chain streams (y forward, stashed means backward) are prefetched PF steps ahead
//     into registers.
#pragma once
#include "rxg_lgssm_common.cuh"

namespace rxg {

// uniform (same address for every lane) loads of a table segment from global memory
template <int N>
__device__ __forceinline__ void load_uniform(const float* __restrict__ p, float* dst) {
    if (N % 4 == 0) {
        const float4* p4 = reinterpret_cast<const float4*>(p);
#pragma unroll
        for (int i = 0; i < N / 4; ++i) {
            float4 v = __ldg(p4 + i);
            dst[4 * i] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; ++i) dst[i] = __ldg(p + i);
    }
}
// broadcast reads of a table segment staged in shared memory (N is a multiple of 4)
template <int N>
__device__ __forceinline__ void load_smem(const float* p, float* dst) {
    const float4* p4 = reinterpret_cast<const float4*>(p);
#pragma unroll
    for (int i = 0; i < N / 4; ++i) {
        float4 v = p4[i];
        dst[4 * i] = v.x; dst[4 * i + 1] = v.y; dst[4 * i + 2] = v.z; dst[4 * i + 3] = v.w;
    }
}

template <int CPT> struct Pack;
template <> struct Pack<1> {
    static __device__ __forceinline__ void ld(const float* p, float* v) { v[0] = __ldg(p); }
    static __device__ __forceinline__ void ld_rw(const float* p, float* v) { v[0] = *p; }
    static __device__ __forceinline__ void st(float* p, const float* v) { *p = v[0]; }
};
template <> struct Pack<2> {
    static __device__ __forceinline__ void ld(const float* p, float* v) {
        float2 t = __ldg(reinterpret_cast<const float2*>(p)); v[0] = t.x; v[1] = t.y;
    }
    static __device__ __forceinline__ void ld_rw(const float* p, float* v) {
        float2 t = *reinterpret_cast<const float2*>(p); v[0] = t.x; v[1] = t.y;
    }
    static __device__ __forceinline__ void st(float* p, const float* v) {
        *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
    }
};
template <> struct Pack<4> {
    static __device__ __forceinline__ void ld(const float* p, float* v) {
        float4 t = __ldg(reinterpret_cast<const float4*>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void ld_rw(const float* p, float* v) {
        float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void st(float* p, const float* v) {
        *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    }
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// Stage TC consecutive table records (REC floats each, REC % 4 == 0) into shared memory.
// `first` is the record index of slot 0, `dir` = +1 (forward in t) or -1 (backward in t).
template <int REC, int TC>
__device__ __forceinline__ void stage_tables(float* sdst, const float* __restrict__ tab, int first, int dir,
                                             int T, int lane) {
    constexpr int PIECES = REC / 4;   // 16-byte pieces per record
#pragma unroll
    for (int p = lane; p < TC * PIECES; p += 32) {
        const int slot = p / PIECES, part = p % PIECES;
        const int t = first + dir * slot;
        if (t >= 0 && t < T) cp_async16(sdst + slot * REC + part * 4, tab + (size_t)t * REC + part * 4);
    }
    cp_async_commit();
}

// One step's posteriors to every peer: ONE rolled loop over the peers per step (not one per store site).
template <int D, int CPT>
__device__ __forceinline__ void peer_store(const PeerOut& po, int write_cov, int t, int64_t batch, int64_t b,
                                           const float (&ms)[D][CPT], const float* Sst) {
#pragma unroll 1
    for (int g = 0; g < po.n_mean; ++g) {
        float* pm = po.mean[g] + (int64_t)t * D * batch + b;
#pragma unroll
        for (int i = 0; i < D; ++i) Pack<CPT>::st(pm + (int64_t)i * batch, ms[i]);      // NVLink P2P stores
    }
    if (write_cov) {
#pragma unroll 1
        for (int g = 0; g < po.n_cov; ++g) {
            float* pc = po.cov[g] + (int64_t)t * D * D * batch + b;
#pragma unroll
            for (int i = 0; i < D * D; ++i) {
                float v[CPT];
#pragma unroll
                for (int c = 0; c < CPT; ++c) v[c] = Sst[i];
                Pack<CPT>::st(pc + (int64_t)i * batch, v);
            }
        }
    }
}

// u[t] of one step for this thread's CPT chains: per-chain input sequence useq[rows][D][batch]
template <int D, int CPT>
__device__ __forceinline__ void load_input(const float* __restrict__ useq, int t, int64_t batch, int64_t b, float (&u)[D][CPT]) {
#pragma unroll
    for (int i = 0; i < D; ++i) Pack<CPT>::ld(useq + ((int64_t)t * D + i) * batch + b, u[i]);
}

// USEQ forward step: nm = F mu + K (y_t - B u_t) + u_t
template <int D, int M, int CPT>
__device__ __forceinline__ void input_step(const float* Ft, const float* Kt, const float* Bm, const float (&mu)[D][CPT],
                                           const float (&yt)[M][CPT], const float (&ut)[D][CPT], float (&nm)[D][CPT]) {
    float ye[M][CPT];
#pragma unroll
    for (int k = 0; k < M; ++k)
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
            float a = yt[k][c];
#pragma unroll
            for (int j = 0; j < D; ++j) a = __fmaf_rn(-Bm[k * D + j], ut[j][c], a);
            ye[k][c] = a;
        }
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
            float a = __fmaf_rn(Ft[i * D], mu[0][c], ut[i][c]);
#pragma unroll
            for (int j = 1; j < D; ++j) a = __fmaf_rn(Ft[i * D + j], mu[j][c], a);
#pragma unroll
            for (int k = 0; k < M; ++k) a = __fmaf_rn(Kt[i * M + k], ye[k][c], a);
            nm[i][c] = a;
        }
}
// USEQ backward step: nm = E mu_f[t] + G (mu_s[t+1] - u_{t+1})   (record T-1 has G = 0: no row T is read)
template <int D, int CPT>
__device__ __forceinline__ void input_back(const float* Et, const float* Gt, const float (&fm)[D][CPT], const float (&ms)[D][CPT],
                                           const float* __restrict__ useq, int t, int T, int64_t batch, int64_t b,
                                           float (&nm)[D][CPT]) {
    float gv[D][CPT];
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int c = 0; c < CPT; ++c) gv[i][c] = ms[i][c];
    if (t + 1 < T) {
        float un[D][CPT];
        load_input<D, CPT>(useq, t + 1, batch, b, un);
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int c = 0; c < CPT; ++c) gv[i][c] -= un[i][c];
    }
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
            float a = Et[i * D] * fm[0][c];
#pragma unroll
            for (int j = 1; j < D; ++j) a = __fmaf_rn(Et[i * D + j], fm[j][c], a);
#pragma unroll
            for (int j = 0; j < D; ++j) a = __fmaf_rn(Gt[i * D + j], gv[j][c], a);
            nm[i][c] = a;
        }
}

// PEER: the final posteriors are also stored to the peer ranks' gathered buffers (fused all-gather, rxg_peer.cu).
// A separate instantiation, because the kernel is instruction-cache sensitive: the loops over peers inside the
// unrolled step bodies took the single-GPU kernel from 3.4 K to 11 K instructions.
// USEQ = 1: per-chain input sequence (RXG_U_SEQ_CHAIN, useq[rows][D][batch]), streamed beside y; the gain tables are
// those without inputs (OFFSET = false) and the inputs enter the mean recursions directly:
//     forward   mu_f[t] = F_t mu_f[t-1] + K_t (y_t - B u_t) + u_t     (EVID: innovation y_t - B (A mu_f[t-1] + u_t))
//     backward  mu_s[t] = E_t mu_f[t] + G_t (mu_s[t+1] - u_{t+1})
// USEQ = 2: shared input sequence (RXG_U_SEQ_SHARED, useq[rows][D]) with evidence: the tables carry the offsets
// gf_t, gb_t (OFFSET = true) and only the explicit evidence form reads u_t (uniform over the warp) where the constant
// offset reads mdl.u.
// Separate instantiations: every other one compiles to the code it had without them.
// (USEQ at d * m > 16 with one chain per thread: <= 168 registers, 128 would spill)
template <int D, int M, int CPT, int PF, bool SMOOTH, bool EVID, bool OFFSET, bool CKPT, bool PEER = false, int USEQ = 0>
__global__ void __launch_bounds__(32, (USEQ != 0 && D * M > 16 && CPT == 1) ? 12 : 16 / CPT)   // CPT=1: <= 128 regs so ~14 warps/SM stay resident; wider CPT trades warps for ILP
lgssm_shared_kernel(const __grid_constant__ ModelF<D, M> mdl, const float* __restrict__ fwd_tab,
                    const float* __restrict__ bwd_tab, const float* __restrict__ sf_tab,
                    const float* __restrict__ y, float* __restrict__ mean, float* __restrict__ cov,
                    float* __restrict__ nle, int T, int64_t batch, int transition_first,
                    int write_cov, const float* __restrict__ mu0c, const __grid_constant__ PeerOut po,
                    const float* __restrict__ useq = nullptr) {
    static_assert(USEQ == 0 || (!PEER && OFFSET == (USEQ == 2) && (USEQ == 1 || EVID)),
                  "input sequences: per chain without table offsets, shared with them (evidence form only); no peer stores");
    using TB = Tab<D, M>;
    // CKPT (smoothing only): the forward pass keeps one filtered mean per TC-step chunk; the backward
    // pass re-reads y and recomputes the chunk's filtered means into s_f (lane-contiguous, private
    // to each thread), which replaces the 2 x 4d bytes/step stash by 4m bytes/step of y re-read.
    constexpr bool CK = SMOOTH && CKPT && (D * D <= 16);   // larger states exceed the static smem budget: stash path
    // table chunk, in time steps.  With CK, 12-step chunks keep the static shared memory at 22.6 KB (d = m = 4, CPT = 2),
    // so 9 CTAs fit in an SM and a 65 536-chain grid (1024 one-warp CTAs) is resident in one wave on 132 SMs; 16-step
    // chunks (30.2 KB, 7 CTAs per SM) leave a second wave of 100 CTAs.
    constexpr int TC = CK ? 3 * PF : 4 * PF;
    constexpr int REC_MAX = TB::FWD_REC > TB::BWD_REC ? TB::FWD_REC : TB::BWD_REC;
    __shared__ __align__(16) float s_tab[2][TC * (CK ? (TB::FWD_REC + TB::BWD_REC) : REC_MAX)];
    __shared__ float s_f[CK ? TC * D * CPT * 32 : 1];

    const int lane = threadIdx.x;
    const int64_t b0 = ((int64_t)blockIdx.x * 32 + lane) * CPT;
    const bool active = b0 < batch;
    const int64_t b = active ? b0 : 0;      // inactive lanes shadow chain 0 (loads only, no stores)

    // prior mean: shared (parameter block) or per chain (mu0c[d][batch]: the streaming engine's carry,
    // @autoupdates x_min_t_mean = mean(q(x_t)), /root/reference/src/inference/autoupdates.jl:614-659)
    float mu[D][CPT];
#pragma unroll
    for (int i = 0; i < D; ++i) {
        if (mu0c) Pack<CPT>::ld(mu0c + (int64_t)i * batch + b, mu[i]);
        else
#pragma unroll
            for (int c = 0; c < CPT; ++c) mu[i][c] = mdl.m0[i];
    }
    float ev[CPT];
    double ev_hi[CPT];
#pragma unroll
    for (int c = 0; c < CPT; ++c) { ev[c] = 0.f; ev_hi[c] = 0.0; }

    // ---------------------------------------------------------------- forward
    float ycur[PF][M][CPT], ynxt[PF][M][CPT];
#pragma unroll
    for (int s = 0; s < PF; ++s)
        if (s < T)
#pragma unroll
            for (int k = 0; k < M; ++k) Pack<CPT>::ld(y + ((int64_t)s * M + k) * batch + b, ycur[s][k]);

    stage_tables<TB::FWD_REC, TC>(s_tab[0], fwd_tab, 0, +1, T, lane);
    for (int t0 = 0; t0 < T; t0 += PF) {
        if ((t0 % TC) == 0) {
            const int c = t0 / TC;
            __syncwarp();                       // all lanes are done with the buffer about to be refilled
            stage_tables<TB::FWD_REC, TC>(s_tab[(c + 1) & 1], fwd_tab, (c + 1) * TC, +1, T, lane);
            cp_async_wait<1>();                 // chunk c has landed (this lane's pieces)
            __syncwarp();                       // ... and every other lane's
        }
#pragma unroll
        for (int s = 0; s < PF; ++s)
            if (t0 + PF + s < T)
#pragma unroll
                for (int k = 0; k < M; ++k)
                    Pack<CPT>::ld(y + ((int64_t)(t0 + PF + s) * M + k) * batch + b, ynxt[s][k]);
#pragma unroll
        for (int s = 0; s < PF; ++s) {
            const int t = t0 + s;
            if (t < T) {
                const float* rec = s_tab[(t / TC) & 1] + (t % TC) * TB::FWD_REC;
                float Kt[pad4(D * M)];
                load_smem<pad4(D * M)>(rec + TB::K_OFF, Kt);
                float nm[D][CPT];
                float ut[D][CPT];                   // u_t (USEQ; zero at a step without a transition)
                if constexpr (USEQ == 2) {
#pragma unroll
                    for (int i = 0; i < D; ++i) {
                        const float v = (t > 0 || transition_first) ? __ldg(useq + (size_t)t * D + i) : 0.f;
#pragma unroll
                        for (int c = 0; c < CPT; ++c) ut[i][c] = v;
                    }
                }
                if constexpr (USEQ == 1) {
                    if (t > 0 || transition_first) load_input<D, CPT>(useq, t, batch, b, ut);
                    else
#pragma unroll
                        for (int i = 0; i < D; ++i)
#pragma unroll
                            for (int c = 0; c < CPT; ++c) ut[i][c] = 0.f;
                }
                if (!EVID) {
                    // mu_f[t] = F_t mu_f[t-1] + K_t y_t,  F_t = (I - K_t B) A   (rules #1-#4 + product)
                    float Ft[pad4(D * D)], gf[pad4(D)];
                    load_smem<pad4(D * D)>(rec + TB::F_OFF, Ft);
                    if (OFFSET) load_smem<pad4(D)>(rec + TB::GF_OFF, gf);        // (I - K B) u: the fused `+` rule
                    if constexpr (USEQ == 1) {
                        // mu_f[t] = F_t mu_f[t-1] + K_t (y_t - B u_t) + u_t
                        input_step<D, M, CPT>(Ft, Kt, mdl.B, mu, ycur[s], ut, nm);
                    } else {
#pragma unroll
                    for (int i = 0; i < D; ++i)
#pragma unroll
                        for (int c = 0; c < CPT; ++c) {
                            float a = OFFSET ? __fmaf_rn(Ft[i * D], mu[0][c], gf[i]) : Ft[i * D] * mu[0][c];
#pragma unroll
                            for (int j = 1; j < D; ++j) a = __fmaf_rn(Ft[i * D + j], mu[j][c], a);
#pragma unroll
                            for (int k = 0; k < M; ++k) a = __fmaf_rn(Kt[i * M + k], ycur[s][k][c], a);
                            nm[i][c] = a;
                        }
                    }
                } else {
                    // explicit form so that the innovation is available for the evidence
                    float Li[pad4(M * M)], cc[4];
                    load_smem<pad4(M * M)>(rec + TB::LI_OFF, Li);
                    load_smem<4>(rec + TB::C_OFF, cc);
                    const bool pred = (t > 0) || transition_first;
#pragma unroll
                    for (int c = 0; c < CPT; ++c) {
                        float mp[D], e[M];
#pragma unroll
                        for (int i = 0; i < D; ++i) {
                            if (pred) {
                                float a;
                                if constexpr (USEQ != 0) a = __fmaf_rn(mdl.A[i * D], mu[0][c], ut[i][c]);
                                else a = OFFSET ? __fmaf_rn(mdl.A[i * D], mu[0][c], mdl.u[i]) : mdl.A[i * D] * mu[0][c];
#pragma unroll
                                for (int j = 1; j < D; ++j) a = __fmaf_rn(mdl.A[i * D + j], mu[j][c], a);
                                mp[i] = a;
                            } else {
                                mp[i] = mu[i][c];
                            }
                        }
#pragma unroll
                        for (int k = 0; k < M; ++k) {
                            float a = ycur[s][k][c];
#pragma unroll
                            for (int j = 0; j < D; ++j) a = __fmaf_rn(-mdl.B[k * D + j], mp[j], a);
                            e[k] = a;
                        }
                        float q = 0.f;
#pragma unroll
                        for (int k = 0; k < M; ++k) {
                            float a = 0.f;
#pragma unroll
                            for (int j = 0; j <= k; ++j) a = __fmaf_rn(Li[k * M + j], e[j], a);
                            q = __fmaf_rn(a, a, q);
                        }
                        ev[c] += __fmaf_rn(0.5f, q, cc[0]);
#pragma unroll
                        for (int i = 0; i < D; ++i) {
                            float a = mp[i];
#pragma unroll
                            for (int k = 0; k < M; ++k) a = __fmaf_rn(Kt[i * M + k], e[k], a);
                            nm[i][c] = a;
                        }
                    }
                    if ((t & 63) == 63) {   // flush the fp32 partial sum into fp64 every 64 steps
#pragma unroll
                        for (int c = 0; c < CPT; ++c) { ev_hi[c] += (double)ev[c]; ev[c] = 0.f; }
                    }
                }
#pragma unroll
                for (int i = 0; i < D; ++i) {
#pragma unroll
                    for (int c = 0; c < CPT; ++c) mu[i][c] = nm[i][c];
                    if (active && (!CK || (t % TC) == TC - 1)) Pack<CPT>::st(mean + ((int64_t)t * D + i) * batch + b, mu[i]);
                }
                if (!SMOOTH && write_cov && active) {
                    float Sf[pad4(D * D)];
                    load_uniform<pad4(D * D)>(sf_tab + (size_t)t * TB::SF_REC, Sf);
#pragma unroll
                    for (int i = 0; i < D * D; ++i) {
                        float v[CPT];
#pragma unroll
                        for (int c = 0; c < CPT; ++c) v[c] = Sf[i];
                        Pack<CPT>::st(cov + ((int64_t)t * D * D + i) * batch + b, v);
                    }
                }
            }
        }
#pragma unroll
        for (int s = 0; s < PF; ++s)
#pragma unroll
            for (int k = 0; k < M; ++k)
#pragma unroll
                for (int c = 0; c < CPT; ++c) ycur[s][k][c] = ynxt[s][k][c];
    }
    if (EVID && nle && active) {
#pragma unroll
        for (int c = 0; c < CPT; ++c) nle[b + c] = (float)(ev_hi[c] + (double)ev[c]);
    }
    cp_async_wait<0>();
    if (!SMOOTH) return;

    if (CK) {
        // ------------------------------------------------------------ backward, chunk by chunk (descending)
        const int nch = (T + TC - 1) / TC;
        float ms[D][CPT];
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int c = 0; c < CPT; ++c) ms[i][c] = 0.f;
        auto stage_chunk = [&](int k, int buf) {       // forward + backward records of steps [k TC, k TC + TC)
            float* dst = s_tab[buf];
            constexpr int PF_ = TB::FWD_REC / 4, PB_ = TB::BWD_REC / 4;
            if (k >= 0) {
#pragma unroll
                for (int p = lane; p < TC * PF_; p += 32) {
                    const int slot = p / PF_, part = p % PF_, t = k * TC + slot;
                    if (t < T) cp_async16(dst + slot * TB::FWD_REC + part * 4, fwd_tab + (size_t)t * TB::FWD_REC + part * 4);
                }
#pragma unroll
                for (int p = lane; p < TC * PB_; p += 32) {
                    const int slot = p / PB_, part = p % PB_, t = k * TC + slot;
                    if (t < T) cp_async16(dst + TC * TB::FWD_REC + slot * TB::BWD_REC + part * 4,
                                          bwd_tab + (size_t)t * TB::BWD_REC + part * 4);
                }
            }
            cp_async_commit();
        };
        // y prefetch runs over the recompute order: chunk nch-1, nch-2, ..., each ascending in t
        auto blk_t0 = [&](int j) { return (nch - 1 - j / (TC / PF)) * TC + (j % (TC / PF)) * PF; };
        const int nblk = nch * (TC / PF);
        {
            const int t0 = blk_t0(0);
#pragma unroll
            for (int s = 0; s < PF; ++s)
                if (t0 + s < T)
#pragma unroll
                    for (int k = 0; k < M; ++k) Pack<CPT>::ld(y + ((int64_t)(t0 + s) * M + k) * batch + b, ycur[s][k]);
        }
        float ck[D][CPT];                      // checkpoint (filtered mean at the step before the chunk)
        {
            const int k = nch - 1;
#pragma unroll
            for (int i = 0; i < D; ++i) {
                if (k == 0) {
                    if (mu0c) Pack<CPT>::ld(mu0c + (int64_t)i * batch + b, ck[i]);
                    else
#pragma unroll
                        for (int c = 0; c < CPT; ++c) ck[i][c] = mdl.m0[i];
                } else {
                    Pack<CPT>::ld_rw(mean + ((int64_t)(k * TC - 1) * D + i) * batch + b, ck[i]);
                }
            }
        }
        __syncwarp();
        stage_chunk(nch - 1, 0);
        int j = 0;
        for (int k = nch - 1; k >= 0; --k) {
            const int buf = (nch - 1 - k) & 1;
            __syncwarp();
            stage_chunk(k - 1, buf ^ 1);
            cp_async_wait<1>();
            __syncwarp();
            const float* sF = s_tab[buf];
            const float* sB = s_tab[buf] + TC * TB::FWD_REC;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int c = 0; c < CPT; ++c) mu[i][c] = ck[i][c];
            // prefetch the checkpoint of the next (earlier) chunk
            if (k >= 1) {
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    if (k == 1) {
                        if (mu0c) Pack<CPT>::ld(mu0c + (int64_t)i * batch + b, ck[i]);
                        else
#pragma unroll
                            for (int c = 0; c < CPT; ++c) ck[i][c] = mdl.m0[i];
                    } else {
                        Pack<CPT>::ld_rw(mean + ((int64_t)((k - 1) * TC - 1) * D + i) * batch + b, ck[i]);
                    }
                }
            }
            // ---- recompute the filtered means of the chunk
            for (int blk = 0; blk < TC / PF; ++blk, ++j) {
                const int t0 = k * TC + blk * PF;
                if (j + 1 < nblk) {
                    const int tn = blk_t0(j + 1);
#pragma unroll
                    for (int s = 0; s < PF; ++s)
                        if (tn + s < T)
#pragma unroll
                            for (int kk = 0; kk < M; ++kk)
                                Pack<CPT>::ld(y + ((int64_t)(tn + s) * M + kk) * batch + b, ynxt[s][kk]);
                }
#pragma unroll
                for (int s = 0; s < PF; ++s) {
                    const int t = t0 + s;
                    if (t < T) {
                        const float* rec = sF + (blk * PF + s) * TB::FWD_REC;
                        float Kt[pad4(D * M)], Ft[pad4(D * D)], gf[pad4(D)];
                        load_smem<pad4(D * M)>(rec + TB::K_OFF, Kt);
                        load_smem<pad4(D * D)>(rec + TB::F_OFF, Ft);
                        if (OFFSET) load_smem<pad4(D)>(rec + TB::GF_OFF, gf);
                        float nm[D][CPT];
                        const bool first_no_pred = (t == 0) && !transition_first && EVID;
                        if constexpr (USEQ == 1) {
                            // the recompute re-reads u_t beside y_t
                            float ut[D][CPT];
                            if (t > 0 || transition_first) load_input<D, CPT>(useq, t, batch, b, ut);
                            else
#pragma unroll
                                for (int i = 0; i < D; ++i)
#pragma unroll
                                    for (int c = 0; c < CPT; ++c) ut[i][c] = 0.f;
                            input_step<D, M, CPT>(Ft, Kt, mdl.B, mu, ycur[s], ut, nm);
                        } else {
#pragma unroll
                        for (int i = 0; i < D; ++i)
#pragma unroll
                            for (int c = 0; c < CPT; ++c) {
                                float a = OFFSET ? __fmaf_rn(Ft[i * D], mu[0][c], gf[i]) : Ft[i * D] * mu[0][c];
#pragma unroll
                                for (int jj = 1; jj < D; ++jj) a = __fmaf_rn(Ft[i * D + jj], mu[jj][c], a);
#pragma unroll
                                for (int kk = 0; kk < M; ++kk) a = __fmaf_rn(Kt[i * M + kk], ycur[s][kk][c], a);
                                nm[i][c] = a;
                            }
                        }
                        (void)first_no_pred;
#pragma unroll
                        for (int i = 0; i < D; ++i)
#pragma unroll
                            for (int c = 0; c < CPT; ++c) {
                                mu[i][c] = nm[i][c];
                                s_f[(((blk * PF + s) * D + i) * CPT + c) * 32 + lane] = nm[i][c];
                            }
                    }
                }
#pragma unroll
                for (int s = 0; s < PF; ++s)
#pragma unroll
                    for (int kk = 0; kk < M; ++kk)
#pragma unroll
                        for (int c = 0; c < CPT; ++c) ycur[s][kk][c] = ynxt[s][kk][c];
            }
            // ---- backward over the chunk
#pragma unroll 4
            for (int slot = TC - 1; slot >= 0; --slot) {
                const int t = k * TC + slot;
                if (t < T) {
                    const float* rec = sB + slot * TB::BWD_REC;
                    float Et[pad4(D * D)], Gt[pad4(D * D)], gb[pad4(D)];
                    load_smem<pad4(D * D)>(rec + TB::E_OFF, Et);
                    load_smem<pad4(D * D)>(rec + TB::G_OFF, Gt);
                    if (OFFSET) load_smem<pad4(D)>(rec + TB::GB_OFF, gb);
                    float fm[D][CPT], nm[D][CPT];
#pragma unroll
                    for (int i = 0; i < D; ++i)
#pragma unroll
                        for (int c = 0; c < CPT; ++c) fm[i][c] = s_f[((slot * D + i) * CPT + c) * 32 + lane];
                    if constexpr (USEQ == 1) {
                        input_back<D, CPT>(Et, Gt, fm, ms, useq, t, T, batch, b, nm);
                    } else {
#pragma unroll
                    for (int i = 0; i < D; ++i)
#pragma unroll
                        for (int c = 0; c < CPT; ++c) {
                            float a = OFFSET ? __fmaf_rn(Et[i * D], fm[0][c], gb[i]) : Et[i * D] * fm[0][c];
#pragma unroll
                            for (int jj = 1; jj < D; ++jj) a = __fmaf_rn(Et[i * D + jj], fm[jj][c], a);
#pragma unroll
                            for (int jj = 0; jj < D; ++jj) a = __fmaf_rn(Gt[i * D + jj], ms[jj][c], a);
                            nm[i][c] = a;
                        }
                    }
#pragma unroll
                    for (int i = 0; i < D; ++i) {
#pragma unroll
                        for (int c = 0; c < CPT; ++c) ms[i][c] = nm[i][c];
                        if (active) Pack<CPT>::st(mean + ((int64_t)t * D + i) * batch + b, ms[i]);
                    }
                    float Sst[pad4(D * D)];
                    if (write_cov && active) {
                        load_smem<pad4(D * D)>(rec + TB::SS_OFF, Sst);
#pragma unroll
                        for (int i = 0; i < D * D; ++i) {
                            float v[CPT];
#pragma unroll
                            for (int c = 0; c < CPT; ++c) v[c] = Sst[i];
                            Pack<CPT>::st(cov + ((int64_t)t * D * D + i) * batch + b, v);
                        }
                    }
                    if (PEER && active) peer_store<D, CPT>(po, write_cov, t, batch, b, ms, Sst);
                }
            }
        }
        cp_async_wait<0>();
        return;
    }

    // ---------------------------------------------------------------- backward (r = T-1-t ascending)
    // mu_s[t] = E_t mu_f[t] + G_t mu_s[t+1]  (rules #3', #4 backward + 3-way marginal);
    // record T-1 holds E = I, G = 0.  Sigma_s[t] is chain-independent: broadcast store.
    float ms[D][CPT];
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int c = 0; c < CPT; ++c) ms[i][c] = 0.f;
    float fcur[PF][D][CPT], fnxt[PF][D][CPT];
#pragma unroll
    for (int s = 0; s < PF; ++s)
        if (T - 1 - s >= 0)
#pragma unroll
            for (int i = 0; i < D; ++i)
                Pack<CPT>::ld_rw(mean + ((int64_t)(T - 1 - s) * D + i) * batch + b, fcur[s][i]);

    __syncwarp();
    stage_tables<TB::BWD_REC, TC>(s_tab[0], bwd_tab, T - 1, -1, T, lane);
    for (int r0 = 0; r0 < T; r0 += PF) {
        if ((r0 % TC) == 0) {
            const int c = r0 / TC;
            __syncwarp();
            stage_tables<TB::BWD_REC, TC>(s_tab[(c + 1) & 1], bwd_tab, T - 1 - (c + 1) * TC, -1, T, lane);
            cp_async_wait<1>();
            __syncwarp();
        }
#pragma unroll
        for (int s = 0; s < PF; ++s)
            if (T - 1 - (r0 + PF + s) >= 0)
#pragma unroll
                for (int i = 0; i < D; ++i)
                    Pack<CPT>::ld_rw(mean + ((int64_t)(T - 1 - (r0 + PF + s)) * D + i) * batch + b, fnxt[s][i]);
#pragma unroll
        for (int s = 0; s < PF; ++s) {
            const int r = r0 + s;
            const int t = T - 1 - r;
            if (t >= 0) {
                const float* rec = s_tab[(r / TC) & 1] + (r % TC) * TB::BWD_REC;
                float Et[pad4(D * D)], Gt[pad4(D * D)], gb[pad4(D)];
                load_smem<pad4(D * D)>(rec + TB::E_OFF, Et);
                load_smem<pad4(D * D)>(rec + TB::G_OFF, Gt);
                if (OFFSET) load_smem<pad4(D)>(rec + TB::GB_OFF, gb);            // -G u
                float nm[D][CPT];
                if constexpr (USEQ == 1) {
                    input_back<D, CPT>(Et, Gt, fcur[s], ms, useq, t, T, batch, b, nm);
                } else {
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int c = 0; c < CPT; ++c) {
                        float a = OFFSET ? __fmaf_rn(Et[i * D], fcur[s][0][c], gb[i]) : Et[i * D] * fcur[s][0][c];
#pragma unroll
                        for (int j = 1; j < D; ++j) a = __fmaf_rn(Et[i * D + j], fcur[s][j][c], a);
#pragma unroll
                        for (int j = 0; j < D; ++j) a = __fmaf_rn(Gt[i * D + j], ms[j][c], a);
                        nm[i][c] = a;
                    }
                }
#pragma unroll
                for (int i = 0; i < D; ++i) {
#pragma unroll
                    for (int c = 0; c < CPT; ++c) ms[i][c] = nm[i][c];
                    if (active) Pack<CPT>::st(mean + ((int64_t)t * D + i) * batch + b, ms[i]);
                }
                float Sst[pad4(D * D)];
                if (write_cov && active) {
                    load_smem<pad4(D * D)>(rec + TB::SS_OFF, Sst);
#pragma unroll
                    for (int i = 0; i < D * D; ++i) {
                        float v[CPT];
#pragma unroll
                        for (int c = 0; c < CPT; ++c) v[c] = Sst[i];
                        Pack<CPT>::st(cov + ((int64_t)t * D * D + i) * batch + b, v);
                    }
                }
                if (PEER && active) peer_store<D, CPT>(po, write_cov, t, batch, b, ms, Sst);
            }
        }
#pragma unroll
        for (int s = 0; s < PF; ++s)
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int c = 0; c < CPT; ++c) fcur[s][i][c] = fnxt[s][i][c];
    }
    cp_async_wait<0>();
}

}  // namespace rxg
