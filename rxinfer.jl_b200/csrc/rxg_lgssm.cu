// Fused forward/backward sum-product sweeps for batched linear-Gaussian state-space models.
//
// What this replaces: for `batch` independent chains, the whole per-message schedule that
// infer(model = linear_gaussian_ssm_smoothing(...), data = (y = ...,)) runs through ReactiveMP
// and Rocket  [ref: /root/reference/src/inference/batch.jl:391-430 (iteration loop),
// benchmarks/Linear Multivariate Gaussian State Space Model Benchmark.ipynb:95-105 (model),
// src/model/plugins/reactivemp_inference.jl:365-374 (left-to-right product fold),
// src/rocket.jl:51-75 (stack-limited schedule)].  Per (chain, step) the reference evaluates
//   #1 *(:out)  #2 MvNormalMeanCovariance(:out)  #3 MvNormalMeanCovariance(:mu) from data
//   #4 *(:in)   #3' MvNormalMeanCovariance(:mu) backward   #4 *(:in) backward
// plus two outbound products and one 3-way marginal.  The kernels below compute the same
// messages in Kalman-gain / RTS form (algebraically identical, one SPD solve per direction
// instead of four cholinv), with (mu, Sigma) resident in registers for the whole sweep and
// the observation stream read coalesced over the batch axis.
//
// Two kernel families:
//  * lgssm_chain_kernel      one thread = one chain, full covariance recursion per chain
//                            (per-chain models, missing-data masks, or RXG_PATH_PER_CHAIN).
//  * lgssm_shared_kernel     shared (A,B,P,Q,S0): the covariance / gain trajectory is
//                            data-independent and identical across chains, so it is computed
//                            once into gain tables (fp64, gain_* kernels) and every chain only
//                            runs the mean recursions; covariances are broadcast-stored.
// In both, post_mean / post_cov double as the forward->backward stash.
#include <math.h>
#include <stdlib.h>

#include <utility>

#include "rxg_chain_step.cuh"
#include "rxg_gain.cuh"
#include "rxg_internal.h"
#include "rxg_linalg.cuh"
#include "rxg_lgssm_cluster.cuh"
#include "rxg_lgssm_common.cuh"
#include "rxg_lgssm_shared.cuh"
#include "rxg_lgssm_seg.cuh"
#include "rxg_sweep_select.h"

namespace rxg {

// ============================================================================================
// Family 1: one thread per chain, full (mu, Sigma) recursion
// ============================================================================================
// USEQ: per-step inputs, u[t] = useq[(t * D + i) * ustride + b * uchain] (a per-chain [rows][D][batch] sequence, or a
// shared [rows][D] one with ustride = 1, uchain = 0) replaces the constant offset.
template <int D, int M, bool PER_CHAIN, bool SMOOTH, bool USEQ = false>
__global__ void __launch_bounds__(128)
lgssm_chain_kernel(const __grid_constant__ ModelF<D, M> mdl, PerChainPtrs pc,
                   const float* __restrict__ y, const uint8_t* __restrict__ mask,
                   float* __restrict__ mean, float* __restrict__ cov, float* __restrict__ nle,
                   int32_t* __restrict__ status, int T, int64_t batch, int transition_first,
                   const float* __restrict__ useq = nullptr, int64_t ustride = 0, int uchain = 0) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;

    Mat<float, D, D> A, P, S0;
    Mat<float, M, D> B;
    Mat<float, M, M> Q;
    Vec<float, D> mu, u;
    if (PER_CHAIN) {
        A = load_strided<float, D, D>(pc.A + b, batch);
        B = load_strided<float, M, D>(pc.B + b, batch);
        P = load_strided<float, D, D>(pc.P + b, batch);
        Q = load_strided<float, M, M>(pc.Q + b, batch);
        S0 = load_strided<float, D, D>(pc.S0 + b, batch);
#pragma unroll
        for (int i = 0; i < D; ++i) mu(i) = __ldg(pc.m0 + i * batch + b);
#pragma unroll
        for (int i = 0; i < D; ++i) u(i) = pc.u ? __ldg(pc.u + i * batch + b) : 0.f;
    } else {
        A = load_const<float, D, D>(mdl.A);
        B = load_const<float, M, D>(mdl.B);
        P = load_const<float, D, D>(mdl.P);
        Q = load_const<float, M, M>(mdl.Q);
        S0 = load_const<float, D, D>(mdl.S0);
#pragma unroll
        for (int i = 0; i < D; ++i) { mu(i) = mdl.m0[i]; u(i) = mdl.u[i]; }
    }
    Mat<float, D, D> S = S0;
    bool bad = false;
    double acc_nle = 0.0;
    const bool want_nle = (nle != nullptr);

    // ---------------------------------------------------------------- forward (rules #1-#4)
    float ynext[M];
#pragma unroll
    for (int k = 0; k < M; ++k) ynext[k] = __ldg(y + (int64_t)k * batch + b);
    uint8_t onext = mask ? mask[b] : (uint8_t)1;

    for (int t = 0; t < T; ++t) {
        Vec<float, M> yt;
#pragma unroll
        for (int k = 0; k < M; ++k) yt(k) = ynext[k];
        const bool observed = onext != 0;
        if (t + 1 < T) {   // prefetch next step's datum while this step's arithmetic runs
#pragma unroll
            for (int k = 0; k < M; ++k) ynext[k] = __ldg(y + ((int64_t)(t + 1) * M + k) * batch + b);
            if (mask) onext = mask[(int64_t)(t + 1) * batch + b];
        }
        if (t > 0 || transition_first) {
            if constexpr (USEQ)
                chain_predict(A, P, u, [&](Vec<float, D>& uu) {
#pragma unroll
                    for (int i = 0; i < D; ++i) uu(i) = __ldg(useq + ((int64_t)t * D + i) * ustride + b * uchain);
                }, mu, S);
            else
                chain_predict(A, P, u, NoInput{}, mu, S);
        }
        if (observed) chain_update(B, Q, yt, want_nle, mu, S, bad, acc_nle);
        // filtered (mu, Sigma): the filter's output, the smoother's stash (lower triangle only)
#pragma unroll
        for (int i = 0; i < D; ++i) mean[((int64_t)t * D + i) * batch + b] = mu(i);
        const bool full = !SMOOTH || (t == T - 1);
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int j = 0; j < D; ++j)
                if (full || j <= i) cov[(((int64_t)t * D + i) * D + j) * batch + b] = S(i, j);
    }
    if (want_nle) nle[b] = (float)acc_nle;

    // ---------------------------------------------------------------- backward (rules #3',#4 + marginal)
    if (SMOOTH) {
        Vec<float, D> mus = mu;          // smoothed at t+1
        Mat<float, D, D> Ss = S;
        // prefetch stash of step T-2
        float pm[D], pS[D * (D + 1) / 2];
        if (T >= 2) {
            const int t = T - 2;
#pragma unroll
            for (int i = 0; i < D; ++i) pm[i] = mean[((int64_t)t * D + i) * batch + b];
            int q = 0;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j <= i; ++j) pS[q++] = cov[(((int64_t)t * D + i) * D + j) * batch + b];
        }
        for (int t = T - 2; t >= 0; --t) {
            Vec<float, D> muf;
            Mat<float, D, D> Sf;
#pragma unroll
            for (int i = 0; i < D; ++i) muf(i) = pm[i];
            {
                int q = 0;
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int j = 0; j <= i; ++j) { Sf(i, j) = pS[q]; Sf(j, i) = pS[q]; ++q; }
            }
            if (t > 0) {
                const int tp = t - 1;
#pragma unroll
                for (int i = 0; i < D; ++i) pm[i] = mean[((int64_t)tp * D + i) * batch + b];
                int q = 0;
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int j = 0; j <= i; ++j) pS[q++] = cov[(((int64_t)tp * D + i) * D + j) * batch + b];
            }
            if constexpr (USEQ)
                chain_rts(A, P, u, [&](Vec<float, D>& uu) {      // the transition into x[t+1]
#pragma unroll
                    for (int i = 0; i < D; ++i) uu(i) = __ldg(useq + ((int64_t)(t + 1) * D + i) * ustride + b * uchain);
                }, muf, Sf, mus, Ss, bad);
            else
                chain_rts(A, P, u, NoInput{}, muf, Sf, mus, Ss, bad);
#pragma unroll
            for (int i = 0; i < D; ++i) mean[((int64_t)t * D + i) * batch + b] = mus(i);
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j < D; ++j) cov[(((int64_t)t * D + i) * D + j) * batch + b] = Ss(i, j);
        }
        mu = mus;
    }
    if (status) {
        bool nan = false;
#pragma unroll
        for (int i = 0; i < D; ++i) nan |= !(mu(i) == mu(i));
        status[b] = bad ? RXG_ERR_NOT_SPD : (nan ? RXG_ERR_NAN : RXG_OK);
    }
}

// ============================================================================================
// Family 2: shared model -- gain tables (fp64) + mean-only sweeps
// ============================================================================================
// Phase 1 (sequential in t): Riccati recursion for the predicted / filtered covariances.
template <int D, int M>
__global__ void gain_riccati_seq(const __grid_constant__ ModelF<D, M> mdl, GainWs ws, int T,
                                 int transition_first, int* __restrict__ bad_out, const uint8_t* __restrict__ tmask) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const Mat<double, D, D> A = load_const<double, D, D>(mdl.A), P = load_const<double, D, D>(mdl.P);
    const Mat<double, M, D> B = load_const<double, M, D>(mdl.B);
    const Mat<double, M, M> Q = load_const<double, M, M>(mdl.Q);
    Mat<double, D, D> S = load_const<double, D, D>(mdl.S0);
    bool bad = false;
    for (int t = 0; t < T; ++t) {
        if (t > 0 || transition_first) {
            Mat<double, D, D> AS = mul(A, S);
            S = sym_mul_nt_add(AS, A, P);
        }
        store_d(ws.Sp + (size_t)t * D * D, S);
        if (!tmask || tmask[t] != 0) {
            Mat<double, M, D> BS = mul(B, S);
            Mat<double, M, M> Sinn = sym_mul_nt_add(BS, B, Q);
            Chol<double, M> ch = cholesky<double, M, false>(Sinn, bad);
            Mat<double, D, M> V = solve_right_Lt(transpose(BS), ch.L);
            S = sym_downdate(S, V);
        }
        store_d(ws.Sf + (size_t)t * D * D, S);
    }
    if (bad) atomicOr(bad_out, 1);
}

// Phase 2 (parallel in t): gains, innovation factors, conditional covariances.
template <int D, int M>
__global__ void gain_tables(const __grid_constant__ ModelF<D, M> mdl, GainWs ws, int T,
                            int transition_first, int* __restrict__ bad_out, const uint8_t* __restrict__ tmask,
                            const float* __restrict__ useq) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    using TB = Tab<D, M>;
    const Mat<double, D, D> A = load_const<double, D, D>(mdl.A);
    const Mat<double, M, D> B = load_const<double, M, D>(mdl.B);
    const Mat<double, M, M> Q = load_const<double, M, M>(mdl.Q);
    bool bad = false;
    const Mat<double, D, D> Sp = load_d<D, D>(ws.Sp + (size_t)t * D * D);
    const Mat<double, D, D> Sf = load_d<D, D>(ws.Sf + (size_t)t * D * D);
    {
        Mat<double, D, M> K;
        Mat<double, M, M> Li;
        double cconst = 0.0;
#pragma unroll
        for (int i = 0; i < D * M; ++i) K.a[i] = 0.0;
#pragma unroll
        for (int i = 0; i < M * M; ++i) Li.a[i] = 0.0;
        if (!tmask || tmask[t] != 0) {
            Mat<double, M, D> BS = mul(B, Sp);
            Mat<double, M, M> Sinn = sym_mul_nt_add(BS, B, Q);
            Chol<double, M> ch = cholesky<double, M, true>(Sinn, bad);
            Mat<double, D, M> V = solve_right_Lt(transpose(BS), ch.L);
            K = solve_right_L(V, ch.L);
#pragma unroll
            for (int j = 0; j < M; ++j) {
                Li(j, j) = ch.L(j, j);
#pragma unroll
                for (int i = j + 1; i < M; ++i) {
                    double sacc = 0.0;
#pragma unroll
                    for (int k = j; k < i; ++k) sacc -= ch.L(i, k) * Li(k, j);
                    Li(i, j) = sacc * ch.L(i, i);
                }
            }
            cconst = M * RXG_HALF_LOG_2PI - ch.neg_half_logdet;
        }
        Mat<double, D, D> IKB = identity<double, D>();
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int j = 0; j < D; ++j)
#pragma unroll
                for (int k = 0; k < M; ++k) IKB(i, j) -= K(i, k) * B(k, j);
        Mat<double, D, D> F = (t > 0 || transition_first) ? mul(IKB, A) : IKB;
        float* rec = ws.fwd + (size_t)t * TB::FWD_REC;
        store_f(rec + TB::F_OFF, F);
        store_f(rec + TB::K_OFF, K);
        store_f(rec + TB::LI_OFF, Li);
        rec[TB::C_OFF] = (float)cconst;
        Vec<double, D> uu, gf;
#pragma unroll
        for (int i = 0; i < D; ++i) uu(i) = (double)(useq ? useq[(size_t)t * D + i] : mdl.u[i]);
        gf = mulv(IKB, uu);
        if (!(t > 0 || transition_first)) {
#pragma unroll
            for (int i = 0; i < D; ++i) gf(i) = 0.0;
        }
        store_fv(rec + TB::GF_OFF, gf);
        store_f(ws.sf + (size_t)t * TB::SF_REC, Sf);
    }
    float* brec = ws.bwd + (size_t)t * TB::BWD_REC;
    Vec<double, D> gb;
#pragma unroll
    for (int i = 0; i < D; ++i) gb(i) = 0.0;
    if (t < T - 1) {
        const Mat<double, D, D> Sp1 = load_d<D, D>(ws.Sp + (size_t)(t + 1) * D * D);
        Chol<double, D> ch = cholesky<double, D, false>(Sp1, bad);
        Mat<double, D, D> AS = mul(A, Sf);
        Mat<double, D, D> U = solve_right_Lt(transpose(AS), ch.L);
        Mat<double, D, D> G = solve_right_L(U, ch.L);
        Mat<double, D, D> C = sym_downdate(Sf, U);
        Mat<double, D, D> E = identity<double, D>();
        Mat<double, D, D> GA = mul(G, A);
#pragma unroll
        for (int i = 0; i < D * D; ++i) E.a[i] -= GA.a[i];
        store_f(brec + TB::E_OFF, E);
        store_f(brec + TB::G_OFF, G);
        {
            Vec<double, D> uu;
#pragma unroll
            for (int i = 0; i < D; ++i) uu(i) = -(double)(useq ? useq[(size_t)(t + 1) * D + i] : mdl.u[i]);
            gb = mulv(G, uu);
        }
        store_d(ws.Cc + (size_t)t * D * D, C);
        store_d(ws.Gd + (size_t)t * D * D, G);
    } else {
        Mat<double, D, D> E = identity<double, D>();
        Mat<double, D, D> Z;
#pragma unroll
        for (int i = 0; i < D * D; ++i) Z.a[i] = 0.0;
        store_f(brec + TB::E_OFF, E);
        store_f(brec + TB::G_OFF, Z);
    }
    store_fv(brec + TB::GB_OFF, gb);
    if (bad) atomicOr(bad_out, 1);
}

// Phase 3 (sequential in t): smoothed covariances  Ss[t] = C[t] + G[t] Ss[t+1] G[t]'.
template <int D, int M>
__global__ void gain_smooth_seq(GainWs ws, int T, float* cov_shared_out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    using TB = Tab<D, M>;
    Mat<double, D, D> Ss = load_d<D, D>(ws.Sf + (size_t)(T - 1) * D * D);
    store_f(ws.bwd + (size_t)(T - 1) * TB::BWD_REC + TB::SS_OFF, Ss);
    if (cov_shared_out) store_f(cov_shared_out + (size_t)(T - 1) * D * D, Ss);
    for (int t = T - 2; t >= 0; --t) {
        const Mat<double, D, D> G = load_d<D, D>(ws.Gd + (size_t)t * D * D);
        const Mat<double, D, D> C = load_d<D, D>(ws.Cc + (size_t)t * D * D);
        Mat<double, D, D> GS = mul(G, Ss);
        Ss = sym_mul_nt_add(GS, G, C);
        store_f(ws.bwd + (size_t)t * TB::BWD_REC + TB::SS_OFF, Ss);
        if (cov_shared_out) store_f(cov_shared_out + (size_t)t * D * D, Ss);
    }
}

// Filter with shared cov output requested: copy the sf table (padded records) to [T][D][D].
static __global__ void copy_table_kernel(const float* __restrict__ tab, int rec, int n, int T, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < T * n) out[i] = tab[(size_t)(i / n) * rec + (i % n)];
}

// ============================================================================================
// host-side dispatch
// ============================================================================================
template <int D, int M>
static void fill_model(ModelF<D, M>& mdl, const LgssmCall& c) {
    for (int i = 0; i < D * D; ++i) { mdl.A[i] = c.A[i]; mdl.P[i] = c.P[i]; mdl.S0[i] = c.S0[i]; }
    for (int i = 0; i < M * D; ++i) mdl.B[i] = c.B[i];
    for (int i = 0; i < M * M; ++i) mdl.Q[i] = c.Q[i];
    for (int i = 0; i < D; ++i) { mdl.m0[i] = c.m0[i]; mdl.u[i] = c.u ? c.u[i] : 0.f; }
}

template <int D, int M, bool PER_CHAIN, bool SMOOTH>
static void launch_chain(rxg_ctx* ctx, const LgssmCall& c, const ModelF<D, M>& mdl, const PerChainPtrs& pc) {
    const int threads = 64;
    const unsigned blocks = (unsigned)((c.batch + threads - 1) / threads);
    const int tf = (c.flags & RXG_TRANSITION_FIRST) ? 1 : 0;
    if (c.useq)
        lgssm_chain_kernel<D, M, PER_CHAIN, SMOOTH, true><<<blocks, threads, 0, ctx->stream>>>(
            mdl, pc, c.y, c.ymask, c.mean, c.cov, c.nle, c.status, c.T, c.batch, tf, c.useq, c.useq_chain ? c.batch : 1,
            c.useq_chain ? 1 : 0);
    else
        lgssm_chain_kernel<D, M, PER_CHAIN, SMOOTH><<<blocks, threads, 0, ctx->stream>>>(
            mdl, pc, c.y, c.ymask, c.mean, c.cov, c.nle, c.status, c.T, c.batch, tf);
}

template <int D, int M>
static int run_chain_family(rxg_ctx* ctx, LgssmCall& c) {
    ModelF<D, M> mdl = {};
    PerChainPtrs pc = {};
    const bool per_chain = (c.flags & RXG_MODEL_PER_CHAIN) != 0;
    if (per_chain) pc = PerChainPtrs{c.A, c.B, c.P, c.Q, c.m0, c.S0, c.u};
    else fill_model<D, M>(mdl, c);
    if (ctx->profile) { cudaEventRecord(ctx->ev[0], ctx->stream); cudaEventRecord(ctx->ev[1], ctx->stream); }
    if (per_chain) (c.smooth ? launch_chain<D, M, true, true> : launch_chain<D, M, true, false>)(ctx, c, mdl, pc);
    else           (c.smooth ? launch_chain<D, M, false, true> : launch_chain<D, M, false, false>)(ctx, c, mdl, pc);
    if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "lgssm_chain_kernel launch");
}

// Launches lgssm_shared_kernel if pick index I is the call's pick.  Only the picks select_shared_sweep can return
// (sweep_pick_reachable) are instantiated.
template <int D, int M, int I>
static bool launch_sweep_if(int pick, rxg_ctx* ctx, const LgssmCall& c, const ModelF<D, M>& mdl, const GainWs& ws,
                            int write_cov) {
    constexpr SweepPick p = sweep_pick_at(I);
    if constexpr (sweep_pick_reachable(D, M, p)) {
        if (pick == I) {
            const int threads = 32;                     // one warp per CTA (see rxg_lgssm_shared.cuh)
            const unsigned blocks = (unsigned)((c.batch / p.cpt + threads - 1) / threads);
            const int tf = (c.flags & RXG_TRANSITION_FIRST) ? 1 : 0;
            lgssm_shared_kernel<D, M, p.cpt, 4, p.smooth, p.evid, p.offset, p.ckpt, p.peer, p.useq>
                <<<blocks, threads, 0, ctx->stream>>>(mdl, ws.fwd, ws.bwd, ws.sf, c.y, c.mean, c.cov, c.nle, c.T, c.batch,
                                                      tf, write_cov, c.mean0_chain, c.po, p.useq ? c.useq : nullptr);
            return true;
        }
    }
    return false;
}
template <int D, int M, int... I>
static bool launch_sweep(int pick, rxg_ctx* ctx, const LgssmCall& c, const ModelF<D, M>& mdl, const GainWs& ws,
                         int write_cov, std::integer_sequence<int, I...>) {
    return (launch_sweep_if<D, M, I>(pick, ctx, c, mdl, ws, write_cov) || ...);
}

template <int D, int M>
static int launch_shared(rxg_ctx* ctx, LgssmCall& c, const ModelF<D, M>& mdl, const GainWs& ws, int write_cov,
                         const SweepPick& p) {
    const int pick = sweep_pick_index(p);
    if (ctx->profile) cudaEventRecord(ctx->ev[1], ctx->stream);
    if (!launch_sweep<D, M>(pick, ctx, c, mdl, ws, write_cov, std::make_integer_sequence<int, SWEEP_PICK_COUNT>{}))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm: no lgssm_shared_kernel instantiation for sweep pick %d", pick);
    if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
    ctx->launches += 1;
    // the PEER instantiation stores the final posteriors to c.po itself; otherwise the caller pushes the finished slab
    c.fused_peer_stores = p.peer;
    return check_cuda(ctx, cudaGetLastError(), "lgssm_shared_kernel launch");
}

// time-segmented sweep (rxg_lgssm_seg.cuh): smoothing without evidence, d^2 <= 16, T up to the shared-memory budget
template <int D, int M>
static bool seg_sweep_eligible(const LgssmCall& c) {
    using ST = SegTab<D, M>;
    if (!c.smooth || c.nle || D * D > 16) return false;
    const int nseg = (c.T + ST::L - 1) / ST::L;
    const size_t smem = (size_t)nseg * 2 * D * 32 * 4 + (size_t)8 * 2 * ST::L * ST::REC * 4;
    return smem <= 200 * 1024;
}
template <int D, int M>
static int launch_seg(rxg_ctx* ctx, LgssmCall& c, const ModelF<D, M>& mdl, const GainWs& ws, const SegWs& sw, int write_cov,
                      bool hints) {
    using ST = SegTab<D, M>;
    constexpr int NW = 8;
    const int nseg = (c.T + ST::L - 1) / ST::L;
    seg_tables_kernel<D, M><<<(nseg + 63) / 64, 64, 0, ctx->stream>>>(ws, sw, c.T);
    const size_t smem = (size_t)nseg * 2 * D * 32 * 4 + (size_t)NW * 2 * ST::L * ST::REC * 4;
    const int64_t ntiles = (c.batch + 31) / 32;
    const unsigned grid = (unsigned)(ntiles < ctx->sm_count ? ntiles : ctx->sm_count);
    bool has_u = false;
    for (int i = 0; i < D; ++i) has_u |= (mdl.u[i] != 0.f);
#define RXG_LAUNCH_SEG(OF, HI)                                                                                        \
    do {                                                                                                               \
        RXG_CUDA(ctx, cudaFuncSetAttribute(lgssm_seg_kernel<D, M, NW, OF, HI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        if (ctx->profile) cudaEventRecord(ctx->ev[1], ctx->stream);                                                    \
        lgssm_seg_kernel<D, M, NW, OF, HI><<<grid, 32 * NW, smem, ctx->stream>>>(mdl, sw, c.y, c.mean, c.cov, c.T, c.batch, \
                                                                                 write_cov, c.mean0_chain, c.po, nseg);  \
    } while (0)
    (void)hints;
    if (has_u) RXG_LAUNCH_SEG(true, 1); else RXG_LAUNCH_SEG(false, 1);
#undef RXG_LAUNCH_SEG
    if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
    ctx->launches += 2;
    c.fused_peer_stores = false;
    return check_cuda(ctx, cudaGetLastError(), "lgssm_seg_kernel launch");
}

// cluster sweep (rxg_lgssm_cluster.cuh): plain smoothing (no evidence, offset, inputs or per-chain prior mean -- the
// streaming chunk, the only caller with one, filters) at d * d <= 16, m >= d, whole 32-chain tiles of 16-byte aligned
// buffers, the default dispatch options, T within the shared-memory budget, and a cluster shape the device can hold
// resident.  Every other call keeps lgssm_shared_kernel / lgssm_seg_kernel.  A fused gather takes the PEER instantiation:
// the gathered buffers must hold the bits of the plain sweep.
template <int D, int M>
static int launch_cluster_if_eligible(rxg_ctx* ctx, LgssmCall& c, const ModelF<D, M>& mdl, const GainWs& ws, float* cl_tab,
                                      int write_cov, bool& launched) {
    launched = false;
    if constexpr (D * D <= 16 && M >= D) {
        using CT = ClusterTab<D, M>;
        bool offset = false;
        for (int i = 0; i < D; ++i) offset |= (mdl.u[i] != 0.f);
        const bool aligned = (((uintptr_t)c.y | (uintptr_t)c.mean | (uintptr_t)c.cov) & 15) == 0;
        if (!c.smooth || c.nle || c.useq || offset || c.mean0_chain || c.batch % 32 != 0 || !aligned ||
            ctx->opt[RXG_OPT_SWEEP_VARIANT] != 0 || ctx->opt[RXG_OPT_FORCE_CPT] != 0)
            return RXG_OK;
        const size_t smem = CT::smem_bytes(c.T);
        int smem_max = 0;
        RXG_CUDA(ctx, cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
        if (smem > (size_t)smem_max) return RXG_OK;
        const bool peer = c.po.n_mean > 0 || c.po.n_cov > 0;
        auto kern = peer ? lgssm_cluster_sweep_kernel<D, M, true> : lgssm_cluster_sweep_kernel<D, M, false>;
        RXG_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        cudaLaunchConfig_t cfg = {};
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = CL_CTAS;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.gridDim = dim3((unsigned)(c.batch / 32 * CL_CTAS));
        cfg.blockDim = dim3(32 * CL_WARPS);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = ctx->stream;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int nclusters = 0;
        RXG_CUDA(ctx, cudaOccupancyMaxActiveClusters(&nclusters, kern, &cfg));
        if (nclusters < 1) return RXG_OK;

        const int spc = CT::spc(c.T);
        cluster_tables_kernel<D, M><<<1, 256, 0, ctx->stream>>>(ws, cl_tab, c.T, spc);
        if (ctx->profile) cudaEventRecord(ctx->ev[1], ctx->stream);
        RXG_CUDA(ctx, cudaLaunchKernelEx(&cfg, kern, (const float*)ws.fwd, (const float*)ws.bwd, (const float*)cl_tab, c.y,
                                         c.mean, c.cov, c.T, c.batch, write_cov, mdl, c.po));
        if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
        ctx->launches += 2;
        c.fused_peer_stores = peer;
        launched = true;
        return check_cuda(ctx, cudaGetLastError(), "lgssm_cluster_sweep_kernel launch");
    }
    return RXG_OK;
}

template <int D, int M>
static int run_shared_family(rxg_ctx* ctx, LgssmCall& c) {
    using TB = Tab<D, M>;
    ModelF<D, M> mdl = {};
    fill_model<D, M>(mdl, c);
    const size_t T = (size_t)c.T;
    // carve the workspace
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
    const size_t o_fwd = carve(T * TB::FWD_REC * sizeof(float));
    const size_t o_bwd = carve(T * TB::BWD_REC * sizeof(float));
    const size_t o_sf = carve(T * TB::SF_REC * sizeof(float));
    const size_t o_Sp = carve(T * D * D * sizeof(double));
    const size_t o_Sf = carve(T * D * D * sizeof(double));
    const size_t o_Cc = carve(T * D * D * sizeof(double));
    const size_t o_Gd = carve(T * D * D * sizeof(double));
    const size_t o_fel = carve(T * 3 * D * D * sizeof(double));
    const size_t o_ftot = carve((size_t)2 * GS_NT * 3 * D * D * sizeof(double));
    const size_t o_bel = carve(T * 2 * D * D * sizeof(double));
    const size_t o_btot = carve((size_t)2 * GS_NT * 2 * D * D * sizeof(double));
    using ST = SegTab<D, M>;
    const size_t nseg = (T + ST::L - 1) / ST::L;
    const size_t o_srec_t = carve(T * ST::REC * sizeof(float)), o_snrec = carve(T * ST::NREC * sizeof(float));
    const size_t o_ssrec = carve(nseg * ST::SREC * sizeof(float));
    const size_t o_ctab = carve(c.want_cov_table ? T * D * D * sizeof(float) : 0);
    const size_t o_cl = carve(ClusterTab<D, M>::table_floats(c.T) * sizeof(float));
    char* base = (char*)workspace(ctx, off);
    if (!base) return RXG_ERR_CUDA;
    GainWs ws;
    ws.fwd = (float*)(base + o_fwd); ws.bwd = (float*)(base + o_bwd); ws.sf = (float*)(base + o_sf);
    ws.Sp = (double*)(base + o_Sp); ws.Sf = (double*)(base + o_Sf);
    ws.Cc = (double*)(base + o_Cc); ws.Gd = (double*)(base + o_Gd);
    ScanWs sw;
    sw.fel = (double*)(base + o_fel); sw.ftot = (double*)(base + o_ftot);
    sw.bel = (double*)(base + o_bel); sw.btot = (double*)(base + o_btot);

    const int tf = (c.flags & RXG_TRANSITION_FIRST) ? 1 : 0;
    const bool cov_shared = (c.flags & RXG_COV_SHARED_OUT) != 0;
    c.cov_table = (c.want_cov_table && c.smooth) ? (float*)(base + o_ctab) : nullptr;
    if (ctx->profile) cudaEventRecord(ctx->ev[0], ctx->stream);
    float* cov_once = (cov_shared && c.cov && c.smooth) ? c.cov : (c.smooth ? c.cov_table : nullptr);
    // a shared input sequence goes into the tables' offset terms; a per-chain one into the sweep (tables without inputs)
    const float* useq_tab = c.useq_chain ? nullptr : c.useq;
    if (ctx->opt[RXG_OPT_GAIN_SEQ] != 0) {
        // sequential Riccati recursion (cross-check of the scan; ~70x slower at T = 1000)
        gain_riccati_seq<D, M><<<1, 32, 0, ctx->stream>>>(mdl, ws, c.T, tf, bad_flag(ctx), c.tmask);
        gain_tables<D, M><<<(c.T + 63) / 64, 64, 0, ctx->stream>>>(mdl, ws, c.T, tf, bad_flag(ctx), c.tmask, useq_tab);
        ctx->launches += 2;
        if (c.smooth) {
            gain_smooth_seq<D, M><<<1, 32, 0, ctx->stream>>>(ws, c.T, cov_once);
            ctx->launches += 1;
        }
    } else {
        // time-parallel associative scans in one 8-CTA cluster
        gain_scan_kernel<D, M><<<GS_CTAS, GS_THREADS, 0, ctx->stream>>>(mdl, ws, sw, c.T, tf, cov_once, bad_flag(ctx), c.tmask,
                                                                          useq_tab);
        ctx->launches += 1;
    }
    if (!c.smooth && cov_shared && c.cov) {
        const int n = c.T * D * D;
        copy_table_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(ws.sf, TB::SF_REC, D * D, c.T, c.cov);
        ctx->launches += 1;
    }
    int rc = check_cuda(ctx, cudaGetLastError(), "gain table kernels launch");
    if (rc != RXG_OK) return rc;
    if (c.ev_tables) RXG_CUDA(ctx, cudaEventRecord(c.ev_tables, ctx->stream));
    if (c.tables_only) return RXG_OK;
    const int write_cov = (c.cov != nullptr && !cov_shared) ? 1 : 0;
    bool launched = false;
    rc = launch_cluster_if_eligible<D, M>(ctx, c, mdl, ws, (float*)(base + o_cl), write_cov, launched);
    if (rc != RXG_OK || launched) return rc;
    // sweep variant (RXG_OPT_SWEEP_VARIANT): 3 / 4 = time-segmented kernel with / without L2 eviction hints
    const long long variant = ctx->opt[RXG_OPT_SWEEP_VARIANT];
    if (variant == 3 && !c.useq && seg_sweep_eligible<D, M>(c)) {      // inputs: the lock-step kernel
        SegWs sgw;
        sgw.rec = (float*)(base + o_srec_t); sgw.nrec = (float*)(base + o_snrec); sgw.srec = (float*)(base + o_ssrec);
        return launch_seg<D, M>(ctx, c, mdl, ws, sgw, write_cov, variant == 3);
    }
    SweepQuery q = {};
    q.d = D;
    q.m = M;
    q.batch = c.batch;
    q.sm_count = ctx->sm_count;
    q.force_cpt = ctx->opt[RXG_OPT_FORCE_CPT];
    q.aligned16 = (((uintptr_t)c.y | (uintptr_t)c.mean | (uintptr_t)c.cov | (uintptr_t)c.nle | (uintptr_t)c.mean0_chain |
                    (uintptr_t)(c.useq_chain ? c.useq : nullptr)) & 15) == 0;
    q.smooth = c.smooth;
    q.evid = c.nle != nullptr;
    for (int i = 0; i < D; ++i) q.offset |= (mdl.u[i] != 0.f);
    q.input = !c.useq ? InputSeq::none : (c.useq_chain ? InputSeq::per_chain : InputSeq::shared);
    q.peer_out = c.po.n_mean > 0 || c.po.n_cov > 0;
    q.sweep_variant = variant;
    return launch_shared<D, M>(ctx, c, mdl, ws, write_cov, select_shared_sweep(q));
}

template <int D, int M>
int run_dm(rxg_ctx* ctx, LgssmCall& c) {
    const bool per_chain = (c.flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN)) != 0 || c.ymask != nullptr;
    if (per_chain) return run_chain_family<D, M>(ctx, c);
    int rc = run_shared_family<D, M>(ctx, c);
    if (rc == RXG_OK && c.status) rc = fill_status_from_flag(ctx, c.status, c.batch);
    return rc;
}

// This translation unit is compiled once per (d, m) shape with -DRXG_INST_D / -DRXG_INST_M (explicit instantiation
// of run_dm: the kernel variants of one shape), in parallel, and once without them for the dispatch below.
#ifdef RXG_INST_D
template int run_dm<RXG_INST_D, RXG_INST_M>(rxg_ctx*, LgssmCall&);
#else
extern template int run_dm<1, 1>(rxg_ctx*, LgssmCall&);
extern template int run_dm<2, 1>(rxg_ctx*, LgssmCall&);
extern template int run_dm<2, 2>(rxg_ctx*, LgssmCall&);
extern template int run_dm<3, 3>(rxg_ctx*, LgssmCall&);
extern template int run_dm<4, 1>(rxg_ctx*, LgssmCall&);
extern template int run_dm<4, 2>(rxg_ctx*, LgssmCall&);
extern template int run_dm<4, 4>(rxg_ctx*, LgssmCall&);
extern template int run_dm<6, 6>(rxg_ctx*, LgssmCall&);

// shared model: a failed Cholesky of the chain-independent covariance recursion fails every chain alike
__global__ void fill_status_kernel(int32_t* s, int64_t n, const int* __restrict__ bad) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) s[i] = (*bad != 0) ? (int32_t)RXG_ERR_NOT_SPD : (int32_t)RXG_OK;
}
int fill_status_from_flag(rxg_ctx* ctx, int32_t* status, int64_t n) {
    fill_status_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(status, n, bad_flag(ctx));
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "fill_status launch");
}

int lgssm_dispatch_native(rxg_ctx* ctx, LgssmCall& c) {
    switch (c.d * 16 + c.m) {
        case 1 * 16 + 1: return run_dm<1, 1>(ctx, c);
        case 2 * 16 + 1: return run_dm<2, 1>(ctx, c);
        case 2 * 16 + 2: return run_dm<2, 2>(ctx, c);
        case 3 * 16 + 3: return run_dm<3, 3>(ctx, c);
        case 4 * 16 + 1: return run_dm<4, 1>(ctx, c);
        case 4 * 16 + 2: return run_dm<4, 2>(ctx, c);
        case 4 * 16 + 4: return run_dm<4, 4>(ctx, c);
        case 6 * 16 + 6: return run_dm<6, 6>(ctx, c);
        default:
            return fail(ctx, RXG_ERR_UNSUPPORTED,
                        "lgssm: (d=%d, m=%d) is outside the register-resident kernel families", c.d, c.m);
    }
}

#endif  // RXG_INST_D

}  // namespace rxg
