// Gain-table precompute for the shared-model LGSSM path, parallel in TIME.
//
// With shared (A, B, P, Q, S0) every covariance-valued message of the reference's schedule is
// data independent (SURVEY.md appendix A.1): predicted / filtered / smoothed covariances and the
// Kalman / RTS gains are the same for all chains.  They are computed once per call, in fp64, by
// ONE thread-block cluster (8 CTAs x 128 threads, distributed over 8 SMs, cluster.sync between
// phases) using associative scans over time instead of the sequential Riccati recursion:
//
//   forward   elements a_k = (A_k, C_k, J_k) of Sarkka & Garcia-Fernandez, "Temporal
//             parallelization of Bayesian smoothers" (2021), covariance parts only:
//               a_i (x) a_j = ( A_j W A_i,  A_j W C_i A_j' + C_j,  A_i' J_j W A_i + J_i ),
//               W = (I + C_i J_j)^-1 ;   prefix(a_1..a_k).C = filtered covariance at k
//   per-t     Kalman gain, innovation factor, RTS gain, conditional covariance (parallel over t)
//   backward  elements (E_k, L_k) = (G_k, Sigma_f,k - G_k Sigma_p,k+1 G_k'):
//               a_i (x) a_j = ( E_i E_j,  E_i L_j E_i' + L_i );  suffix(a_k..a_T).L = smoothed cov
//
// Depth is O(T / 1024 + log 1024) combines instead of O(T) Riccati steps.  The sequential kernels in rxg_lgssm.cu remain as the
// cross-check (RXG_GAIN_SEQ=1).
#pragma once
#include <cooperative_groups.h>

#include "rxg_lgssm_common.cuh"

namespace rxg {
namespace cg = cooperative_groups;

constexpr int GS_CTAS = 8;
constexpr int GS_THREADS = 128;
constexpr int GS_NT = GS_CTAS * GS_THREADS;

struct ScanWs {
    double* fel;    // [T][3*D*D]      forward local prefixes (only used when T > GS_NT)
    double* ftot;   // [2][GS_NT][3*D*D]
    double* bel;    // [T][2*D*D]      backward elements / local prefixes
    double* btot;   // [2][GS_NT][2*D*D]
};

template <int R, int C>
__device__ __forceinline__ Mat<double, R, C> ldcg_d(const double* p) {
    Mat<double, R, C> o;
#pragma unroll
    for (int i = 0; i < R * C; ++i) o.a[i] = __ldcg(p + i);
    return o;
}
// Scan elements live in global scratch as structure-of-arrays over the element index (component
// c of element i at p[c * n + i]) so that the 32 lanes of a warp touch consecutive doubles.
template <int R, int C>
__device__ __forceinline__ Mat<double, R, C> ld_soa_d(const double* p, size_t n, size_t i) {
    Mat<double, R, C> o;
#pragma unroll
    for (int c = 0; c < R * C; ++c) o.a[c] = __ldcg(p + (size_t)c * n + i);
    return o;
}
template <int R, int C>
__device__ __forceinline__ void st_soa_d(double* p, size_t n, size_t i, const Mat<double, R, C>& A) {
#pragma unroll
    for (int c = 0; c < R * C; ++c) p[(size_t)c * n + i] = A.a[c];
}

// X = M^-1 R  by Gaussian elimination with partial pivoting (M is I + C J: nonsymmetric).
template <int N, int K>
__device__ __forceinline__ Mat<double, N, K> solve_general(Mat<double, N, N> Mx, Mat<double, N, K> Rh) {
#pragma unroll
    for (int c = 0; c < N; ++c) {
        int p = c;
        double best = fabs(Mx(c, c));
#pragma unroll
        for (int r = c + 1; r < N; ++r) {
            const double v = fabs(Mx(r, c));
            if (v > best) { best = v; p = r; }
        }
#pragma unroll
        for (int r = c + 1; r < N; ++r) {
            if (r == p) {
#pragma unroll
                for (int j = c; j < N; ++j) { const double t = Mx(c, j); Mx(c, j) = Mx(r, j); Mx(r, j) = t; }
#pragma unroll
                for (int j = 0; j < K; ++j) { const double t = Rh(c, j); Rh(c, j) = Rh(r, j); Rh(r, j) = t; }
            }
        }
        const double inv = 1.0 / Mx(c, c);
#pragma unroll
        for (int r = c + 1; r < N; ++r) {
            const double f = Mx(r, c) * inv;
#pragma unroll
            for (int j = c + 1; j < N; ++j) Mx(r, j) = fma(-f, Mx(c, j), Mx(r, j));
#pragma unroll
            for (int j = 0; j < K; ++j) Rh(r, j) = fma(-f, Rh(c, j), Rh(r, j));
        }
    }
    Mat<double, N, K> X;
#pragma unroll
    for (int c = N - 1; c >= 0; --c) {
        const double inv = 1.0 / Mx(c, c);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double s = Rh(c, k);
#pragma unroll
            for (int j = c + 1; j < N; ++j) s = fma(-Mx(c, j), X(j, k), s);
            X(c, k) = s * inv;
        }
    }
    return X;
}

template <int D>
struct FwdEl {
    Mat<double, D, D> A, C, J;
};
template <int D>
struct BwdEl {
    Mat<double, D, D> E, L;
};

template <int D>
__device__ __forceinline__ FwdEl<D> fwd_identity() {
    FwdEl<D> e;
    e.A = identity<double, D>();
#pragma unroll
    for (int i = 0; i < D * D; ++i) { e.C.a[i] = 0.0; e.J.a[i] = 0.0; }
    return e;
}
template <int D>
__device__ __forceinline__ void fwd_store(double* p, size_t n, size_t i, const FwdEl<D>& e) {
    st_soa_d<D, D>(p, n, i, e.A);
    st_soa_d<D, D>(p + (size_t)D * D * n, n, i, e.C);
    st_soa_d<D, D>(p + (size_t)2 * D * D * n, n, i, e.J);
}
template <int D>
__device__ __forceinline__ FwdEl<D> fwd_load(const double* p, size_t n, size_t i) {
    FwdEl<D> e;
    e.A = ld_soa_d<D, D>(p, n, i);
    e.C = ld_soa_d<D, D>(p + (size_t)D * D * n, n, i);
    e.J = ld_soa_d<D, D>(p + (size_t)2 * D * D * n, n, i);
    return e;
}
// a_i (x) a_j, i earlier in time
template <int D, bool C_ONLY>
__device__ __forceinline__ FwdEl<D> fwd_combine(const FwdEl<D>& ei, const FwdEl<D>& ej) {
    Mat<double, D, D> Mx = mul(ei.C, ej.J);
#pragma unroll
    for (int i = 0; i < D; ++i) Mx(i, i) += 1.0;
    Mat<double, D, 2 * D> Rh;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) { Rh(i, j) = ei.A(i, j); Rh(i, D + j) = ei.C(i, j); }
    Mat<double, D, 2 * D> X = solve_general<D, 2 * D>(Mx, Rh);
    Mat<double, D, D> X1, X2;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) { X1(i, j) = X(i, j); X2(i, j) = X(i, D + j); }
    FwdEl<D> o;
    Mat<double, D, D> T2 = mul(ej.A, X2);
    o.C = sym_mul_nt_add(T2, ej.A, ej.C);
    if (!C_ONLY) {
        o.A = mul(ej.A, X1);
        Mat<double, D, D> JX = mul(ej.J, X1);
        Mat<double, D, D> AtJX = mul_tn(ei.A, JX);
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int j = 0; j <= i; ++j) {
                const double s = 0.5 * (AtJX(i, j) + AtJX(j, i)) + ei.J(i, j);
                o.J(i, j) = s; o.J(j, i) = s;
            }
    }
    return o;
}

template <int D>
__device__ __forceinline__ void bwd_store(double* p, size_t n, size_t i, const BwdEl<D>& e) {
    st_soa_d<D, D>(p, n, i, e.E);
    st_soa_d<D, D>(p + (size_t)D * D * n, n, i, e.L);
}
template <int D>
__device__ __forceinline__ BwdEl<D> bwd_load(const double* p, size_t n, size_t i) {
    BwdEl<D> e;
    e.E = ld_soa_d<D, D>(p, n, i);
    e.L = ld_soa_d<D, D>(p + (size_t)D * D * n, n, i);
    return e;
}
// (earlier-in-time element) (x) (accumulated later-in-time element)
template <int D, bool L_ONLY>
__device__ __forceinline__ BwdEl<D> bwd_combine(const BwdEl<D>& early, const BwdEl<D>& late) {
    BwdEl<D> o;
    Mat<double, D, D> EL = mul(early.E, late.L);
    o.L = sym_mul_nt_add(EL, early.E, early.L);
    if (!L_ONLY) o.E = mul(early.E, late.E);
    return o;
}

template <int D, int M>
__global__ void __cluster_dims__(GS_CTAS, 1, 1) __launch_bounds__(GS_THREADS, 1)
gain_scan_kernel(const __grid_constant__ ModelF<D, M> mdl, GainWs ws, ScanWs sw, int T, int transition_first,
                 float* __restrict__ cov_shared_out, int* __restrict__ bad_out, const uint8_t* __restrict__ tmask,
                 const float* __restrict__ useq) {
    // useq[T][D] (or null for the constant mdl.u): a shared input sequence (RXG_U_SEQ_SHARED) -- the offset terms
    // become gf_t = (I - K_t B) u_t and gb_t = -G_t u_{t+1}; nothing else depends on it.
    // tmask[T] (or null): 1 = the datum of step t exists for EVERY chain, 0 = missing for every chain (RXG_MASK_SHARED).
    // A missing step is a pure transition: scan element (A, P, 0), no gain, no evidence term -- the covariances stay
    // chain independent, so the whole batch stays on this path instead of the per-chain covariance recursion.
    using TB = Tab<D, M>;
    cg::cluster_group cluster = cg::this_cluster();
    const int g = (int)cluster.block_rank() * GS_THREADS + (int)threadIdx.x;
    const int E = (T + GS_NT - 1) / GS_NT;
    const int k0 = g * E, k1 = min(k0 + E, T);
    constexpr int FE = 3 * D * D, BE = 2 * D * D;
    bool bad = false;

    const Mat<double, D, D> A = load_const<double, D, D>(mdl.A), P = load_const<double, D, D>(mdl.P);
    const Mat<double, M, D> B = load_const<double, M, D>(mdl.B);
    const Mat<double, M, M> Q = load_const<double, M, M>(mdl.Q);

    // ------------------------------------------------------------------ F1: elements + local prefixes
    {
        FwdEl<D> acc = fwd_identity<D>();
        if (k0 < k1) {
            FwdEl<D> gen;   // time-invariant element for k >= 1
            {
                Mat<double, M, D> BP = mul(B, P);
                Mat<double, M, M> Sinn = sym_mul_nt_add(BP, B, Q);
                Chol<double, M> ch = cholesky<double, M, false>(Sinn, bad);
                Mat<double, D, M> V = solve_right_Lt(transpose(BP), ch.L);   // P B' L^-T
                Mat<double, D, M> K = solve_right_L(V, ch.L);
                Mat<double, D, D> IKB = identity<double, D>();
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int j = 0; j < D; ++j)
#pragma unroll
                        for (int k = 0; k < M; ++k) IKB(i, j) -= K(i, k) * B(k, j);
                gen.A = mul(IKB, A);
                gen.C = sym_downdate(P, V);
                Mat<double, M, D> BA = mul(B, A);
                // W = L^-1 (B A): column by column forward substitution
                Mat<double, M, D> Wm;
#pragma unroll
                for (int c = 0; c < D; ++c) {
                    Vec<double, M> col;
#pragma unroll
                    for (int r = 0; r < M; ++r) col(r) = BA(r, c);
                    Vec<double, M> z = solve_L(ch.L, col);
#pragma unroll
                    for (int r = 0; r < M; ++r) Wm(r, c) = z(r);
                }
                Mat<double, D, D> Z;
#pragma unroll
                for (int i = 0; i < D * D; ++i) Z.a[i] = 0.0;
                gen.J = sym_mul_nt_add(transpose(Wm), transpose(Wm), Z);
            }
            for (int k = k0; k < k1; ++k) {
                if (k == 0) {
                    Mat<double, D, D> S = load_const<double, D, D>(mdl.S0);
                    if (transition_first) { Mat<double, D, D> AS = mul(A, S); S = sym_mul_nt_add(AS, A, P); }
                    FwdEl<D> first;
#pragma unroll
                    for (int i = 0; i < D * D; ++i) { first.A.a[i] = 0.0; first.J.a[i] = 0.0; }
                    if (!tmask || tmask[0] != 0) {
                        Mat<double, M, D> BS = mul(B, S);
                        Mat<double, M, M> Sinn = sym_mul_nt_add(BS, B, Q);
                        Chol<double, M> ch = cholesky<double, M, false>(Sinn, bad);
                        Mat<double, D, M> V = solve_right_Lt(transpose(BS), ch.L);
                        first.C = sym_downdate(S, V);
                    } else {
                        first.C = S;
                    }
                    acc = first;
                } else {
                    const bool obs_k = !tmask || tmask[k] != 0;
                    if (obs_k) {
                        acc = (k == k0) ? gen : fwd_combine<D, false>(acc, gen);
                    } else {
                        FwdEl<D> miss;
                        miss.A = A; miss.C = P;
#pragma unroll
                        for (int i = 0; i < D * D; ++i) miss.J.a[i] = 0.0;
                        acc = (k == k0) ? miss : fwd_combine<D, false>(acc, miss);
                    }
                }
                if (E > 1) fwd_store<D>(sw.fel, T, k, acc);
            }
        }
        fwd_store<D>(sw.ftot, GS_NT, g, acc);
    }
    cluster.sync();
    // ------------------------------------------------------------------ F2: Hillis-Steele over thread totals
    int cur = 0;
    for (int off = 1; off < GS_NT; off <<= 1) {
        const double* src = sw.ftot + (size_t)cur * GS_NT * FE;
        double* dst = sw.ftot + (size_t)(cur ^ 1) * GS_NT * FE;
        FwdEl<D> mine = fwd_load<D>(src, GS_NT, g);
        if (g >= off && (g - off) * E < T && k0 < T) {
            FwdEl<D> prev = fwd_load<D>(src, GS_NT, g - off);
            mine = fwd_combine<D, false>(prev, mine);
        }
        fwd_store<D>(dst, GS_NT, g, mine);
        cluster.sync();
        cur ^= 1;
    }
    // ------------------------------------------------------------------ F3: filtered covariances
    {
        const double* tot = sw.ftot + (size_t)cur * GS_NT * FE;
        if (E == 1) {
            if (g < T) store_d(ws.Sf + (size_t)g * D * D, ld_soa_d<D, D>(tot + (size_t)D * D * GS_NT, GS_NT, g));
        } else if (k0 < k1) {
            if (g == 0) {
                for (int k = k0; k < k1; ++k)
                    store_d(ws.Sf + (size_t)k * D * D, ld_soa_d<D, D>(sw.fel + (size_t)D * D * T, T, k));
            } else {
                const FwdEl<D> excl = fwd_load<D>(tot, GS_NT, g - 1);
                for (int k = k0; k < k1; ++k) {
                    const FwdEl<D> pk = fwd_load<D>(sw.fel, T, k);
                    store_d(ws.Sf + (size_t)k * D * D, fwd_combine<D, true>(excl, pk).C);
                }
            }
        }
    }
    cluster.sync();
    // ------------------------------------------------------------------ G: per-step gains (parallel over t)
    for (int t = g; t < T; t += GS_NT) {
        const Mat<double, D, D> Sf = ldcg_d<D, D>(ws.Sf + (size_t)t * D * D);
        Mat<double, D, D> Sp;
        if (t > 0) {
            Mat<double, D, D> Sfm = ldcg_d<D, D>(ws.Sf + (size_t)(t - 1) * D * D);
            Mat<double, D, D> AS = mul(A, Sfm);
            Sp = sym_mul_nt_add(AS, A, P);
        } else {
            Sp = load_const<double, D, D>(mdl.S0);
            if (transition_first) { Mat<double, D, D> AS = mul(A, Sp); Sp = sym_mul_nt_add(AS, A, P); }
        }
        const bool obs_t = !tmask || tmask[t] != 0;
        {
            Mat<double, D, M> K;
            Mat<double, M, M> Li;
            double cconst = 0.0;
#pragma unroll
            for (int i = 0; i < D * M; ++i) K.a[i] = 0.0;
#pragma unroll
            for (int i = 0; i < M * M; ++i) Li.a[i] = 0.0;
            if (obs_t) {
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
        BwdEl<D> be;
        Vec<double, D> gb;
#pragma unroll
        for (int i = 0; i < D; ++i) gb(i) = 0.0;
        if (t < T - 1) {
            Mat<double, D, D> AS = mul(A, Sf);
            Mat<double, D, D> Sp1 = sym_mul_nt_add(AS, A, P);
            Chol<double, D> ch = cholesky<double, D, false>(Sp1, bad);
            Mat<double, D, D> U = solve_right_Lt(transpose(AS), ch.L);
            be.E = solve_right_L(U, ch.L);
            be.L = sym_downdate(Sf, U);
            Mat<double, D, D> Em = identity<double, D>();
            Mat<double, D, D> GA = mul(be.E, A);
#pragma unroll
            for (int i = 0; i < D * D; ++i) Em.a[i] -= GA.a[i];
            store_f(brec + TB::E_OFF, Em);
            store_f(brec + TB::G_OFF, be.E);
            Vec<double, D> uu;
#pragma unroll
            for (int i = 0; i < D; ++i) uu(i) = -(double)(useq ? useq[(size_t)(t + 1) * D + i] : mdl.u[i]);
            gb = mulv(be.E, uu);
        } else {
#pragma unroll
            for (int i = 0; i < D * D; ++i) be.E.a[i] = 0.0;
            be.L = Sf;
            store_f(brec + TB::E_OFF, identity<double, D>());
            store_f(brec + TB::G_OFF, be.E);
        }
        store_fv(brec + TB::GB_OFF, gb);
        bwd_store<D>(sw.bel, T, t, be);
    }
    cluster.sync();
    // ------------------------------------------------------------------ B1: local suffix products (r = T-1-t)
    {
        BwdEl<D> acc;
        acc.E = identity<double, D>();
#pragma unroll
        for (int i = 0; i < D * D; ++i) acc.L.a[i] = 0.0;
        for (int r = k0; r < k1; ++r) {
            const int t = T - 1 - r;
            const BwdEl<D> el = bwd_load<D>(sw.bel, T, t);
            acc = (r == k0) ? el : bwd_combine<D, false>(el, acc);
            if (E > 1) bwd_store<D>(sw.bel, T, t, acc);    // in place: element t is consumed
        }
        bwd_store<D>(sw.btot, GS_NT, g, acc);
    }
    cluster.sync();
    cur = 0;
    for (int off = 1; off < GS_NT; off <<= 1) {
        const double* src = sw.btot + (size_t)cur * GS_NT * BE;
        double* dst = sw.btot + (size_t)(cur ^ 1) * GS_NT * BE;
        BwdEl<D> mine = bwd_load<D>(src, GS_NT, g);
        if (g >= off && k0 < T) {
            BwdEl<D> prev = bwd_load<D>(src, GS_NT, g - off);    // later in time
            mine = bwd_combine<D, false>(mine, prev);
        }
        bwd_store<D>(dst, GS_NT, g, mine);
        cluster.sync();
        cur ^= 1;
    }
    {
        const double* tot = sw.btot + (size_t)cur * GS_NT * BE;
        BwdEl<D> excl;
        if (E > 1 && g > 0 && k0 < k1) excl = bwd_load<D>(tot, GS_NT, g - 1);
        for (int r = k0; r < k1; ++r) {
            const int t = T - 1 - r;
            Mat<double, D, D> Ss;
            if (E == 1) {
                Ss = ld_soa_d<D, D>(tot + (size_t)D * D * GS_NT, GS_NT, g);
            } else {
                const BwdEl<D> pr = bwd_load<D>(sw.bel, T, t);
                Ss = (g == 0) ? pr.L : bwd_combine<D, true>(pr, excl).L;
            }
            store_f(ws.bwd + (size_t)t * TB::BWD_REC + TB::SS_OFF, Ss);
            if (cov_shared_out) store_f(cov_shared_out + (size_t)t * D * D, Ss);
        }
    }
    if (bad) atomicOr(bad_out, 1);
}

}  // namespace rxg
