// Per-chain Kalman / RTS step bodies (one thread = one chain, (mu, Sigma) in registers), shared by
// lgssm_chain_kernel (rxg_lgssm.cu) and the Wishart-precision VMP kernel (rxg_lgssm_vmp.cu).
#pragma once
#include "rxg_lgssm_common.cuh"
#include "rxg_linalg.cuh"

namespace rxg {

// load_u of a transition without per-step inputs (the constant offset u stays as loaded)
struct NoInput {
    template <int D>
    __device__ __forceinline__ void operator()(Vec<float, D>&) const {}
};

// rule #1  *(:out): (A mu, A S A')   rule #2  MvNormalMeanCovariance(:out): + P
// (+ the `+` rule with a PointMass operand: pure mean shift by u; load_u(u) refreshes a per-step input first)
template <int D, typename LoadU>
__device__ __forceinline__ void chain_predict(const Mat<float, D, D>& A, const Mat<float, D, D>& P, Vec<float, D>& u,
                                              LoadU load_u, Vec<float, D>& mu, Mat<float, D, D>& S) {
    mu = mulv(A, mu);
    load_u(u);
#pragma unroll
    for (int i = 0; i < D; ++i) mu(i) += u(i);
    Mat<float, D, D> AS = mul(A, S);
    S = sym_mul_nt_add(AS, A, P);
}

// rules #3,#4 (observation message) folded with the product at x_t, gain form:
//   Sinn = B S B' + Q = L L',  V = S B' L^-T,  mu += V L^-1 (y - B mu),  S -= V V'
// want_nle: acc_nle += 1/2 (z'z + log det Sinn + M log 2 pi), the step's negative log-evidence increment.
template <int D, int M>
__device__ __forceinline__ void chain_update(const Mat<float, M, D>& B, const Mat<float, M, M>& Q, const Vec<float, M>& yt,
                                             bool want_nle, Vec<float, D>& mu, Mat<float, D, D>& S, bool& bad,
                                             double& acc_nle) {
    Mat<float, M, D> BS = mul(B, S);
    Mat<float, M, M> Sinn = sym_mul_nt_add(BS, B, Q);
    Chol<float, M> ch = want_nle ? cholesky<float, M, true>(Sinn, bad)
                                 : cholesky<float, M, false>(Sinn, bad);
    Mat<float, D, M> V = solve_right_Lt(transpose(BS), ch.L);
    Vec<float, M> e = mulv(B, mu);
#pragma unroll
    for (int k = 0; k < M; ++k) e(k) = yt(k) - e(k);
    Vec<float, M> z = solve_L(ch.L, e);
    Vec<float, D> dm = mulv(V, z);
#pragma unroll
    for (int i = 0; i < D; ++i) mu(i) += dm(i);
    S = sym_downdate(S, V);
    if (want_nle) {
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < M; ++k) q = __fmaf_rn(z(k), z(k), q);
        acc_nle += (double)(0.5f * q - ch.neg_half_logdet) + M * RXG_HALF_LOG_2PI;
    }
}

// absorb the factor exp(-1/2 x' L L' x) into (mu, S), covariance form (nothing singular is inverted):
//   Sm = I + L' S L = Ls Ls',  Z = S L Ls^-T,  S -= Z Z',  mu -= Z Ls^-1 L' mu
// want_nle: acc_nle += 1/2 (|Ls^-1 L' mu|^2 + log det Sm), the factor's negative log-normaliser under N(mu, S).
template <int D>
__device__ __forceinline__ void chain_tilt(const Mat<float, D, D>& L, bool want_nle, Vec<float, D>& mu,
                                           Mat<float, D, D>& S, bool& bad, double& acc_nle) {
    Mat<float, D, D> SL = mul(S, L);
    Mat<float, D, D> Sm = sym_mul_nt_add(transpose(SL), transpose(L), identity<float, D>());
    Chol<float, D> ch = want_nle ? cholesky<float, D, true>(Sm, bad) : cholesky<float, D, false>(Sm, bad);
    Mat<float, D, D> Z = solve_right_Lt(SL, ch.L);
    Vec<float, D> z = solve_L(ch.L, mulv_t(L, mu));
    Vec<float, D> dm = mulv(Z, z);
#pragma unroll
    for (int i = 0; i < D; ++i) mu(i) -= dm(i);
    S = sym_downdate(S, Z);
    if (want_nle) {
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < D; ++k) q = __fmaf_rn(z(k), z(k), q);
        acc_nle += (double)(0.5f * q - ch.neg_half_logdet);
    }
}

// pair hook of an RTS step without lag-one statistics
struct NoPair {
    template <int D>
    __device__ __forceinline__ void operator()(const Mat<float, D, D>&, const Mat<float, D, D>&,
                                               const Mat<float, D, D>&) const {}
};

// one RTS step: filtered (muf, Sf) at t and smoothed (mus, Ss) at t+1 -> smoothed at t (in place).
// Sp = A Sf A' + P (the forward message into x_{t+1}); RTS gain G = Sf A' Sp^-1; load_u(u) refreshes the input of the
// transition into x_{t+1}.  pair(G, C, Ss) sees the gain, C = cov(x_t | x_{t+1}, y_{1:t}) and the smoothed covariance at
// t+1 before Ss is overwritten (the lag-one statistics of the pairwise marginal).
template <int D, typename LoadU, typename Pair = NoPair>
__device__ __forceinline__ void chain_rts(const Mat<float, D, D>& A, const Mat<float, D, D>& P, Vec<float, D>& u,
                                          LoadU load_u, const Vec<float, D>& muf, const Mat<float, D, D>& Sf,
                                          Vec<float, D>& mus, Mat<float, D, D>& Ss, bool& bad, Pair pair = Pair{}) {
    Mat<float, D, D> AS = mul(A, Sf);
    Mat<float, D, D> Sp = sym_mul_nt_add(AS, A, P);
    Chol<float, D> ch = cholesky<float, D, false>(Sp, bad);
    Mat<float, D, D> U = solve_right_Lt(transpose(AS), ch.L);   // Sf A' L^-T
    Mat<float, D, D> G = solve_right_L(U, ch.L);
    Mat<float, D, D> C = sym_downdate(Sf, U);                   // cov(x_t | x_{t+1})
    pair(G, C, Ss);
    Mat<float, D, D> GS = mul(G, Ss);
    Ss = sym_mul_nt_add(GS, G, C);
    Vec<float, D> mup = mulv(A, muf);
    load_u(u);
#pragma unroll
    for (int i = 0; i < D; ++i) mup(i) = mus(i) - (mup(i) + u(i));
    Vec<float, D> dm = mulv(G, mup);
#pragma unroll
    for (int i = 0; i < D; ++i) mus(i) = muf(i) + dm(i);
}

}  // namespace rxg
