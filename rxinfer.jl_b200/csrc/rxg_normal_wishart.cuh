// The NormalMixture component with a Gaussian prior on its mean and a Wishart prior on its precision, shared by the
// Gaussian mixture (rxg_mixture.cu, DESIGN 3.17) and the Gaussian-emission HMM (rxg_hmm_gauss.cuh, DESIGN 3.20):
//     m_k ~ MvNormal(mu0, V0);  W_k ~ Wishart(nu0, S0);  q(m_k) q(W_k)
// Both kernels keep per component k, in this thread's shared memory with slot q at [q * ss], the fp64 statistics
// N_k = sum r, b_k = sum r (y - c_k), C_k = sum r (y - c_k)(y - c_k)' (lower) of their data pass (acc_slots) and the fp32
// constants that pass reads (st_slots): the centre c_k = E[m_k], E[W_k] (lower, off-diagonals doubled) and the offset
// 1/2 E log|W_k| - d/2 log 2 pi - 1/2 tr(E[W_k] V_k).  Everything here is fp64 on raw row-major arrays and __host__
// __device__, so that the HMM's body also compiles for the host (tests/c/hmm_gauss_host_harness.cu).
#pragma once
#include <math.h>
#include <stdint.h>

#include "rxg_hmm.cuh"          // RXG_HD, hmm::digamma
#include "rxg_internal.h"       // fail, host_spd_inv (pack, host only)

namespace rxg {
namespace nw {

constexpr double LOG2PI = 1.8378770664093453;
constexpr double LOGPI = 1.1447298858494002;
constexpr double LOG2 = 0.6931471805599453;
using hmm::digamma;

RXG_HD constexpr int packed(int d) { return d * (d + 1) / 2; }
RXG_HD constexpr int acc_slots(int d) { return 1 + d + packed(d); }      // N_k, b_k, C_k (lower), fp64
RXG_HD constexpr int st_slots(int d) { return d + packed(d) + 1; }       // c_k, E[W_k] (lower, doubled), offset, fp32

// The fp64 host constants of one component, blk doubles: mu0, inv(V0), inv(V0) mu0, log|V0|, inv(S0), log|S0|, nu0,
// log Gamma_d(nu0 / 2), m_init, Vm_init, nu_init, inv(S_init)
struct Layout {
    int mu0, V0i, xi0, ldV0, S0i, ldS0, nu0, lgd0, mi, Vi, nui, iSi, blk;
};
RXG_HD constexpr Layout layout(int d) {
    const int dd = d * d;
    return Layout{0, d, d + dd, 2 * d + dd, 2 * d + dd + 1, 2 * d + 2 * dd + 1, 2 * d + 2 * dd + 2, 2 * d + 2 * dd + 3,
                  2 * d + 2 * dd + 4, 3 * d + 2 * dd + 4, 3 * d + 3 * dd + 4, 3 * d + 3 * dd + 5, 3 * d + 4 * dd + 5};
}

// inv(A) and log|A| of a D x D SPD matrix from one Cholesky factorisation; false at a non-positive (or NaN) pivot.
// rxg_linalg.cuh's cholesky is device-only, so the d <= 4 factorisation is written here for both sides.
template <int D>
RXG_HD bool spd_inv(const double* A, double* Ai, double& logdet) {
    double L[D][D], Li[D][D], ri[D];                       // ri: the reciprocal pivots, one division per column
    logdet = 0.0;
#pragma unroll
    for (int j = 0; j < D; ++j) {
        double s = A[j * D + j];
#pragma unroll
        for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
        if (!(s > 0.0)) {
            for (int i = 0; i < D * D; ++i) Ai[i] = NAN;
            return false;
        }
        L[j][j] = sqrt(s);
        logdet += 2.0 * log(L[j][j]);
        ri[j] = 1.0 / L[j][j];
#pragma unroll
        for (int i = j + 1; i < D; ++i) {
            double t = A[i * D + j];
#pragma unroll
            for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k];
            L[i][j] = t * ri[j];
        }
    }
#pragma unroll
    for (int j = 0; j < D; ++j) {                          // L^-1 (lower), column by column
        Li[j][j] = ri[j];
#pragma unroll
        for (int i = j + 1; i < D; ++i) {
            double s = 0.0;
#pragma unroll
            for (int k = j; k < i; ++k) s += L[i][k] * Li[k][j];
            Li[i][j] = -s * ri[i];
        }
    }
#pragma unroll
    for (int i = 0; i < D; ++i)                            // L^-T L^-1
#pragma unroll
        for (int j = 0; j <= i; ++j) {
            double s = 0.0;
#pragma unroll
            for (int k = i; k < D; ++k) s += Li[k][i] * Li[k][j];
            Ai[i * D + j] = s;
            Ai[j * D + i] = s;
        }
    return true;
}

template <int D>
RXG_HD double lgamma_mv(double a) {                       // log Gamma_D(a)
    double s = 0.25 * D * (D - 1) * LOGPI;
    for (int i = 0; i < D; ++i) s += lgamma(a - 0.5 * i);
    return s;
}

// From q(m_k) = N(m, Vm) and q(W_k) = Wishart(nu, inv(iS)): the fp32 constants of the data pass into st and E[W_k] into
// EW; returns E[log|W_k|].  The mixture adds E[log s_k] to the offset once every alpha is known.
template <int D>
RXG_HD double derive(const double* m, const double* Vm, double nu, const double* iS, float* st, int ss, bool& bad,
                     double* EW) {
    double S[D * D], ldiS;
    if (!spd_inv<D>(iS, S, ldiS)) bad = true;
    double elog = D * LOG2 - ldiS;                                              // log|S| = -log|iS|
    for (int i = 0; i < D; ++i) elog += digamma(0.5 * (nu - i));
    double tr = 0.0;
#pragma unroll
    for (int i = 0; i < D * D; ++i) { EW[i] = nu * S[i]; tr += EW[i] * Vm[i]; }
#pragma unroll
    for (int i = 0; i < D; ++i) st[i * ss] = (float)m[i];
    int p = D;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j, ++p) st[p * ss] = (float)((i == j ? 1.0 : 2.0) * EW[i * D + j]);
    st[p * ss] = (float)(0.5 * elog - 0.5 * D * LOG2PI - 0.5 * tr);
    return elog;
}

// One component's updates, q(m_k) with the E[W_k] of the data pass, then q(W_k) with the new q(m_k), from its block pk,
// its statistics ak and its constants sk; sk is rewritten for the next pass.  E[W_k] and c_k are the fp32 constants the
// pass used: c_k exactly (the statistics are taken around it), E[W_k] rounded to fp32 (relative 6e-8, DESIGN 3.17).
// Hands back E[m_k] = m, Vm, nu and the inverse scale iS; returns KL(q(m_k)||p) + KL(q(W_k)||p) +
// N_k (d/2 log 2 pi - 1/2 E log|W_k|) + 1/2 tr(E[W_k] (R_k + N_k Vm)).  A non-positive pivot sets bad.
template <int D>
RXG_HD double update(const double* pk, const double* ak, float* sk, int ss, bool& bad, double* m, double* Vm, double& nu,
                     double* iS) {
    constexpr Layout LY = layout(D);
    const double Nk = ak[0];
    double c[D], bk[D], EW[D * D], Ck[D * D];
#pragma unroll
    for (int i = 0; i < D; ++i) { c[i] = (double)sk[i * ss]; bk[i] = ak[(1 + i) * ss]; }
    int p = D, pc = 1 + D;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j, ++p, ++pc) {
            const double w = (double)sk[p * ss] * (i == j ? 1.0 : 0.5);
            EW[i * D + j] = w; EW[j * D + i] = w;
            Ck[i * D + j] = ak[pc * ss]; Ck[j * D + i] = Ck[i * D + j];
        }
    // q(m_k): precision inv(V0) + N_k E[W_k], weighted mean inv(V0) mu0 + E[W_k] sum_i r_ik y_i
    double Lm[D * D], sy[D], xi[D], ldL;
#pragma unroll
    for (int i = 0; i < D * D; ++i) Lm[i] = pk[LY.V0i + i] + Nk * EW[i];
#pragma unroll
    for (int i = 0; i < D; ++i) sy[i] = bk[i] + Nk * c[i];
    if (!spd_inv<D>(Lm, Vm, ldL)) bad = true;                       // ldL = log|Lm| = -log|Vm|
#pragma unroll
    for (int i = 0; i < D; ++i) {
        double s = pk[LY.xi0 + i];
#pragma unroll
        for (int j = 0; j < D; ++j) s += EW[i * D + j] * sy[j];
        xi[i] = s;
    }
#pragma unroll
    for (int i = 0; i < D; ++i) {
        double s = 0.0;
#pragma unroll
        for (int j = 0; j < D; ++j) s += Vm[i * D + j] * xi[j];
        m[i] = s;
    }
    // q(W_k): nu0 + N_k, inverse scale inv(S0) + R_k + N_k Vm, R_k = sum_i r_ik (y_i - m)(y_i - m)' = C_k moved by
    // delta = m - c_k
    double dm[D], R[D * D];
#pragma unroll
    for (int i = 0; i < D; ++i) dm[i] = m[i] - c[i];
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) {
            R[i * D + j] = Ck[i * D + j] - bk[i] * dm[j] - dm[i] * bk[j] + Nk * dm[i] * dm[j];
            iS[i * D + j] = pk[LY.S0i + i * D + j] + R[i * D + j] + Nk * Vm[i * D + j];
        }
    nu = pk[LY.nu0] + Nk;
    double EWn[D * D];
    const double elog = derive<D>(m, Vm, nu, iS, sk, ss, bad, EWn);
    double trV = 0.0, quad = 0.0, trS = 0.0, trR = 0.0, e[D];
#pragma unroll
    for (int i = 0; i < D; ++i) e[i] = m[i] - pk[LY.mu0 + i];
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) {
            const double v0i = pk[LY.V0i + i * D + j];
            trV += v0i * Vm[j * D + i];
            quad += e[i] * v0i * e[j];
            trS += pk[LY.S0i + i * D + j] * EWn[j * D + i];             // nu tr(inv(S0) S)
            trR += EWn[i * D + j] * (R[j * D + i] + Nk * Vm[j * D + i]);
        }
    const double nu0 = pk[LY.nu0];
    double psum = 0.0;
    for (int i = 0; i < D; ++i) psum += digamma(0.5 * (nu - i));
    const double logdetS = elog - D * LOG2 - psum;                        // log|S| of the new q(W_k)
    const double kl_m = 0.5 * (trV + quad - D + pk[LY.ldV0] + ldL);
    const double kl_w = 0.5 * (nu - nu0) * elog - 0.5 * nu * D + 0.5 * trS - 0.5 * (nu - nu0) * D * LOG2
                        - 0.5 * nu * logdetS + 0.5 * nu0 * pk[LY.ldS0] - lgamma_mv<D>(0.5 * nu) + pk[LY.lgd0];
    return kl_m + kl_w + Nk * (0.5 * D * LOG2PI - 0.5 * elog) + 0.5 * trR;
}

// m, Vm, nu, iS as row r (k, or it * K + k) of the fp32 outputs [..][D][nb], [..][D][D][nb], [..][nb], [..][D][D][nb];
// a null output is skipped
template <int D>
RXG_HD void store(int64_t r, int64_t nb, int64_t b, const double* m, const double* Vm, double nu, const double* iS,
                  float* mean, float* cov, float* df, float* inv_scale) {
    if (df) df[r * nb + b] = (float)nu;
#pragma unroll
    for (int i = 0; i < D; ++i)
        if (mean) mean[(r * D + i) * nb + b] = (float)m[i];
#pragma unroll
    for (int i = 0; i < D * D; ++i) {
        if (cov) cov[(r * D * D + i) * nb + b] = (float)Vm[i];
        if (inv_scale) inv_scale[(r * D * D + i) * nb + b] = (float)iS[i];
    }
}

// Host: checks component k of the C entries' arrays (nu0, nu_init > d - 1; finite mu0, m_init; V0, S0, Vm_init, S_init
// SPD) and packs its block at pk, Vm_init symmetrised as host_spd_inv reads every host matrix.  RXG_OK, or RXG_ERR_BAD_ARG
// with a message naming the entry fn and k as "<what> k".
inline int pack(rxg_ctx* ctx, const char* fn, const char* what, int k, int d, const float* mu0, const float* V0,
                const float* nu0, const float* S0, const float* m_init, const float* Vm_init, const float* nu_init,
                const float* S_init, double* pk) {
    const Layout LY = layout(d);
    const int dd = d * d;
    if (!(nu0[k] > (float)(d - 1)) || !(nu_init[k] > (float)(d - 1)) || !isfinite(nu0[k]) || !isfinite(nu_init[k]))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: nu0 and nu_init must exceed d - 1 (%s %d)", fn, what, k);
    for (int i = 0; i < d; ++i)
        if (!isfinite(mu0[k * d + i]) || !isfinite(m_init[k * d + i]))
            return fail(ctx, RXG_ERR_BAD_ARG, "%s: mu0 and m_init must be finite (%s %d)", fn, what, k);
    double ld, tmp[16];
    if (!host_spd_inv(V0 + k * dd, d, pk + LY.V0i, &ld)) return fail(ctx, RXG_ERR_BAD_ARG, "%s: V0[%d] is not SPD", fn, k);
    pk[LY.ldV0] = ld;
    if (!host_spd_inv(S0 + k * dd, d, pk + LY.S0i, &ld)) return fail(ctx, RXG_ERR_BAD_ARG, "%s: S0[%d] is not SPD", fn, k);
    pk[LY.ldS0] = ld;
    if (!host_spd_inv(Vm_init + k * dd, d, tmp, &ld))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: Vm_init[%d] is not SPD", fn, k);
    for (int i = 0; i < d; ++i)
        for (int j = 0; j < d; ++j)
            pk[LY.Vi + i * d + j] = 0.5 * ((double)Vm_init[k * dd + i * d + j] + (double)Vm_init[k * dd + j * d + i]);
    if (!host_spd_inv(S_init + k * dd, d, pk + LY.iSi, &ld))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: S_init[%d] is not SPD", fn, k);
    for (int i = 0; i < d; ++i) {
        pk[LY.mu0 + i] = mu0[k * d + i];
        pk[LY.mi + i] = m_init[k * d + i];
        double s = 0.0;
        for (int j = 0; j < d; ++j) s += pk[LY.V0i + i * d + j] * (double)mu0[k * d + j];
        pk[LY.xi0 + i] = s;
    }
    pk[LY.nu0] = nu0[k];
    pk[LY.nui] = nu_init[k];
    double lgd = 0.25 * d * (d - 1) * LOGPI;
    for (int i = 0; i < d; ++i) lgd += lgamma(0.5 * ((double)nu0[k] - i));
    pk[LY.lgd0] = lgd;
    return RXG_OK;
}

}  // namespace nw
}  // namespace rxg
