// Bayesian multinomial regression, mean-field Polya-Gamma VMP for the MultinomialPolya node, `batch` independent chains in
// one launch (DESIGN 3.22; ref: test/models/regression/multinomialreg_tests.jl).  Per chain, with D = K - 1:
//     psi ~ MvNormalWeightedMeanPrecision(xi0, W0);  y[i] ~ MultinomialPolya(N_i, psi),  y_i in N^K, N_i = sum_k y_ik
// read through stick-breaking as y_ik ~ Binomial(N_ik, sigmoid(psi_k)), k = 1..D, N_ik = sum_{j >= k} y_ij.  Node i sends
// psi MvNormalWeightedMeanPrecision(b_i, diag(N_ik g(c_k))), b_ik = y_ik - N_ik / 2, g(c) = tanh(c/2) / (2c), with
// c_k = sqrt(m_k^2 + S_kk) at the current q = N(m, S).  One step, "base N(m0, S0) (x) a diagonal-precision message
// (b, n) -> q", serves both entries:
//     d_k = n_k g(c_k);  S = (S0^-1 + diag d)^-1 as D Sherman-Morrison updates of S0 (d_k = 0 skipped);
//     m = m0 + S (b - d o m0)
// and its byproducts give KL(q || base) in O(D): log|Lam| / |Lam0| = sum_k log pivot_k, tr(Lam0 S) = D - sum_k d_k S_kk,
// (m - m0)' Lam0 (m - m0) = (m - m0)' (b - d o m).  The free energy is the collapsed Jaakkola-Jordan bound
//     F(q) = KL(q || base) - [lc + b'm - sum_k n_k log cosh(c_k / 2)],  c at q,
// lc = the log multinomial coefficient - sum_k n_k log 2.  A whole data set enters through its per-category totals only
// (base = the prior); online, datum t's base is q_{t-1}.  All state is fp64.
// The functions work on the columns j = lane, lane + nl, ... of fp64 arrays (row-major, symmetric S): the kernels call
// them with (lane, 32) on one warp per chain, tests/c/multinomial_host_harness.cu with (0, 1).
// A negative count flags the chain RXG_ERR_BAD_ARG and its sample is read as all-zero; an all-zero sample contributes
// nothing (ragged batches are padded so).
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef RXG_HD
#define RXG_HD __host__ __device__ __forceinline__
#endif

namespace rxg {
namespace mnp {

constexpr int MAX_K = 64, MAX_D = MAX_K - 1;
constexpr int ST_BAD = 1, ST_NOT_SPD = 4, ST_NAN = 5;        // RXG_ERR_BAD_ARG, RXG_ERR_NOT_SPD, RXG_ERR_NAN
constexpr double LOG2 = 0.6931471805599453;
constexpr int LF_N = 1024;                                   // the table of log k! covers k < LF_N

RXG_HD void sync_lanes() {
#ifdef __CUDA_ARCH__
    __syncwarp();
#endif
}

// the sum over the lanes, the same bits on every lane (each butterfly step adds a + b on one lane, b + a on the other)
RXG_HD double lane_sum(double v) {
#ifdef __CUDA_ARCH__
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
    return v;
}

// NOT_SPD over NAN over BAD_ARG
RXG_HD void flag(int& st, int code) {
    const auto rank = [](int s) { return s == ST_NOT_SPD ? 3 : s == ST_NAN ? 2 : s == ST_BAD ? 1 : 0; };
    if (rank(code) > rank(st)) st = code;
}

// E[omega] / n of PG(n, c): tanh(c/2) / (2c), and 1/4 - c^2/48 below c = 1e-3
RXG_HD double pg_mean(double c) { return c < 1e-3 ? 0.25 - c * c * (1.0 / 48.0) : tanh(0.5 * c) / (2.0 * c); }
// log cosh(c/2), c >= 0
RXG_HD double log_cosh_half(double c) { return 0.5 * c + log1p(exp(-c)) - LOG2; }
RXG_HD double log_fact(long long k, const double* lf) { return k < LF_N ? lf[k] : lgamma((double)k + 1.0); }

// One chain's fp64 arrays: q = N(m, S) and the step's scratch
struct Work {
    double* S;            // [D][D]
    double* m;            // [D]
    double *d, *u, *r;    // [D]: message precisions, the Sherman-Morrison row, b - d o m0
};

// One step: the message at the current q (cm, cS; may be w's own arrays), then q = base (m0, S0) (x) message into w.
// Returns F(q) relative to the base; a non-positive pivot or S_kk flags NOT_SPD, a non-finite result NAN.
RXG_HD double step(int lane, int nl, int D, const double* m0, const double* S0, const double* b, const double* n,
                   double lc, const double* cm, const double* cS, const Work& w, int& st) {
    for (int k = lane; k < D; k += nl) w.d[k] = n[k] * pg_mean(sqrt(fmax(fma(cm[k], cm[k], cS[k * D + k]), 0.0)));
    sync_lanes();
    for (int j = lane; j < D; j += nl)
        for (int i = 0; i < D; ++i) w.S[i * D + j] = S0[i * D + j];
    sync_lanes();
    double logdet = 0.0;
    bool spd = true;
    for (int k = 0; k < D; ++k) {
        const double dk = w.d[k];
        if (dk == 0.0) continue;
        for (int j = lane; j < D; j += nl) w.u[j] = w.S[k * D + j];
        sync_lanes();
        const double skk = w.u[k], piv = fma(dk, skk, 1.0), a = dk / piv;
        spd = spd && skk > 0.0 && piv > 0.0;
        for (int j = lane; j < D; j += nl) {
            const double uj = w.u[j];
            for (int i = 0; i < D; ++i) w.S[i * D + j] = fma(-a, w.u[i] * uj, w.S[i * D + j]);   // u_i u_j: symmetric
        }
        logdet += log(piv);
        sync_lanes();
    }
    for (int k = lane; k < D; k += nl) w.r[k] = b[k] - w.d[k] * m0[k];
    sync_lanes();
    double tr = 0.0, quad = 0.0, bm = 0.0, g = 0.0, nonfinite = 0.0;
    for (int j = lane; j < D; j += nl) {
        double t = 0.0;
        for (int i = 0; i < D; ++i) t = fma(w.S[i * D + j], w.r[i], t);
        const double mj = m0[j] + t, sjj = w.S[j * D + j], dj = w.d[j];
        w.m[j] = mj;
        tr += dj * sjj;
        quad += t * (b[j] - dj * mj);
        bm += b[j] * mj;
        g += n[j] * log_cosh_half(sqrt(fmax(fma(mj, mj, sjj), 0.0)));
        if (!isfinite(mj) || !isfinite(sjj)) nonfinite = 1.0;
    }
    tr = lane_sum(tr);
    quad = lane_sum(quad);
    bm = lane_sum(bm);
    g = lane_sum(g);
    nonfinite = lane_sum(nonfinite);
    sync_lanes();
    const double F = 0.5 * (quad - tr + logdet) - lc - bm + g;
    if (!spd) flag(st, ST_NOT_SPD);
    else if (nonfinite != 0.0 || !isfinite(F)) flag(st, ST_NAN);
    return F;
}

// q into fp32 outputs (NULL = not wanted): mean[D][B], cov[D][D][B], chain c
RXG_HD void store(int lane, int nl, int D, const Work& w, int64_t B, int64_t c, float* mean, float* cov) {
    for (int j = lane; j < D; j += nl) {
        if (mean) mean[j * B + c] = (float)w.m[j];
        if (cov)
            for (int i = 0; i < D; ++i) cov[((int64_t)i * D + j) * B + c] = (float)w.S[i * D + j];
    }
}

// ------------------------------------------------------------------------------------ whole data sets
// One sample's counts y[K] into the running totals Y[K] and sum log N! - sum_k log y_k!; false (nothing added) when a
// count is negative.
template <int KB>
RXG_HD bool add_sample(int K, const int32_t (&y)[KB], const double* lf, double (&Y)[KB], double& lcoef) {
    bool ok = true;
    long long N = 0;
#pragma unroll
    for (int k = 0; k < KB; ++k)
        if (k < K) {
            ok = ok && y[k] >= 0;
            N += y[k];
        }
    if (!ok) return false;
    double s = log_fact(N, lf);
#pragma unroll
    for (int k = 0; k < KB; ++k)
        if (k < K) {
            Y[k] += (double)y[k];
            s -= log_fact(y[k], lf);
        }
    lcoef += s;
    return true;
}

// The whole data set's message from the totals, in place: Y[k] becomes S_k = sum_{j >= k} Y_j, so that n_k = S_k and
// b_k = (S_k - S_{k+1}) - S_k / 2, k < D; returns lc = lcoef - log 2 sum_{k < D} S_k.
template <int KB>
RXG_HD double suffix_totals(int K, double (&Y)[KB], double lcoef) {
    double S = 0.0, sn = 0.0;
#pragma unroll
    for (int k = KB - 1; k >= 0; --k)
        if (k < K) {
            S += Y[k];
            Y[k] = S;
            if (k < K - 1) sn += S;
        }
    return lcoef - LOG2 * sn;
}

// Every iteration of one chain: q_{k+1} = prior (x) the message at q_k, from q_0 = the prior.  Outputs (NULL = not
// wanted): fe[iters][B], hist_mean[iters][D][B], hist_cov[iters][D][D][B], and the last q into mean / cov.
struct Out {
    int64_t batch;
    float *mean, *cov, *hist_mean, *hist_cov;
    double* fe;
};

RXG_HD void offline(int lane, int nl, int D, int iters, const double* m0, const double* S0, const double* b,
                    const double* n, double lc, const Work& w, const Out& o, int64_t c, int& st) {
    const int64_t B = o.batch;
    const double *cm = m0, *cS = S0;
    for (int k = 0; k < iters; ++k) {
        const double F = step(lane, nl, D, m0, S0, b, n, lc, cm, cS, w, st);
        cm = w.m;
        cS = w.S;
        if (o.fe && lane == 0) o.fe[(int64_t)k * B + c] = F;
        store(lane, nl, D, w, B, c, o.hist_mean ? o.hist_mean + (int64_t)k * D * B : nullptr,
              o.hist_cov ? o.hist_cov + (int64_t)k * D * D * B : nullptr);
        if (k == iters - 1) store(lane, nl, D, w, B, c, o.mean, o.cov);
    }
}

// ------------------------------------------------------------------------------------ online
// Datum y[K] (cnt, shared by the lanes) into its message: n_k = N_tk, b_k = y_k - n_k / 2, k < D; returns lc.  A negative
// count sets bad and the datum is read as all-zero.
RXG_HD double datum(int lane, int nl, int K, const int32_t* cnt, const double* lf, double* b, double* n, bool& bad) {
    const int D = K - 1;
    bool ok = true;
    long long N = 0, sn = 0;
    double lcoef = 0.0;
    for (int k = 0; k < K; ++k) {
        const int32_t v = cnt[k];
        ok = ok && v >= 0;
        N += v;
        sn += (long long)v * (k < D ? k + 1 : D);          // sum_k n_k = sum_j y_j (min(j, D - 1) + 1)
        if (v >= 0) lcoef -= log_fact(v, lf);
    }
    for (int k = lane; k < D; k += nl) {
        long long s = 0;
        for (int j = k; j < K; ++j) s += cnt[j];
        n[k] = ok ? (double)s : 0.0;
        b[k] = ok ? (double)cnt[k] - 0.5 * (double)s : 0.0;
    }
    sync_lanes();
    if (!ok) {
        bad = true;
        return 0.0;
    }
    return lcoef + log_fact(N, lf) - LOG2 * (double)sn;
}

// Data t = 0..T-1 of chain c (y[T][K][B]): each runs iters steps from the base q_{t-1}, and q_t becomes the next base.
// `base` holds the carry on entry and q_{T-1} on return; the outputs hold per datum ([T][D][B], [T][D][D][B], fe[T][B]).
// PER = the counts each lane holds, ceil(K / nl) at most: the next datum is loaded while the current one is processed.
template <int PER>
RXG_HD void online(int lane, int nl, int K, int T, int iters, const int32_t* y, int64_t c, const double* lf, Work& base,
                   Work& w, int32_t* cnt, double* b, double* n, const Out& o, int& st) {
    const int D = K - 1;
    const int64_t B = o.batch;
    int32_t cur[PER];
#pragma unroll
    for (int q = 0; q < PER; ++q) {
        const int k = lane + q * nl;
        cur[q] = k < K ? y[(int64_t)k * B + c] : 0;
    }
    bool bad = false;
    for (int t = 0; t < T; ++t) {
#pragma unroll
        for (int q = 0; q < PER; ++q)
            if (lane + q * nl < K) cnt[lane + q * nl] = cur[q];
        sync_lanes();
        if (t + 1 < T)
#pragma unroll
            for (int q = 0; q < PER; ++q) {
                const int k = lane + q * nl;
                if (k < K) cur[q] = y[((int64_t)(t + 1) * K + k) * B + c];
            }
        const double lc = datum(lane, nl, K, cnt, lf, b, n, bad);
        const double *cm = base.m, *cS = base.S;
        double F = 0.0;
        for (int it = 0; it < iters; ++it) {
            F = step(lane, nl, D, base.m, base.S, b, n, lc, cm, cS, w, st);
            cm = w.m;
            cS = w.S;
        }
        if (o.fe && lane == 0) o.fe[(int64_t)t * B + c] = F;
        store(lane, nl, D, w, B, c, o.hist_mean ? o.hist_mean + (int64_t)t * D * B : nullptr,
              o.hist_cov ? o.hist_cov + (int64_t)t * D * D * B : nullptr);
        const Work q = base;
        base = w;
        w = q;
    }
    if (bad) flag(st, ST_BAD);
}

}  // namespace mnp
}  // namespace rxg
