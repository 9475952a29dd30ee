// Bayesian binomial / logistic regression, mean-field Polya-Gamma VMP, `batch` independent chains in one launch
// (DESIGN 3.21; ref: test/models/regression/binomialreg_tests.jl:32-43).  Per chain:
//     beta ~ MvNormalWeightedMeanPrecision(xi0, W0);  y[i] ~ BinomialPolya(x[i], n[i], beta),  i = 1..N
// Each node sends beta the message MvNormalWeightedMeanPrecision((y_i - n_i/2) x_i, E[omega_i] x_i x_i'), so with
// q_k(beta) = N(m, S) an iteration is one pass over the chain's samples:
//     psi_i = x_i' m,  c_i = sqrt(psi_i^2 + x_i' S x_i),  E[omega_i] = n_i tanh(c_i / 2) / (2 c_i)
//     Lambda = W0 + sum_i E[omega_i] x_i x_i',  xi = xi0 + sum_i (y_i - n_i/2) x_i,  q_{k+1} = N(Lambda^-1 xi, Lambda^-1)
// and the free energy of a Gaussian q is the collapsed Polya-Gamma (Jaakkola-Jordan) bound
//     F(q) = KL(q || prior) - sum_i [log C(n_i, y_i) - n_i log 2 + (y_i - n_i/2) psi_i - n_i log cosh(c_i / 2)].
// The data term sum_i (y_i - n_i/2) x_i does not depend on q: it and sum_i log C(n_i, y_i) - n_i log 2 are accumulated in
// the first pass only, so F(q) = [KL(q) - xi_d' m] - lc + sum_i n_i log cosh(c_i / 2), the bracket taken when q is made
// and the last sum in the next pass, which computes c_i at q anyway.  With the free energy one closing pass follows the
// last iteration.  Lambda, xi and F accumulate in fp64; the per-sample arithmetic is fp32.
// A sample with n = 0 contributes nothing (ragged batches are padded so); a sample with a non-finite x, y < 0, n < 0 or
// y > n flags its chain RXG_ERR_BAD_ARG and is read as n = 0.
// Two kernels share sample() and end_pass(): one thread per chain (chain(), also compiled for the host by
// tests/c/binomial_host_harness.cu) and, for small batches, GROUP chains per CTA whose threads stride over the samples.
#pragma once
#include <math.h>
#include <stdint.h>

#include "rxg_normal_wishart.cuh"   // RXG_HD, nw::spd_inv, nw::packed

namespace rxg {
namespace polya {

constexpr int MAX_P = 8;
constexpr int ST_BAD = 1, ST_NOT_SPD = 4, ST_NAN = 5;        // RXG_ERR_BAD_ARG, RXG_ERR_NOT_SPD, RXG_ERR_NAN
constexpr double LOG2 = 0.6931471805599453;

// the chain-group path: GROUP consecutive chains per CTA (one 32-byte sector per feature and sample), SLOTS threads each
constexpr int GROUP = 8;
constexpr int GROUP_THREADS = 256;
constexpr int SLOTS = GROUP_THREADS / GROUP;
constexpr int PATH_AUTO = 0, PATH_THREAD = 1, PATH_GROUP = 2;   // RXG_OPT_POLYA_PATH
// The chain-group path runs while the batch is at most GROUP_CHAINS_PER_SM chains per SM (measured on the H100, DESIGN
// 3.21: chain groups are faster up to 16 384 chains, one thread per chain at 65 536) and a chain has at least one sample
// per slot.
constexpr int64_t GROUP_CHAINS_PER_SM = 128;
constexpr int GROUP_MIN_N = SLOTS;

RXG_HD int select_path(int64_t batch, int N, int p, int sm_count) {
    (void)p;
    return (batch <= GROUP_CHAINS_PER_SM * sm_count && N >= GROUP_MIN_N) ? PATH_GROUP : PATH_THREAD;
}

// fp64 host constants shared by every chain: the prior N(m0, S0) with S0 = inv(W0), m0 = S0 xi0, log|W0|, xi0' m0
struct Prior {
    double xi0[MAX_P], W0[MAX_P * MAX_P], m0[MAX_P], S0[MAX_P * MAX_P];
    double logdetW0, quad0;
};

struct Args {
    int N, iters;
    int64_t batch;
    const float* X;            // [N][p][batch]
    const int32_t* y;          // [N][batch]
    const int32_t* n;          // [N][batch], or NULL: every n = 1
    float* mean;               // [p][batch]
    float* cov;                // [p][p][batch] or NULL
    double* fe;                // [iters][batch] or NULL
    float *hist_mean, *hist_cov;   // [iters][p][batch], [iters][p][p][batch] or NULL
};

// One pass's sums over samples.  L (lower, packed row-major) and g = sum n log cosh(c/2) every pass; xi_d and lc =
// sum log C(n, y) - n log 2 in the first pass only.
template <int P>
struct Acc {
    double L[nw::packed(P)];
    double xi[P];
    double g, lc;
    bool bad;
};

template <int P>
RXG_HD void zero_pass(Acc<P>& a) {
#pragma unroll
    for (int q = 0; q < nw::packed(P); ++q) a.L[q] = 0.0;
    a.g = 0.0;
}

// q as the data pass reads it: m[P] and the lower triangle of S, packed (fp32)
template <int P>
struct Q {
    float m[P];
    float S[nw::packed(P)];
};

// One sample of one chain at q: its E[omega] x x' into L, its log cosh into g (want_g), and in the first pass its
// (y - n/2) x into xi and its log-binomial constant into lc (want_lc).
template <int P>
RXG_HD void sample(const float (&x)[P], int y, int n, const Q<P>& q, Acc<P>& a, bool first, bool want_lc, bool want_g) {
    bool ok = y >= 0 && n >= y;
#pragma unroll
    for (int j = 0; j < P; ++j) ok = ok && isfinite(x[j]);
    if (!ok) {
        a.bad = true;
        return;
    }
    if (n == 0) return;
    float psi = 0.f, s = 0.f, o[nw::packed(P)];
#pragma unroll
    for (int j = 0; j < P; ++j) {
        psi = fmaf(x[j], q.m[j], psi);
#pragma unroll
        for (int k = 0; k <= j; ++k) {
            const int t = j * (j + 1) / 2 + k;
            o[t] = x[j] * x[k];
            s = fmaf(k == j ? q.S[t] : 2.f * q.S[t], o[t], s);
        }
    }
    const float c2 = fmaxf(fmaf(psi, psi, s), 0.f), c = sqrtf(c2), nf = (float)n;
    const float w = c < 1e-3f ? nf * (0.25f - c2 * (1.f / 48.f)) : nf * tanhf(0.5f * c) / (2.f * c);
#pragma unroll
    for (int t = 0; t < nw::packed(P); ++t) a.L[t] += (double)(w * o[t]);
    if (want_g) a.g += (double)(nf * (0.5f * c + log1pf(expf(-c)) - (float)LOG2));   // n log cosh(c/2), c >= 0
    if (first) {
        const double r = (double)y - 0.5 * (double)n;
#pragma unroll
        for (int j = 0; j < P; ++j) a.xi[j] += r * (double)x[j];
        if (want_lc) {
            a.lc -= n * LOG2;
            if (n > 1) a.lc += lgamma(n + 1.0) - lgamma(y + 1.0) - lgamma(n - y + 1.0);
        }
    }
}

// q_{k+1} from the sums of pass k, into q and the outputs; fk = KL(q_{k+1} || prior) - xi_d' m_{k+1}.
template <int P>
RXG_HD void finish(int k, int64_t b, const Args& a, const Prior& pr, const Acc<P>& acc, Q<P>& q, double& fk, int& st) {
    double Lam[P * P], S[P * P], xi[P], m[P], ld;
#pragma unroll
    for (int j = 0; j < P; ++j) {
        xi[j] = pr.xi0[j] + acc.xi[j];
#pragma unroll
        for (int i = 0; i <= j; ++i) {
            const double v = acc.L[j * (j + 1) / 2 + i];
            Lam[j * P + i] = pr.W0[j * MAX_P + i] + v;
            Lam[i * P + j] = pr.W0[i * MAX_P + j] + v;
        }
    }
    if (!nw::spd_inv<P>(Lam, S, ld)) st = ST_NOT_SPD;
    double kl = ld - pr.logdetW0 - P + pr.quad0, lin = 0.0;   // 2 KL(q || prior), then - xi_d' m
#pragma unroll
    for (int j = 0; j < P; ++j) {
        double t = 0.0;
#pragma unroll
        for (int i = 0; i < P; ++i) t += S[j * P + i] * xi[i];
        m[j] = t;
    }
    bool finite = true;
#pragma unroll
    for (int j = 0; j < P; ++j) {
        double wm = 0.0;
#pragma unroll
        for (int i = 0; i < P; ++i) {
            kl += pr.W0[j * MAX_P + i] * S[i * P + j];
            wm += pr.W0[j * MAX_P + i] * m[i];
        }
        kl += m[j] * (wm - 2.0 * pr.xi0[j]);
        lin += acc.xi[j] * m[j];
        q.m[j] = (float)m[j];
        finite = finite && isfinite(m[j]);
#pragma unroll
        for (int i = 0; i <= j; ++i) {
            q.S[j * (j + 1) / 2 + i] = (float)S[j * P + i];
            finite = finite && isfinite(S[j * P + i]);
        }
    }
    fk = 0.5 * kl - lin;
    if (!finite && st != ST_NOT_SPD) st = ST_NAN;
    const int64_t B = a.batch;
    const bool last = k == a.iters - 1;
    float* hm = a.hist_mean ? a.hist_mean + (int64_t)k * P * B : nullptr;
    float* hc = a.hist_cov ? a.hist_cov + (int64_t)k * P * P * B : nullptr;
#pragma unroll
    for (int j = 0; j < P; ++j) {
        if (hm) hm[j * B + b] = q.m[j];
        if (last) a.mean[j * B + b] = q.m[j];
#pragma unroll
        for (int i = 0; i < P; ++i) {
            const float v = q.S[j >= i ? j * (j + 1) / 2 + i : i * (i + 1) / 2 + j];
            if (hc) hc[(j * P + i) * B + b] = v;
            if (last && a.cov) a.cov[(j * P + i) * B + b] = v;
        }
    }
}

template <int P>
RXG_HD void init_q(const Prior& pr, Q<P>& q) {
#pragma unroll
    for (int j = 0; j < P; ++j) {
        q.m[j] = (float)pr.m0[j];
#pragma unroll
        for (int i = 0; i <= j; ++i) q.S[j * (j + 1) / 2 + i] = (float)pr.S0[j * MAX_P + i];
    }
}

// After pass k's sums are complete: F(q_k) into fe[k - 1], then (k < iters) q_{k+1}.
template <int P>
RXG_HD void end_pass(int k, int64_t b, const Args& a, const Prior& pr, const Acc<P>& acc, Q<P>& q, double& fk, int& st) {
    if (k == 0 && acc.bad) st = ST_BAD;
    if (k >= 1 && a.fe) a.fe[(int64_t)(k - 1) * a.batch + b] = fk - acc.lc + acc.g;
    if (k < a.iters) finish<P>(k, b, a, pr, acc, q, fk, st);
}

RXG_HD int passes(const Args& a) { return a.iters + (a.fe ? 1 : 0); }

// sample i of chain b
template <int P>
RXG_HD void load(const Args& a, int i, int64_t b, float (&x)[P], int& y, int& n) {
    const int64_t B = a.batch;
#pragma unroll
    for (int j = 0; j < P; ++j) x[j] = a.X[((int64_t)i * P + j) * B + b];
    y = a.y[(int64_t)i * B + b];
    n = a.n ? a.n[(int64_t)i * B + b] : 1;
}

// The whole inference of chain b by one thread; returns its status.  The next sample is loaded before the current one
// is used.
template <int P>
RXG_HD int chain(int64_t b, const Args& a, const Prior& pr) {
    Q<P> q;
    init_q<P>(pr, q);
    Acc<P> acc;
#pragma unroll
    for (int j = 0; j < P; ++j) acc.xi[j] = 0.0;
    acc.lc = 0.0;
    acc.bad = false;
    double fk = 0.0;
    int st = 0;
    const int np = passes(a);
    for (int k = 0; k < np; ++k) {
        zero_pass<P>(acc);
        const bool first = k == 0, want_g = a.fe && k >= 1, want_lc = a.fe != nullptr;
        float x[P], xn[P];
        int y, n, yn = 0, nn = 0;
        load<P>(a, 0, b, x, y, n);
        for (int i = 0; i < a.N; ++i) {
            if (i + 1 < a.N) load<P>(a, i + 1, b, xn, yn, nn);
            sample<P>(x, y, n, q, acc, first, want_lc, want_g);
#pragma unroll
            for (int j = 0; j < P; ++j) x[j] = xn[j];
            y = yn;
            n = nn;
        }
        end_pass<P>(k, b, a, pr, acc, q, fk, st);
    }
    return st;
}

}  // namespace polya
}  // namespace rxg
