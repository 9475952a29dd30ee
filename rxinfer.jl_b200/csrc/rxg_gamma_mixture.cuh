// Gamma mixture model, mean-field VMP with a point-mass shape, `batch` independent data sets in one launch
// (DESIGN 3.24; ref: test/models/mixtures/gamma_mixture_tests.jl:7-40).  Per data set of N positive scalars:
//     s ~ Dirichlet(alpha_s);  a[k] ~ Gamma(shape a_shape0[k], rate a_rate0[k]);  b[k] ~ Gamma(b_shape0[k], b_rate0[k])
//     z[i] ~ Categorical(s);   y[i] ~ GammaMixture(switch = z[i], a = a, b = b)   (component k: Gamma(shape a[k], rate b[k]))
//     q(z) q(a) q(b) q(s),  q(a[k]) = PointMass(a_hat[k])  (PointMassFormConstraint)
// With r_ik = q(z_i = k), N_k = sum_i r_ik, S_k = sum_i r_ik y_i, L_k = sum_i r_ik log y_i one iteration updates, in order,
//     a_hat_k = argmax_a (a_shape0 - 1) log a - a_rate0 a + a (N_k E[log b_k] + L_k) - N_k lgamma(a)   (Newton, fp64)
//     q(b_k)  = Gamma(b_shape0 + a_hat_k N_k, b_rate0 + S_k)
//     q(s)    = Dirichlet(alpha_s + N)
//     q(z_i)  propto exp(E[log s_k] + a_hat_k E[log b_k] - lgamma(a_hat_k) + (a_hat_k - 1) log y_i - E[b_k] y_i)
// the last as one pass over the data that also accumulates the next iteration's statistics.  The statistics before the
// first iteration are those of the uniform initial q(z).  After every iteration the free energy at the new marginals is
//     F = KL(q(s)||p(s)) + sum_k KL(q(b_k)||p(b_k)) - sum_k log p(a_hat_k)
//         - sum_k [N_k E[log s_k] + a_hat_k N_k E[log b_k] - N_k lgamma(a_hat_k) + (a_hat_k - 1) L_k - E[b_k] S_k]
//         - sum_i H[q(z_i)]
// (the point mass's entropy left out, its prior evaluated at the point).  q(s) is updated before the first data pass
// reads it, so the initial q(s) (alpha_init) does not enter; the initial q(b) enters the first shape update.  The data
// pass is fp32 per datum (log y on the fly, a max-shifted log-sum-exp over K per-component constants) with fp64
// accumulators; the updates, the Newton iteration and F are fp64.  A datum <= 0 or not finite flags its chain RXG_ERR_BAD_ARG and every output of the chain is
// NaN; a Newton iteration that has not converged (relative step <= NEWTON_RTOL) after NEWTON_CAP steps flags it
// RXG_ERR_NAN and keeps its last iterate.
// chain() is the whole per-chain body: the kernel (rxg_gamma_mixture.cu) runs it with one thread per data set, and
// tests/c/gamma_mixture_host_harness.cu compiles it for the host.
#pragma once
#include <math.h>
#include <stdint.h>

#include "rxg_hmm.cuh"   // RXG_HD, hmm::digamma

namespace rxg {
namespace gamix {

constexpr int MAX_K = 8;
constexpr int NEWTON_CAP = 100;
constexpr double NEWTON_RTOL = 1e-12;
constexpr int ST_BAD = 1, ST_NAN = 5;   // RXG_ERR_BAD_ARG, RXG_ERR_NAN

using hmm::digamma;

// fp64 host constants shared by every chain, each block [K]: a_shape0, a_rate0, b_shape0, b_rate0, alpha_s, alpha_init,
// b_shape_init, b_rate_init, a_start; then sum(alpha_s) and lgamma(sum alpha_s) - sum lgamma(alpha_s)
enum Block { A_SHAPE0, A_RATE0, B_SHAPE0, B_RATE0, ALPHA_S, ALPHA_INIT, B_SHAPE_INIT, B_RATE_INIT, A_START, N_BLOCKS };
RXG_HD int n_params(int K) { return N_BLOCKS * K + 2; }

// Per-chain fp64 state in scratch laid out [slot][chain] with stride ss (shared memory on the device): a_hat, q(b)
// shape and rate, q(s), N, S, L, and E[log s], E[log b] of the marginals the last data pass used
enum Slot { S_A, S_BSH, S_BRT, S_ALPHA, S_N, S_S, S_L, S_ELS, S_ELB, N_SLOTS };

struct Args {
    int K, N, iters;
    int64_t batch;
    const double* prm;
    const float* y;                     // [N][batch]
    float *alpha, *a_hat, *b_shape, *b_rate;   // [K][batch]
    double* fe;                         // [iters][batch] or NULL
    float* z_prob;                      // [N][K][batch] or NULL
    float *hist_a, *hist_b_shape, *hist_b_rate;   // [iters][K][batch] or NULL
};

// psi'(x), x > 0: recurrence up to x >= 10, then the asymptotic series to x^-15 (truncation below 1e-16 there)
RXG_HD double trigamma(double x) {
    double r = 0.0;
    while (x < 10.0) { r += 1.0 / (x * x); x += 1.0; }
    const double i = 1.0 / x, i2 = i * i;
    return r + i + 0.5 * i2 +
           i * i2 * (1.0 / 6 - i2 * (1.0 / 30 - i2 * (1.0 / 42 - i2 * (1.0 / 30 - i2 * (5.0 / 66 - i2 * (691.0 / 2730 -
                                                                                                   i2 * (7.0 / 6)))))));
}

// KL(Gamma(a1, b1) || Gamma(a0, b0)), shape / rate
RXG_HD double kl_gamma(double a1, double b1, double a0, double b0) {
    return (a1 - a0) * digamma(a1) - lgamma(a1) + lgamma(a0) + a0 * (log(b1) - log(b0)) + a1 * (b0 - b1) / b1;
}

// The point-mass update: the maximiser of f(a) = (ash - 1) log a - art a + a c - n lgamma(a), c = n E[log b] + L, by
// Newton's method from a0.  For ash >= 1 and n > 0, f' is decreasing and convex, so an iterate left of the maximiser
// stays left of it and increases towards it; an iterate that would leave a > 0 is replaced by half the current one.
// Returns false when the relative step is still above NEWTON_RTOL after NEWTON_CAP steps.
RXG_HD bool point_mass_shape(double ash, double art, double n, double c, double a0, double& a) {
    a = a0;
    for (int s = 0; s < NEWTON_CAP; ++s) {
        const double g = (ash - 1.0) / a - art + c - n * digamma(a);
        const double h = -(ash - 1.0) / (a * a) - n * trigamma(a);
        double an = a - g / h;
        if (!(an > 0.0)) an = 0.5 * a;
        const bool done = fabs(an - a) <= NEWTON_RTOL * an;
        a = an;
        if (done) return true;
    }
    return false;
}

// log Gamma(a | shape, rate)
RXG_HD double log_gamma_pdf(double a, double shape, double rate) {
    return shape * log(rate) - lgamma(shape) + (shape - 1.0) * log(a) - rate * a;
}

template <int K>
RXG_HD void fill_nan(int64_t b, const Args& a) {
    const float nf = NAN;
    const int64_t nb = a.batch;
    for (int k = 0; k < K; ++k) {
        a.alpha[k * nb + b] = a.a_hat[k * nb + b] = a.b_shape[k * nb + b] = a.b_rate[k * nb + b] = nf;
        for (int it = 0; it < a.iters; ++it) {
            const int64_t o = ((int64_t)it * K + k) * nb + b;
            if (a.hist_a) a.hist_a[o] = nf;
            if (a.hist_b_shape) a.hist_b_shape[o] = nf;
            if (a.hist_b_rate) a.hist_b_rate[o] = nf;
        }
    }
    if (a.fe)
        for (int it = 0; it < a.iters; ++it) a.fe[(int64_t)it * nb + b] = NAN;
    if (a.z_prob)
        for (int64_t j = 0; j < (int64_t)a.N * K; ++j) a.z_prob[j * nb + b] = nf;
}

// The chain's whole VMP: st is its fp64 scratch [N_SLOTS * K] with stride ss.  Returns its status.
template <int K>
RXG_HD int chain(int64_t b, const Args& a, double* st, int ss) {
    const double* p = a.prm;
    const int64_t nb = a.batch;
    auto S = [&](int slot, int k) -> double& { return st[(slot * K + k) * ss]; };

    // the statistics of the uniform initial q(z): N/K, sum y / K, sum log y / K (log y as the data pass forms it)
    double sy = 0.0, sly = 0.0;
    bool bad = false;
    for (int i = 0; i < a.N; ++i) {
        const float v = a.y[(int64_t)i * nb + b];
        if (!(v > 0.f) || !isfinite(v)) bad = true;
        sy += (double)v;
        sly += (double)logf(v);
    }
    if (bad) {
        fill_nan<K>(b, a);
        return ST_BAD;
    }
    for (int k = 0; k < K; ++k) {
        S(S_N, k) = (double)a.N / K;
        S(S_S, k) = sy / K;
        S(S_L, k) = sly / K;
        S(S_BSH, k) = p[B_SHAPE_INIT * K + k];
        S(S_BRT, k) = p[B_RATE_INIT * K + k];
    }
    int status = 0;
    for (int it = 0; it < a.iters; ++it) {
        const bool last = it == a.iters - 1;
        // ---- q(a_k), q(b_k) from the statistics and the previous q(b_k); q(s); the non-data terms of F
        double fe = 0.0, sa = p[N_BLOCKS * K];
        float c0[K], c1[K], eb[K];
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            const double n = S(S_N, k);
            double ah;
            if (!point_mass_shape(p[A_SHAPE0 * K + k], p[A_RATE0 * K + k], n,
                                  n * (digamma(S(S_BSH, k)) - log(S(S_BRT, k))) + S(S_L, k), p[A_START * K + k], ah))
                status = ST_NAN;
            const double bsh = p[B_SHAPE0 * K + k] + ah * n, brt = p[B_RATE0 * K + k] + S(S_S, k);
            S(S_A, k) = ah;
            S(S_BSH, k) = bsh;
            S(S_BRT, k) = brt;
            S(S_ELB, k) = digamma(bsh) - log(brt);
            S(S_ALPHA, k) = p[ALPHA_S * K + k] + n;
            sa += n;
            fe += kl_gamma(bsh, brt, p[B_SHAPE0 * K + k], p[B_RATE0 * K + k]) -
                  log_gamma_pdf(ah, p[A_SHAPE0 * K + k], p[A_RATE0 * K + k]);
            const int64_t o = ((int64_t)it * K + k) * nb + b;
            if (a.hist_a) a.hist_a[o] = (float)ah;
            if (a.hist_b_shape) a.hist_b_shape[o] = (float)bsh;
            if (a.hist_b_rate) a.hist_b_rate[o] = (float)brt;
            if (last) {
                a.a_hat[k * nb + b] = (float)ah;
                a.b_shape[k * nb + b] = (float)bsh;
                a.b_rate[k * nb + b] = (float)brt;
                a.alpha[k * nb + b] = (float)S(S_ALPHA, k);
            }
        }
        // KL(q(s) || p(s)) = log B(alpha_s) - log B(alpha) + sum_k (alpha_k - alpha_s_k) E[log s_k]
        const double psa = digamma(sa);
        fe += lgamma(sa) - p[N_BLOCKS * K + 1];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const double al = S(S_ALPHA, k), els = digamma(al) - psa;
            S(S_ELS, k) = els;
            fe += (al - p[ALPHA_S * K + k]) * els - lgamma(al);
            const double ah = S(S_A, k);
            c0[k] = (float)(els + ah * S(S_ELB, k) - lgamma(ah));
            c1[k] = (float)(ah - 1.0);
            eb[k] = (float)(S(S_BSH, k) / S(S_BRT, k));
        }
        // ---- q(z): one pass over the data, accumulating the next statistics and sum_i sum_k r_ik log r_ik
        double n_[K], s_[K], l_[K], h = 0.0;
#pragma unroll
        for (int k = 0; k < K; ++k) n_[k] = s_[k] = l_[k] = 0.0;
        for (int i = 0; i < a.N; ++i) {
            const float v = a.y[(int64_t)i * nb + b];
            const float lv = logf(v);
            float lr[K], mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                lr[k] = fmaf(c1[k], lv, fmaf(-eb[k], v, c0[k]));
                mx = fmaxf(mx, lr[k]);
            }
            float e[K], se = 0.f;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                lr[k] -= mx;
                e[k] = expf(lr[k]);
                se += e[k];
            }
            const float lse = logf(se), ise = 1.f / se;
            float hi = 0.f;
            const double vd = (double)v, lvd = (double)lv;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const float lrk = lr[k] - lse;
                const float r = e[k] * ise;
                if (last && a.z_prob) a.z_prob[((int64_t)i * K + k) * nb + b] = r;
                hi = fmaf(r, lrk, hi);
                const double rd = (double)r;
                n_[k] += rd;
                s_[k] = fma(rd, vd, s_[k]);
                l_[k] = fma(rd, lvd, l_[k]);
            }
            h += (double)hi;
        }
        // ---- the data terms of F at the new q(z) and the marginals it was formed from
        fe += h;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            S(S_N, k) = n_[k];
            S(S_S, k) = s_[k];
            S(S_L, k) = l_[k];
            const double ah = S(S_A, k);
            fe -= n_[k] * (S(S_ELS, k) + ah * S(S_ELB, k) - lgamma(ah)) + (ah - 1.0) * l_[k] -
                  S(S_BSH, k) / S(S_BRT, k) * s_[k];
        }
        if (a.fe) a.fe[(int64_t)it * nb + b] = fe;
    }
    return status;
}

}  // namespace gamix
}  // namespace rxg
