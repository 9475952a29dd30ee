// Hidden Markov model, structured VMP  q(s, s_0) q(A) q(B)  fused into one kernel: one thread = one chain.
//
//     A ~ DirichletCollection(alpha_A0)  (K x K, column j = p(s_t | s_{t-1} = j));  B likewise (M x K, p(x_t | s_t = j))
//     s_0 ~ Categorical(p0);  s[t] ~ DiscreteTransition(s[t-1], A);  x[t] ~ DiscreteTransition(s[t], B)
// [ref: test/models/statespace/hmm_tests.jl:8-30 (model, constraints, initialisation); either matrix may instead be a known
//  probability matrix, as when A is passed as data in test/inference/inference_tests.jl:2062-2088].
//
// Given q(A), q(B) the chain is exact: a scaled forward-backward sweep with A~ = exp(E[log A]), B~ = exp(E[log B]) (or the
// known matrix itself), in probability space, so exact zeros of a known matrix need no -inf.  Per iteration:
//   forward:  alpha_t = B~[x_t] * (A~ alpha_{t-1}) / c_t, alpha_0 = p0; log Z~ = sum log c_t in fp64; alpha_t goes to the
//             stash [T][K][batch] (the s_prob output);
//   backward: beta_T = 1; w = B~[x_t] * beta_t, beta'_{t-1} = A~' w, Z_t = alpha_{t-1} . beta'_{t-1} (= c_t), beta_{t-1} =
//             beta'_{t-1} / Z_t, so gamma_t = alpha_t * beta_t sums to one; the transition counts
//             sum_t xi_t[i][j] = A~[i][j] sum_t alpha_{t-1}[j] w[i] / Z_t (the outer products in fp32 registers, flushed
//             into fp64 every FLUSH steps) and the emission counts n_B[x_t][i] += gamma_t[i] (fp64, shared memory);
//             gamma_t overwrites the stash in the last iteration (every iteration into hist_s with KeepEach);
//   updates:  alpha_A = alpha_A0 + sum xi, alpha_B = alpha_B0 + n_B (a known matrix is not updated);
//   Bethe free energy in fp64 from the statistics alone (DESIGN 3.18):
//     F = KL(q(A)||p(A)) + KL(q(B)||p(B)) - log Z~ + sum xi (log A~_used - E_new[log A]) + sum n_B (log B~_used - E_new[log B])
//   with A~_used the fp32 matrix the sweep ran with; the terms of a known matrix are omitted (not computed as 0 * -inf).
// Missing steps (x = 255) are pure transitions.  A symbol >= M that is not 255 flags the chain RXG_ERR_BAD_ARG and is
// treated as missing (it never indexes B~); a normaliser c_t that is zero or not finite flags it RXG_ERR_NAN.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef RXG_HD
#define RXG_HD __host__ __device__ __forceinline__
#endif

namespace rxg {
namespace hmm {

constexpr int MAX_M = 16;
constexpr int FLUSH = 32;                 // steps between flushes of the fp32 transition counts into fp64
constexpr uint8_t MISSING = 255;
constexpr int ST_BAD_SYMBOL = 1, ST_NAN = 5;   // RXG_ERR_BAD_ARG, RXG_ERR_NAN

// fp64 host constants: p0[K], then A (prior alpha or known matrix) [K][K], A_init [K][K], B [M][K], B_init [M][K]
RXG_HD int off_A(int K) { return K; }
RXG_HD int off_Ai(int K) { return K + K * K; }
RXG_HD int off_B(int K) { return K + 2 * K * K; }
RXG_HD int off_Bi(int K, int M) { return K + 2 * K * K + M * K; }
RXG_HD int n_params(int K, int M) { return K + 2 * K * K + 2 * M * K; }

struct Args {
    int T, M, iters;
    int64_t batch;
    int learn_A, learn_B;
    const double* prm;
    const uint8_t* x;          // [T][batch]
    float* s_prob;             // [T][K][batch]: the forward stash, gamma of the last iteration at the end
    float* s0_prob;            // [K][batch]
    float *A_alpha, *B_alpha;  // [K][K][batch], [M][K][batch]
    double* fe;                // [iters][batch]
    float *hist_s, *hist_A, *hist_B;
};

// psi(x), x > 0: recurrence up to x >= 10, then the asymptotic series; NaN for x <= 0 or NaN (a flagged chain)
RXG_HD double digamma(double x) {
    if (!(x > 0.0)) return NAN;
    if (isinf(x)) return x;
    double r = 0.0;
    while (x < 10.0) { r -= 1.0 / x; x += 1.0; }
    const double i = 1.0 / x, i2 = i * i;
    return r + log(x) - 0.5 * i - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252 - i2 * (1.0 / 240 - i2 * (1.0 / 132)))));
}

// E[log P[i][j]] = psi(a(i, j)) - psi(sum_i a(i, j)) of column j of a DirichletCollection with R rows, handed to out(i, .)
template <typename F, typename O>
RXG_HD void elog_column(F a, int R, int j, O out) {
    double s = 0.0;
    for (int i = 0; i < R; ++i) s += a(i, j);
    const double ps = digamma(s);
    for (int i = 0; i < R; ++i) out(i, digamma(a(i, j)) - ps);
}

// The free-energy terms of a learned matrix without those of the counts n against the used matrix: with alpha = alpha0 + n,
// KL(q||p) carries sum n E_new[log P], which cancels the -sum n E_new[log P] of the difference term; what is left is
// sum_j [log B(alpha0_j) - log B(alpha_j)], log B(a) = sum_i lgamma(a_i) - lgamma(sum_i a_i).  The caller adds
// sum n log P~used (P~used = exp(E_used[log P]), the fp32 matrix the sweep ran with).
template <typename N>
RXG_HD double log_beta_terms(const double* a0, N n, int R, int C) {
    double f = 0.0;
    for (int j = 0; j < C; ++j) {
        double sa = 0.0, sa0 = 0.0;
        for (int i = 0; i < R; ++i) {
            const double a0i = a0[i * C + j], ai = a0i + n(i, j);
            sa += ai; sa0 += a0i;
            f += lgamma(a0i) - lgamma(ai);
        }
        f += lgamma(sa) - lgamma(sa0);
    }
    return f;
}

// q(A) of the chains here and in rxg_hmm_gauss.cuh, whose Args both carry prm (p0 [K], alpha_A0 [K][K], A_init [K][K] at
// its head), batch, hist_A and A_alpha; xi: the fp64 transition counts [K][K], slot q at xi[q * ss].
// A~ = exp(E[log A]) into At, alpha = A_init in the first iteration, else alpha_A0 + the counts of the previous sweep;
// xi is the scratch (it holds E[log A] on return)
template <int K, typename ArgsT>
RXG_HD void a_tilde(const ArgsT& a, int it, double* xi, int ss, float (&At)[K][K]) {
    const double *pA = a.prm + off_A(K), *ai = a.prm + off_Ai(K);
    for (int q = 0; q < K * K; ++q) xi[q * ss] = it == 0 ? ai[q] : pA[q] + xi[q * ss];   // alpha, in place
    for (int j = 0; j < K; ++j)
        elog_column([&](int r, int c) { return xi[(r * K + c) * ss]; }, K, j,
                    [&](int r, double e) { xi[(r * K + j) * ss] = e; });
#pragma unroll
    for (int i = 0; i < K; ++i)
#pragma unroll
        for (int j = 0; j < K; ++j) At[i][j] = (float)exp(xi[(i * K + j) * ss]);
}

// The free-energy terms of q(A) after the sweep that ran with At and counted xi, added to F; alpha_A0 + xi into hist_A
// (every iteration) and A_alpha (the last)
template <int K, typename ArgsT>
RXG_HD void a_terms(const ArgsT& a, int it, bool last, int64_t b, const double* xi, int ss, const float (&At)[K][K],
                    double& F) {
    const double* pA = a.prm + off_A(K);
    F += log_beta_terms(pA, [&](int r, int c) { return xi[(r * K + c) * ss]; }, K, K);
#pragma unroll
    for (int i = 0; i < K; ++i)
#pragma unroll
        for (int j = 0; j < K; ++j) {                // At > 0 wherever the count is (it is proportional to At)
            const double n = xi[(i * K + j) * ss];
            if (n > 0.0) F += n * log((double)At[i][j]);
        }
    for (int q = 0; q < K * K; ++q) {
        const float v = (float)(pA[q] + xi[q * ss]);
        if (a.hist_A) a.hist_A[((int64_t)it * K * K + q) * a.batch + b] = v;
        if (last && a.A_alpha) a.A_alpha[(int64_t)q * a.batch + b] = v;
    }
}

// One chain.  fsh / dsh: this thread's shared memory, slot q at [q * ss]; fsh holds B~ [M][K] (fp32), dsh the transition
// counts [K][K] then the emission counts [M][K] (fp64).  Returns the status code (0, ST_BAD_SYMBOL or ST_NAN).
template <int K>
RXG_HD int chain(int64_t b, const Args& a, float* fsh, double* dsh, int ss) {
    const int T = a.T, M = a.M;
    const int64_t nb = a.batch;
    const double* prm = a.prm;
    const double* pA = prm + off_A(K);
    const double* pB = prm + off_B(K);
    double* xi64 = dsh;                    // [K][K]
    double* nB64 = dsh + K * K * ss;       // [M][K]
    int status = 0;
    float At[K][K];
    float p0[K];
#pragma unroll
    for (int i = 0; i < K; ++i) p0[i] = (float)prm[i];
    if (!a.learn_A) {
#pragma unroll
        for (int i = 0; i < K; ++i)
#pragma unroll
            for (int j = 0; j < K; ++j) At[i][j] = (float)pA[i * K + j];
    }
    if (!a.learn_B)
        for (int q = 0; q < M * K; ++q) fsh[q * ss] = (float)pB[q];

    for (int it = 0; it < a.iters; ++it) {
        const bool last = it == a.iters - 1;
        // ---- A~, B~ from q(A), q(B): the initial marginals, then prior + counts of the previous sweep
        if (a.learn_A) a_tilde<K>(a, it, xi64, ss, At);
        if (a.learn_B) {
            const double* bi = prm + off_Bi(K, M);
            for (int q = 0; q < M * K; ++q) nB64[q * ss] = it == 0 ? bi[q] : pB[q] + nB64[q * ss];
            for (int j = 0; j < K; ++j)
                elog_column([&](int r, int c) { return nB64[(r * K + c) * ss]; }, M, j,
                            [&](int r, double e) { fsh[(r * K + j) * ss] = (float)exp(e); });
        }
        for (int q = 0; q < K * K; ++q) xi64[q * ss] = 0.0;
        for (int q = 0; q < M * K; ++q) nB64[q * ss] = 0.0;

        // ---- forward
        double logZ = 0.0;
        float al[K];
#pragma unroll
        for (int i = 0; i < K; ++i) al[i] = p0[i];
        for (int t = 0; t < T; ++t) {
            const int xt = a.x[(int64_t)t * nb + b];
            const bool obs = xt < M;
            if (!obs && xt != MISSING) status = ST_BAD_SYMBOL;
            float nx[K], c = 0.f;
#pragma unroll
            for (int i = 0; i < K; ++i) {
                float s = 0.f;
#pragma unroll
                for (int j = 0; j < K; ++j) s = fmaf(At[i][j], al[j], s);
                nx[i] = obs ? s * fsh[(xt * K + i) * ss] : s;
                c += nx[i];
            }
            if (!(c > 0.f) || !(c <= 3.402823466e38f)) { if (!status) status = ST_NAN; }
            const float rc = 1.f / c;
            logZ += (double)logf(c);
#pragma unroll
            for (int i = 0; i < K; ++i) {
                al[i] = nx[i] * rc;
                a.s_prob[((int64_t)t * K + i) * nb + b] = al[i];
            }
        }

        // ---- backward: al holds alpha_t, beta_t in registers, alpha_{t-1} from the stash (p0 at t = 1)
        float be[K], u[K][K];
#pragma unroll
        for (int i = 0; i < K; ++i) {
            be[i] = 1.f;
#pragma unroll
            for (int j = 0; j < K; ++j) u[i][j] = 0.f;
        }
        float* hs = a.hist_s ? a.hist_s + (int64_t)it * T * K * nb : nullptr;
        for (int t = T - 1; t >= 0; --t) {
            const int xt = a.x[(int64_t)t * nb + b];
            const bool obs = xt < M;
            float ap[K];
#pragma unroll
            for (int j = 0; j < K; ++j) ap[j] = t > 0 ? a.s_prob[((int64_t)(t - 1) * K + j) * nb + b] : p0[j];
            float w[K];
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const float g = al[i] * be[i];                               // gamma_t
                if (last) a.s_prob[((int64_t)t * K + i) * nb + b] = g;
                if (hs) hs[((int64_t)t * K + i) * nb + b] = g;
                if (obs) {
                    nB64[(xt * K + i) * ss] += (double)g;
                    w[i] = be[i] * fsh[(xt * K + i) * ss];
                } else {
                    w[i] = be[i];
                }
            }
            float bp[K], Z = 0.f;
#pragma unroll
            for (int j = 0; j < K; ++j) {
                float s = 0.f;
#pragma unroll
                for (int i = 0; i < K; ++i) s = fmaf(At[i][j], w[i], s);
                bp[j] = s;
                Z = fmaf(ap[j], s, Z);
            }
            const float rz = 1.f / Z;
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const float wi = w[i] * rz;
#pragma unroll
                for (int j = 0; j < K; ++j) u[i][j] = fmaf(ap[j], wi, u[i][j]);
            }
#pragma unroll
            for (int j = 0; j < K; ++j) { be[j] = bp[j] * rz; al[j] = ap[j]; }
            if (t % FLUSH == 0) {                                             // fp32 partial sums of <= FLUSH steps
#pragma unroll
                for (int i = 0; i < K; ++i)
#pragma unroll
                    for (int j = 0; j < K; ++j) {
                        xi64[(i * K + j) * ss] += (double)At[i][j] * (double)u[i][j];
                        u[i][j] = 0.f;
                    }
            }
        }
        if (last && a.s0_prob) {
#pragma unroll
            for (int j = 0; j < K; ++j) a.s0_prob[(int64_t)j * nb + b] = p0[j] * be[j];
        }

        // ---- conjugate updates (alpha = alpha0 + counts, kept as counts in shared memory) and the free energy
        double F = -logZ;
        if (a.learn_A) a_terms<K>(a, it, last, b, xi64, ss, At, F);
        if (a.learn_B) {
            F += log_beta_terms(pB, [&](int r, int c) { return nB64[(r * K + c) * ss]; }, M, K);
            for (int q = 0; q < M * K; ++q) {
                const double n = nB64[q * ss];
                if (n > 0.0) F += n * log((double)fsh[q * ss]);
            }
            for (int q = 0; q < M * K; ++q) {
                const float v = (float)(pB[q] + nB64[q * ss]);
                if (a.hist_B) a.hist_B[((int64_t)it * M * K + q) * nb + b] = v;
                if (last && a.B_alpha) a.B_alpha[(int64_t)q * nb + b] = v;
            }
        }
        if (a.fe) a.fe[(int64_t)it * nb + b] = F;
    }
    return status;
}

}  // namespace hmm
}  // namespace rxg
