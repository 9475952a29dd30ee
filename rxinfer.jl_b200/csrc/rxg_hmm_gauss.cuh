// Hidden Markov model with Gaussian emissions, structured VMP  q(s_0, s) q(A) prod_k q(m_k) q(W_k)  fused into one kernel:
// one thread = one chain.
//
//     A ~ DirichletCollection(alpha_A0)  (K x K, column j = p(s_t | s_{t-1} = j)), or a known probability matrix
//     m[k] ~ MvNormal(mu0[k], V0[k]);  W[k] ~ Wishart(nu0[k], S0[k])  (precision)
//     s_0 ~ Categorical(p0);  s[t] ~ DiscreteTransition(s[t-1], A);  y[t] ~ NormalMixture(switch = s[t], m, W)
// The chain of rxg_hmm.cuh with the symbol emission replaced by the NormalMixture(:switch) message of the mixture
// (rxg_mixture.cu), per state k:
//     l_k(y) = 1/2 E log|W_k| - d/2 log 2 pi - 1/2 [(y - E m_k)' E[W_k] (y - E m_k) + tr(E[W_k] V_k)],
// evaluated in fp32 from per-state constants (centre c_k = E[m_k], packed E[W_k] with doubled off-diagonals, offset) and
// shifted by its maximum over k at each step, so that the sweep's weights exp(l_k - max) never underflow all at once.
// Per iteration (DESIGN 3.20):
//   forward:  alpha_t = e_t * (A~ alpha_{t-1}) / c_t, e_tk = exp(l_k(y_t) - max_k l_k(y_t)); alpha_t goes to the stash
//             [T][K][batch] (the s_prob output); sum_t log c_t in fp64;
//   backward: as rxg_hmm.cuh (the transition counts in fp32 registers flushed into fp64), the emission weights recomputed
//             from y; the Gaussian statistics N_k = sum gamma, b_k = sum gamma (y - c_k), C_k = sum gamma (y - c_k)(y - c_k)'
//             around the centre the sweep used, and S = sum_t sum_k gamma_tk (l_k(y_t) - max), all fp64;
//   updates:  q(A) = Dirichlet(alpha_A0 + sum xi) (rxg_hmm.cuh); q(m_k) with the sweep's E[W_k]; q(W_k) with the new
//             q(m_k) (the component of rxg_mixture.cu, rxg_normal_wishart.cuh);
//   free energy, fp64: F = -sum_t log c_t + S + [A terms of rxg_hmm.cuh] + sum_k [KL(q(m_k)||p) + KL(q(W_k)||p) +
//             N_k (d/2 log 2 pi - 1/2 E_new log|W_k|) + 1/2 tr(E_new[W_k] (R_k + N_k V_k))].  -sum log c_t + S is
//             -log Z~ + sum gamma l_used with the per-step shifts cancelled exactly (they are never added), so the fp32
//             rounding of the weights the sweep ran with cancels too.
// A step whose d components are all NaN is missing (a pure transition).  Any other non-finite datum flags the chain
// RXG_ERR_BAD_ARG and its step is read as missing; a normaliser c_t that is zero or not finite flags RXG_ERR_NAN; a
// non-positive Cholesky pivot in an update flags RXG_ERR_NOT_SPD.  Other chains are never touched.
#pragma once
#include <math.h>
#include <stdint.h>

#include "rxg_hmm.cuh"              // RXG_HD, hmm::FLUSH, hmm::a_tilde, hmm::a_terms
#include "rxg_normal_wishart.cuh"

namespace rxg {
namespace hmmg {

using namespace nw;                                        // the component: layout, derive, update, store
constexpr int ST_BAD_ARG = 1, ST_NOT_SPD = 4, ST_NAN = 5;    // RXG_ERR_BAD_ARG, RXG_ERR_NOT_SPD, RXG_ERR_NAN

// Where the fp32 transition partials live: registers up to K = 4; from K = 5 on, K x K fp32 shared-memory slots after the
// sweep constants, since in registers they spill at K >= 5 for d >= 3 and K >= 6 for d = 2 (DESIGN 3.20)
RXG_HD constexpr bool u_shared(int /*d*/, int K) { return K >= 5; }
RXG_HD constexpr int f_slots(int d, int K) { return K * st_slots(d) + (u_shared(d, K) ? K * K : 0); }

// fp64 host constants: p0[K], A (prior alpha or known matrix) [K][K], A_init [K][K], then one nw::Layout block per state
RXG_HD int off_states(int K) { return K + 2 * K * K; }
RXG_HD int n_params(int K, int d) { return off_states(K) + K * layout(d).blk; }

struct Args {
    int T, iters;
    int64_t batch;
    int learn_A;
    const double* prm;
    const float* y;                          // [T][d][batch]
    float* s_prob;                           // [T][K][batch]: the forward stash, gamma of the last iteration at the end
    float* s0_prob;                          // [K][batch]
    float* A_alpha;                          // [K][K][batch]
    float *m_mean, *m_cov, *w_df, *w_inv_scale;   // [K][d][batch], [K][d][d][batch], [K][batch], [K][d][d][batch]
    double* fe;                              // [iters][batch]
    float *hist_s, *hist_A, *hist_m_mean, *hist_m_cov, *hist_w_df, *hist_w_inv_scale;
};

// y_t of chain b into v; false for a missing step (all d components NaN, or any non-finite one, which also flags the chain)
template <int D>
RXG_HD bool read_step(const float* y, int t, int64_t b, int64_t nb, float* v, int& status) {
    int nan = 0;
    bool finite = true;
#pragma unroll
    for (int i = 0; i < D; ++i) {
        v[i] = y[((int64_t)t * D + i) * nb + b];
        nan += isnan(v[i]) ? 1 : 0;
        finite = finite && isfinite(v[i]);
    }
    if (finite) return true;
    if (nan != D) status = ST_BAD_ARG;
    return false;
}

// l_k(v) of every state from the constants st (fp32, explicit fma so that the forward and backward passes compute the
// same bits); returns max_k l_k
template <int D, int K>
RXG_HD float log_weights(const float* st, int ss, const float* v, float* lr) {
    constexpr int SS = st_slots(D);
    float mx = -3.402823466e38f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float* sk = st + k * SS * ss;
        float dl[D];
#pragma unroll
        for (int i = 0; i < D; ++i) dl[i] = v[i] - sk[i * ss];
        float q = 0.f;
        int p = D;
#pragma unroll
        for (int i = 0; i < D; ++i) {
            float row = 0.f;
#pragma unroll
            for (int j = 0; j <= i; ++j, ++p) row = fmaf(sk[p * ss], dl[j], row);
            q = fmaf(row, dl[i], q);
        }
        lr[k] = fmaf(-0.5f, q, sk[(SS - 1) * ss]);
        mx = fmaxf(mx, lr[k]);
    }
    return mx;
}

// One chain.  fsh / dsh: this thread's shared memory, slot q at [q * ss]; fsh holds the sweep constants [K][st_slots]
// (fp32), dsh the transition counts [K][K] then the Gaussian statistics [K][acc_slots] (fp64).  Returns the status code.
template <int D, int K>
RXG_HD int chain(int64_t b, const Args& a, float* fsh, double* dsh, int ss) {
    constexpr int SA = acc_slots(D), SS = st_slots(D);
    constexpr Layout LY = layout(D);
    const int T = a.T;
    const int64_t nb = a.batch;
    const double* prm = a.prm;
    const double* pA = prm + K;
    const double* ps = prm + off_states(K);
    double* xi64 = dsh;                    // [K][K]
    double* acc = dsh + K * K * ss;        // [K][SA]
    int status = 0;
    bool bad = false;
    float At[K][K];
    float p0[K];
#pragma unroll
    for (int i = 0; i < K; ++i) p0[i] = (float)prm[i];
#pragma unroll 1
    for (int k = 0; k < K; ++k) {          // the initial q(m), q(W) -> constants of the first sweep
        const double* pk = ps + k * LY.blk;
        double EW[D * D];
        derive<D>(pk + LY.mi, pk + LY.Vi, pk[LY.nui], pk + LY.iSi, fsh + k * SS * ss, ss, bad, EW);
    }
    if (bad) status = ST_NOT_SPD;          // the first cause is kept; BAD_ARG (a bad datum) overrides every other

    for (int it = 0; it < a.iters; ++it) {
        const bool last = it == a.iters - 1;
        // ---- A~ from q(A): the initial marginal, then prior + counts of the previous sweep; a known A is reloaded every
        // iteration so that it holds no registers through the parameter updates
        if (!a.learn_A) {
#pragma unroll
            for (int i = 0; i < K; ++i)
#pragma unroll
                for (int j = 0; j < K; ++j) At[i][j] = (float)pA[i * K + j];
        } else {
            hmm::a_tilde<K>(a, it, xi64, ss, At);
        }
        for (int q = 0; q < K * K; ++q) xi64[q * ss] = 0.0;
        for (int q = 0; q < K * SA; ++q) acc[q * ss] = 0.0;

        // ---- forward
        double logc = 0.0;                 // sum_t log c_t (log Z~ without the shifts)
        float al[K];
#pragma unroll
        for (int i = 0; i < K; ++i) al[i] = p0[i];
        for (int t = 0; t < T; ++t) {
            float v[D], lr[K];
            const bool obs = read_step<D>(a.y, t, b, nb, v, status);
            const float mx = obs ? log_weights<D, K>(fsh, ss, v, lr) : 0.f;
            float nx[K], c = 0.f;
#pragma unroll
            for (int i = 0; i < K; ++i) {
                float s = 0.f;
#pragma unroll
                for (int j = 0; j < K; ++j) s = fmaf(At[i][j], al[j], s);
                nx[i] = obs ? s * expf(lr[i] - mx) : s;
                c += nx[i];
            }
            if (!(c > 0.f) || !(c <= 3.402823466e38f)) { if (!status) status = ST_NAN; }
            const float rc = 1.f / c;
            logc += (double)logf(c);
#pragma unroll
            for (int i = 0; i < K; ++i) {
                al[i] = nx[i] * rc;
                a.s_prob[((int64_t)t * K + i) * nb + b] = al[i];
            }
        }

        // ---- backward: al holds alpha_t, beta_t in registers, alpha_{t-1} from the stash (p0 at t = 1)
        double Sl = 0.0;                   // sum_t sum_k gamma_tk (l_k(y_t) - max), the weights the sweep ran with
        float be[K];
        constexpr bool USH = u_shared(D, K);
        float ureg[USH ? 1 : K][USH ? 1 : K];
        float* ush = fsh + K * SS * ss;
        auto u = [&](int i, int j) -> float& {
            if constexpr (USH) return ush[(i * K + j) * ss];
            else return ureg[i][j];
        };
#pragma unroll
        for (int i = 0; i < K; ++i) {
            be[i] = 1.f;
#pragma unroll
            for (int j = 0; j < K; ++j) u(i, j) = 0.f;
        }
        float* hs = a.hist_s ? a.hist_s + (int64_t)it * T * K * nb : nullptr;
        for (int t = T - 1; t >= 0; --t) {
            float v[D], lr[K];
            int ignored = 0;               // flagged in the forward pass already
            const bool obs = read_step<D>(a.y, t, b, nb, v, ignored);
            const float mx = obs ? log_weights<D, K>(fsh, ss, v, lr) : 0.f;
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
                    const float li = lr[i] - mx;
                    w[i] = be[i] * expf(li);
                    const double gd = (double)g;
                    Sl += gd * (double)li;
                    double* ak = acc + i * SA * ss;
                    const float* sk = fsh + i * SS * ss;
                    ak[0] += gd;
                    int p = 1 + D;
#pragma unroll
                    for (int r = 0; r < D; ++r) {
                        const double dr = (double)(v[r] - sk[r * ss]);
                        const double gr = gd * dr;
                        ak[(1 + r) * ss] += gr;
#pragma unroll
                        for (int c = 0; c <= r; ++c, ++p) ak[p * ss] = fma(gr, (double)(v[c] - sk[c * ss]), ak[p * ss]);
                    }
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
                for (int j = 0; j < K; ++j) u(i, j) = fmaf(ap[j], wi, u(i, j));
            }
#pragma unroll
            for (int j = 0; j < K; ++j) { be[j] = bp[j] * rz; al[j] = ap[j]; }
            if (t % hmm::FLUSH == 0) {                                        // fp32 partial sums of <= FLUSH steps
#pragma unroll
                for (int i = 0; i < K; ++i)
#pragma unroll
                    for (int j = 0; j < K; ++j) {
                        xi64[(i * K + j) * ss] += (double)At[i][j] * (double)u(i, j);
                        u(i, j) = 0.f;
                    }
            }
        }
        if (last && a.s0_prob) {
#pragma unroll
            for (int j = 0; j < K; ++j) a.s0_prob[(int64_t)j * nb + b] = p0[j] * be[j];
        }

        // ---- q(A) and its free-energy terms; q(m_k) with the sweep's E[W_k], q(W_k) with the new q(m_k), and theirs
        double F = Sl - logc;
        if (a.learn_A) hmm::a_terms<K>(a, it, last, b, xi64, ss, At, F);
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            double m[D], Vm[D * D], nu, iS[D * D];
            F += update<D>(ps + k * LY.blk, acc + k * SA * ss, fsh + k * SS * ss, ss, bad, m, Vm, nu, iS);
            store<D>((int64_t)it * K + k, nb, b, m, Vm, nu, iS, a.hist_m_mean, a.hist_m_cov, a.hist_w_df, a.hist_w_inv_scale);
            if (last) store<D>(k, nb, b, m, Vm, nu, iS, a.m_mean, a.m_cov, a.w_df, a.w_inv_scale);
        }
        if (bad && !status) status = ST_NOT_SPD;
        if (a.fe) a.fe[(int64_t)it * nb + b] = F;
    }
    return status;
}

}  // namespace hmmg
}  // namespace rxg
