// Variational message passing around the per-chain smoother with unknown noise precision MATRICES, one per chain: the
// multivariate twin of vmp_gamma_kernel (rxg_hgf.cu).
//
//   w_p ~ Wishart(nu_p0, inv(Psi_p0)) (else P known);  w_q ~ Wishart(nu_q0, inv(Psi_q0)) (else Q known);
//   x[1] ~ N(m0, S0) (or one transition earlier, RXG_TRANSITION_FIRST);
//   x[t] ~ N(A x[t-1] + u, inv(w_p));    y[t] ~ N(B x[t], inv(w_q));    q(x) q(w_p) q(w_q)
// [ref: docs/src/manuals/model-specification.md:265-271, constraints q(x, w) = q(x)q(w)].  LEARN says which precisions
// are learned: LEARN_Q (rxg_lgssm_vmp_wishart_f32), LEARN_P or both (rxg_lgssm_vmp_noise_f32).
//
// One iteration k, per chain:
//   q(x)  exact Kalman filter + RTS smoother with P = inv(Wbar_p), Q = inv(Wbar_q), Wbar = E[w] under q_{k-1}(w) (init_E_W
//         at k = 0; a known noise keeps its matrix): the average energy of a Gaussian node under q(w) is N(. | ., inv(E[w]))
//         up to constants.
//   q(w_q) = prior x prod_t MvNormalMeanPrecision(:Lambda)(q_out = PointMass(y_t), q_mu = N(B mu_t, B Sigma_t B')), i.e.
//         df = nu_q0 + N_q, Psi = Psi_q0 + R_q, R_q = sum_{observed t} (y_t - B mu_t)(y_t - B mu_t)' + B Sigma_t B'.
//   q(w_p) = prior x prod_t MvNormalMeanPrecision(:Lambda)(q(out, mu) = pairwise marginal of (x_{t+1}, A x_t + u)), i.e.
//         df = nu_p0 + N_p (N_p = T - 1 + tf transitions, masks do not change it), Psi = Psi_p0 + R_p,
//         R_p = sum_t e e' + cov(x_{t+1} - A x_t | y), e = mu_{t+1} - A mu_t - u.  With the RTS gain G_t and
//         C_t = cov(x_t | x_{t+1}, y_{1:t}), x_t = G_t x_{t+1} + eps (cov C_t, independent of x_{t+1}) given all the data, so
//         cov(x_{t+1} - A x_t | y) = (I - A G_t) Sigma_{t+1} (I - A G_t)' + A C_t A': two PSD terms, no cancellation in fp32.
//   F_k   = NLE(Wbar_p, Wbar_q) + per learned noise [N/2 (log det Wbar - E log det w) + 1/2 tr((E w - Wbar) R)
//         + KL(q_k(w) || prior)]   (fp64), q(x) the exact chain posterior under (Wbar_p, Wbar_q) (its Gaussian part
//         collapses to the filter's evidence).
// One thread = one chain, all iterations in one launch; every array is [..][batch] (coalesced).  post_mean / post_cov are
// the forward->backward stash of every iteration; only the last iteration writes the smoothed q(x) over it.  The Kalman and
// RTS step bodies are lgssm_chain_kernel's (rxg_chain_step.cuh).
//
//
// LEARN_A (rxg_lgssm_vmp_transition_f32, d <= 4) also learns the transition matrix per chain, RxInfer's
// ContinuousTransition node with a linear reshape: a = vec(A) (row-major r = i d + j) ~ N(ma0, Va0), q(x) q(a) q(w_p) q(w_q).
// With Abar = E[A] and Xi = E[(A - Abar)' Wbar_p (A - Abar)], Xi[j][k] = sum_{i,l} Wbar_p[i][l] cov(a_ij, a_lk):
//   q(x)  the chain under (Abar, Wbar_p, Wbar_q) with one more factor exp(-1/2 x' Xi x) on the source state of every
//         transition (chain_tilt after the update, so the stash holds the tilted filtered states and the RTS pass and its
//         pair identity are unchanged).  Xi = L L' in fp64 once per iteration.
//   q(a)  Lambda = Va0^-1 + Wbar_p (x) Sxx, E[a] += Lambda^-1 (Va0^-1 (ma0 - E[a]) + vec(Wbar_p Sxr')), cov(a) =
//         Lambda^-1, with Sxx = sum E[x_t x_t'] and Sxr = sum E[x_t r_t'], r_t = x_{t+1} - Abar x_t - u, over the source
//         states (fp64 sums; cov(x_t, r_t) = G Ss (I - Abar G)' - C Abar' from the pair hook).
//   q(w_p) with the new q(a): R_p = R_p(Abar_old) + D Sxx D' - D Sxr - Sxr' D' + K, D = Abar_new - Abar_old,
//         K[i][l] = sum_{j,k} cov(a_ij, a_lk) Sxx[j][k]; no cancellation of large second moments.
//   F     gains 1/2 tr(Wbar_p (R_p,new - R_p,old)) (the transition energy under the new q(a)) + KL(q(a) || prior).
// The d^2 x d^2 algebra runs in fp64 in per-thread local memory, once per iteration, off the time loops.
//
// This translation unit is compiled once per observation dimension m (-DRXG_VMP_M=m: d = 1..6 of that m, three LEARN
// each, and d = 1..4 of the four LEARN_A values) and once without it for the C entries below.  m is compiled exactly:
// padding y would add dummy coordinates to w_q and change the answer.
#include <math.h>

#include <type_traits>

#include "rxg_chain_step.cuh"
#include "rxg_internal.h"

namespace rxg {

enum : int { LEARN_Q = 1, LEARN_P = 2, LEARN_PQ = 3, LEARN_A = 4 };

struct VmpWishHost {        // host-side model of one call (fp64 where the kernel works in fp64)
    const float *A, *B, *P, *Q, *m0, *S0, *u;    // P / Q: the known matrix, or null when it is learned
    double nu0, logdet_Psi0;                     // observation precision prior
    double Psi0[36], W0[36];   // [m][m], symmetrised
    double nu_p0, logdet_Psi_p0;                 // process precision prior
    double Psi_p0[36], Wp0[36];  // [d][d], symmetrised
    // LEARN_A: prior mean, inverse prior covariance and log det of the prior covariance of a = vec(A); initial q(a)
    double ma0[16], Va0i[256], logdet_Va0, ma_init[16], Sa_init[256];
};
struct VmpWishIO {
    const float* y;
    const uint8_t* ymask;      // [T][batch] or null
    const uint8_t* tmask;      // [T] (shared pattern, device copy) or null
    float *mean, *cov, *df, *inv_scale;
    double* fe;
    int32_t* status;
    int T, iterations, tf;
    int64_t batch;
};
struct VmpNoiseIO : VmpWishIO {
    float *df_p, *inv_scale_p;
};
struct VmpTransIO : VmpNoiseIO {
    float *a_mean, *a_cov;     // [iterations][d][d][batch], [iterations][d*d][d*d][batch]
};
template <int LEARN>
using VmpIO = std::conditional_t<(LEARN & LEARN_A) != 0, VmpTransIO,
                                 std::conditional_t<LEARN == LEARN_Q, VmpWishIO, VmpNoiseIO>>;

template <int K>
struct WishPrior {
    double nu0, logdet_Psi0, Psi0[K * K], W0[K * K];
};
template <int D, int M>
struct VmpWishModel {
    float A[D * D], B[M * D], P[D * D], m0[D], S0[D * D], u[D];
    WishPrior<M> q;
};
template <int D, int M>
struct VmpNoiseModel : VmpWishModel<D, M> {
    float Q[M * M];
    WishPrior<D> p;
};
// LEARN_A: 4.3 KB of fp64 prior and initial q(a) at d = 4, over the classic 4 KB parameter block (CUDA >= 12.1 passes
// up to 32 KB as __grid_constant__ parameters).  The inherited A is unused.
template <int D, int M>
struct VmpTransModel : VmpNoiseModel<D, M> {
    double ma0[D * D], Va0i[D * D * D * D], logdet_Va0, ma_init[D * D], Sa_init[D * D * D * D];
};
template <int D, int M, int LEARN>
using VmpModel = std::conditional_t<(LEARN & LEARN_A) != 0, VmpTransModel<D, M>,
                                    std::conditional_t<LEARN == LEARN_Q, VmpWishModel<D, M>, VmpNoiseModel<D, M>>>;

__device__ __forceinline__ double digamma_d(double x) {      // psi(x), x > 0: recurrence up to x >= 10, asymptotic series
    double r = 0.0;
    while (x < 10.0) { r -= 1.0 / x; x += 1.0; }
    const double i = 1.0 / x, i2 = i * i;
    return r + log(x) - 0.5 * i - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252 - i2 * (1.0 / 240 - i2 * (1.0 / 132)))));
}

// RTS pair hook, Ss the smoothed covariance at t+1 and F = I - A G: with WANT_V (P learned)
// V = cov(x_{t+1} - A x_t | y) = F Ss F' + A C A', with WANT_X (A learned) X = cov(x_t, x_{t+1} - A x_t | y) = G Ss F' - C A'
template <int D, bool WANT_X, bool WANT_V>
struct PairStats {
    const Mat<float, D, D>& A;
    Mat<float, D, D>& V;
    Mat<float, D, D>& X;
    __device__ __forceinline__ void operator()(const Mat<float, D, D>& G, const Mat<float, D, D>& C,
                                               const Mat<float, D, D>& Ss) const {
        Mat<float, D, D> F = mul(A, G);
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int j = 0; j < D; ++j) F(i, j) = (i == j ? 1.f : 0.f) - F(i, j);
        if constexpr (WANT_X) {
            Mat<float, D, D> GS = mul(G, Ss), GSF = mul_nt(GS, F), CA = mul_nt(C, A);
#pragma unroll
            for (int i = 0; i < D * D; ++i) X.a[i] = GSF.a[i] - CA.a[i];
        }
        if constexpr (WANT_V) {
            Mat<float, D, D> AC = mul(A, C), Z = {};
            Mat<float, D, D> FS = mul(F, Ss);
            V = sym_mul_nt_add(FS, F, sym_mul_nt_add(AC, A, Z));
        }
    }
};

// one transition's term (fp32) folded into the fp64 sums, e = mnext - A ms - u: with WANT_RP R_p += e e' + V (lower
// triangle); with WANT_S the source-state statistics Sxx += Ss + ms ms' (lower triangle), Sxr += X + ms e'
template <int D, bool WANT_S, bool WANT_RP>
__device__ __forceinline__ void accumulate_stats(double* Rp, double* Sxx, double* Sxr, const Mat<float, D, D>& A,
                                                 const Vec<float, D>& u, const Vec<float, D>& mnext,
                                                 const Vec<float, D>& ms, const Mat<float, D, D>& Ss,
                                                 const Mat<float, D, D>& V, const Mat<float, D, D>& X) {
    Vec<float, D> e = mulv(A, ms);
#pragma unroll
    for (int k = 0; k < D; ++k) e(k) = mnext(k) - (e(k) + u(k));
    int q = 0;
#pragma unroll
    for (int k = 0; k < D; ++k)
#pragma unroll
        for (int l = 0; l <= k; ++l) {
            if constexpr (WANT_S) Sxx[q] += (double)__fmaf_rn(ms(k), ms(l), Ss(k, l));
            if constexpr (WANT_RP) Rp[q] += (double)__fmaf_rn(e(k), e(l), V(k, l));
            ++q;
        }
    if constexpr (WANT_S) {
#pragma unroll
        for (int k = 0; k < D; ++k)
#pragma unroll
            for (int l = 0; l < D; ++l) Sxr[k * D + l] += (double)__fmaf_rn(ms(k), e(l), X(k, l));
    }
}

// the fp32 factor L (L L' = Xi) of the tilt of one sweep, Xi[j][k] = sum_{i,l} W[i][l] Sa[(i,j),(l,k)] (fp64)
template <int D>
__device__ __forceinline__ Mat<float, D, D> xi_factor(const double* Sa, const Mat<double, D, D>& W, bool& bad) {
    constexpr int N = D * D;
    Mat<double, D, D> Xi;
#pragma unroll
    for (int j = 0; j < D; ++j)
#pragma unroll
        for (int k = 0; k < D; ++k) {
            double s = 0.0;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int l = 0; l < D; ++l) s = fma(W(i, l), Sa[(i * D + j) * N + l * D + k], s);
            Xi(j, k) = s;
        }
    Chol<double, D> c = cholesky<double, D, false>(Xi, bad);
    Mat<float, D, D> L;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) L(i, j) = (float)(i == j ? 1.0 / c.L(i, i) : c.L(i, j));
    return L;
}

// K[i][l] = sum_{j,k} Sa[(i,j),(l,k)] Sxx[j][k] = E[(A - Abar) Sxx (A - Abar)']
template <int D>
__device__ __forceinline__ Mat<double, D, D> kron_contract(const double* Sa, const Mat<double, D, D>& Sxx) {
    constexpr int N = D * D;
    Mat<double, D, D> K;
#pragma unroll 1
    for (int i = 0; i < D; ++i)
#pragma unroll 1
        for (int l = 0; l < D; ++l) {
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < D; ++j)
#pragma unroll
                for (int k = 0; k < D; ++k) s = fma(Sa[(i * D + j) * N + l * D + k], Sxx(j, k), s);
            K.a[i * D + l] = s;
        }
    return K;
}

// q(a) after one sweep (fp64; am, Sa, Lam: local arrays of n = D*D and n*n):
//   Lambda = Va0^-1 + W (x) Sxx,  am += Lambda^-1 (Va0^-1 (ma0 - am) + vec(W Sxr')),  Sa = Lambda^-1.
// On return dR = D Sxx D' - D Sxr - Sxr' D' + K_new (R_p,new = R_p(Abar_old) + dR, D = Abar_new - Abar_old) and fe_a =
// 1/2 tr(W (dR - K_old)) + KL(q(a) || N(ma0, Va0)).
template <int D, typename Mdl>
__device__ __forceinline__ void qa_update(const Mdl& mdl, double* am, double* Sa, double* Lam,
                                          const Mat<double, D, D>& W, const Mat<double, D, D>& Sxx,
                                          const Mat<double, D, D>& Sxr, Mat<double, D, D>& dR, double& fe_a, bool& bad) {
    constexpr int N = D * D;
    const Mat<double, D, D> Kold = kron_contract<D>(Sa, Sxx);
    // Lambda and its Cholesky factor (lower, in place)
#pragma unroll 1
    for (int r = 0; r < N; ++r)
#pragma unroll 1
        for (int c = 0; c <= r; ++c)
            Lam[r * N + c] = mdl.Va0i[r * N + c] + W(r / D, c / D) * Sxx(r % D, c % D);
    double logdet_Lam = 0.0;
#pragma unroll 1
    for (int j = 0; j < N; ++j) {
        double s = Lam[j * N + j];
#pragma unroll 1
        for (int k = 0; k < j; ++k) s -= Lam[j * N + k] * Lam[j * N + k];
        if (!(s > 0.0)) { bad = true; s = 1e-300; }
        const double l = sqrt(s);
        Lam[j * N + j] = l;
        logdet_Lam += 2.0 * log(l);
#pragma unroll 1
        for (int i = j + 1; i < N; ++i) {
            double t = Lam[i * N + j];
#pragma unroll 1
            for (int k = 0; k < j; ++k) t -= Lam[i * N + k] * Lam[j * N + k];
            Lam[i * N + j] = t / l;
        }
    }
    // L^-1 in place, column by column; then Sa = L^-T L^-1
#pragma unroll 1
    for (int j = 0; j < N; ++j) {
        Lam[j * N + j] = 1.0 / Lam[j * N + j];
#pragma unroll 1
        for (int i = j + 1; i < N; ++i) {
            double s = 0.0;
#pragma unroll 1
            for (int k = j; k < i; ++k) s += Lam[i * N + k] * Lam[k * N + j];
            Lam[i * N + j] = -s / Lam[i * N + i];
        }
    }
#pragma unroll 1
    for (int r = 0; r < N; ++r)
#pragma unroll 1
        for (int c = 0; c <= r; ++c) {
            double s = 0.0;
#pragma unroll 1
            for (int k = r; k < N; ++k) s += Lam[k * N + r] * Lam[k * N + c];
            Sa[r * N + c] = s;
            Sa[c * N + r] = s;
        }
    // g = Va0^-1 (ma0 - am) + vec(W Sxr'); am += Sa g (Lam's first row reused as g)
    double* g = Lam;
#pragma unroll 1
    for (int r = 0; r < N; ++r) {
        double s = 0.0;
#pragma unroll 1
        for (int c = 0; c < N; ++c) s += mdl.Va0i[r * N + c] * (mdl.ma0[c] - am[c]);
        const int i = r / D, j = r % D;
#pragma unroll
        for (int l = 0; l < D; ++l) s = fma(W(i, l), Sxr(j, l), s);
        g[r] = s;
    }
    Mat<double, D, D> Dl;
#pragma unroll 1
    for (int r = 0; r < N; ++r) {
        double s = 0.0;
#pragma unroll 1
        for (int c = 0; c < N; ++c) s += Sa[r * N + c] * g[c];
        Dl.a[r] = s;
        am[r] += s;
    }
    // dR = Dl Sxx Dl' - Dl Sxr - Sxr' Dl' + K_new
    const Mat<double, D, D> Knew = kron_contract<D>(Sa, Sxx);
    const Mat<double, D, D> DS = mul(Dl, Sxx), DX = mul(Dl, Sxr);
    double tr = 0.0;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int l = 0; l < D; ++l) {
            double s = Knew(i, l) - DX(i, l) - DX(l, i);
#pragma unroll
            for (int k = 0; k < D; ++k) s = fma(DS(i, k), Dl(l, k), s);
            dR(i, l) = s;
            tr = fma(W(i, l), s - Kold(i, l), tr);
        }
    // KL(N(am, Sa) || N(ma0, Va0)) = 1/2 (tr(Va0^-1 Sa) + (am - ma0)' Va0^-1 (am - ma0) - n + log det Va0 + log det Lambda)
    double q = 0.0;
#pragma unroll 1
    for (int r = 0; r < N; ++r)
#pragma unroll 1
        for (int c = 0; c < N; ++c)
            q += mdl.Va0i[r * N + c] * (Sa[c * N + r] + (am[r] - mdl.ma0[r]) * (am[c] - mdl.ma0[c]));
    fe_a = 0.5 * tr + 0.5 * (q - N + mdl.logdet_Va0 + logdet_Lam);
}

// the noise covariance of one q(x) sweep: inv(Wbar) when the precision is learned, else the known matrix; and log det Wbar
template <bool LEARNED, int K>
__device__ __forceinline__ Mat<float, K, K> noise_cov(const Mat<double, K, K>& Wbar, const float* known, bool& bad) {
    if constexpr (LEARNED) return convert<float>(cholinv(Wbar, bad));
    else return load_const<float, K, K>(known);
}
template <bool LEARNED, int K>
__device__ __forceinline__ double noise_logdet(const Mat<double, K, K>& Wbar, bool& bad) {
    if constexpr (LEARNED) return -2.0 * cholesky<double, K, true>(Wbar, bad).neg_half_logdet;
    else return 0.0;
}
template <int D, int M>
__device__ __forceinline__ const float* known_q(const VmpWishModel<D, M>&) { return nullptr; }
template <int D, int M>
__device__ __forceinline__ const float* known_q(const VmpNoiseModel<D, M>& mdl) { return mdl.Q; }

// q(w) = Wishart(nu0 + N, inv(Psi0 + R)) from the lower triangle of R, written for iteration it; with want_fe, FE gains
// N/2 (log det Wbar - E log det w) + 1/2 tr((E w - Wbar) R) + KL(q(w) || prior) and STORE writes it to io.fe.  WBAR
// becomes E[w].  fp64 throughout.  A macro rather than a function: expanded in the kernel body, the learn-Q kernels
// compile to the same code as before the process noise could be learned (a helper function is optimised before it is
// inlined, which reorders the loop-carried registers).
#define RXG_WISHART_UPDATE(K, PR, R, N, LOGDET_W, WBAR, DF_OUT, IS_OUT, FE, STORE)                                    \
    {                                                                                                               \
        const double df = (PR).nu0 + (double)(N);                                                                   \
        Mat<double, K, K> Psi;                                                                                      \
        {                                                                                                           \
            int q = 0;                                                                                              \
            _Pragma("unroll") for (int k = 0; k < K; ++k)                                                           \
                _Pragma("unroll") for (int l = 0; l <= k; ++l) {                                                    \
                    Psi(k, l) = (PR).Psi0[k * K + l] + R[q];                                                        \
                    Psi(l, k) = Psi(k, l);                                                                          \
                    ++q;                                                                                            \
                }                                                                                                   \
        }                                                                                                           \
        const Mat<double, K, K> Pinv = cholinv(Psi, bad);                                                           \
        DF_OUT[(int64_t)it * batch + b] = (float)df;                                                                \
        _Pragma("unroll") for (int k = 0; k < K; ++k)                                                               \
            _Pragma("unroll") for (int l = 0; l < K; ++l)                                                           \
                IS_OUT[(((int64_t)it * K + k) * K + l) * batch + b] = (float)Psi(k, l);                             \
        Mat<double, K, K> Wn;                                                                                       \
        _Pragma("unroll") for (int i = 0; i < K * K; ++i) Wn.a[i] = df * Pinv.a[i];                                 \
        if (want_fe) {                                                                                              \
            const double logdet_Psi = -2.0 * cholesky<double, K, true>(Psi, bad).neg_half_logdet;                   \
            double psi_m = 0.0, lg = 0.0; /* sum_i psi((df - i)/2), sum_i [lgamma((nu0 - i)/2) - lgamma((df - i)/2)] */ \
            _Pragma("unroll") for (int i = 0; i < K; ++i) {                                                         \
                psi_m += digamma_d(0.5 * (df - i));                                                                 \
                lg += lgamma(0.5 * ((PR).nu0 - i)) - lgamma(0.5 * (df - i));                                        \
            }                                                                                                       \
            const double Elogdet = psi_m + K * 0.69314718055994530942 - logdet_Psi;                                 \
            double trR = 0.0, trP = 0.0; /* tr((E w - Wbar) R), tr(Psi0 inv(Psi)) */                                \
            {                                                                                                       \
                int q = 0;                                                                                          \
                _Pragma("unroll") for (int k = 0; k < K; ++k)                                                       \
                    _Pragma("unroll") for (int l = 0; l <= k; ++l) {                                                \
                        const double f = (k == l) ? 1.0 : 2.0;                                                      \
                        trR += f * (Wn(k, l) - WBAR(k, l)) * R[q++];                                                \
                        trP += f * (PR).Psi0[k * K + l] * Pinv(k, l);                                               \
                    }                                                                                               \
            }                                                                                                       \
            const double kl = -0.5 * (PR).nu0 * ((PR).logdet_Psi0 - logdet_Psi) + 0.5 * df * (trP - K) + lg +       \
                              0.5 * (df - (PR).nu0) * psi_m;                                                        \
            FE = FE + 0.5 * (N) * (LOGDET_W - Elogdet) + 0.5 * trR + kl;                                            \
            if (STORE) io.fe[(int64_t)it * batch + b] = FE;                                                         \
        }                                                                                                           \
        WBAR = Wn;                                                                                                  \
    }

template <int D, int M, int LEARN>
__global__ void __launch_bounds__(128)
lgssm_vmp_wishart_kernel(const __grid_constant__ VmpModel<D, M, LEARN> mdl, const VmpIO<LEARN> io) {
    constexpr bool LQ = (LEARN & LEARN_Q) != 0, LP = (LEARN & LEARN_P) != 0, LA = (LEARN & LEARN_A) != 0;
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t batch = io.batch;
    if (b >= batch) return;
    const int T = io.T;
    const float* __restrict__ y = io.y;
    float* __restrict__ mean = io.mean;
    float* __restrict__ cov = io.cov;
    const Mat<float, D, D> A = load_const<float, D, D>(mdl.A), P = load_const<float, D, D>(mdl.P),
                           S0 = load_const<float, D, D>(mdl.S0);
    const Mat<float, M, D> B = load_const<float, M, D>(mdl.B);
    Vec<float, D> u;
#pragma unroll
    for (int i = 0; i < D; ++i) u(i) = mdl.u[i];
    auto observed_at = [&](int t) -> bool {
        return io.ymask ? io.ymask[(int64_t)t * batch + b] != 0 : (io.tmask ? io.tmask[t] != 0 : true);
    };
    Mat<double, M, M> Wbar;
#pragma unroll
    for (int i = 0; i < M * M; ++i) Wbar.a[i] = mdl.q.W0[i];
    Mat<double, D, D> Wp;                  // E[w_p] under the previous q(w_p)
    bool bad = false;
    if constexpr (LP) {
#pragma unroll
        for (int i = 0; i < D * D; ++i) Wp.a[i] = mdl.p.W0[i];
    } else if constexpr (LA) {
        Wp = cholinv(convert<double>(P), bad);
    }
    constexpr int NA = LA ? D * D : 1;
    double am[NA], Sa[NA * NA], Lam[NA * NA];   // E[a], cov(a) of the previous q(a); q(a) workspace (local memory)
    if constexpr (LA) {
#pragma unroll 1
        for (int i = 0; i < NA; ++i) am[i] = mdl.ma_init[i];
#pragma unroll 1
        for (int i = 0; i < NA * NA; ++i) Sa[i] = mdl.Sa_init[i];
    }
    const bool want_fe = io.fe != nullptr;
    Vec<float, D> mu;

    for (int it = 0; it < io.iterations; ++it) {
        const bool last = it == io.iterations - 1;
        Mat<float, D, D> Al, Lx;            // LEARN_A: E[A] and the factor of Xi of this sweep
        if constexpr (LA) {
#pragma unroll
            for (int i = 0; i < D * D; ++i) Al.a[i] = (float)am[i];
            Lx = xi_factor<D>(Sa, Wp, bad);
        }
        const Mat<float, D, D>& Ab = LA ? Al : A;
        // ---- q(x) under P = inv(Wp) and Q = inv(Wbar) (learned) or the known matrices
        const double logdet_W = noise_logdet<LQ>(Wbar, bad);
        const Mat<float, M, M> Q = noise_cov<LQ>(Wbar, known_q(mdl), bad);
        const double logdet_Wp = noise_logdet<LP>(Wp, bad);
        Mat<float, D, D> Pl;
        if constexpr (LP) Pl = convert<float>(cholinv(Wp, bad));
        const Mat<float, D, D>& Pb = LP ? Pl : P;
#pragma unroll
        for (int i = 0; i < D; ++i) mu(i) = mdl.m0[i];
        Mat<float, D, D> S = S0;
        double nle = 0.0;
        int nobs = 0;
        Vec<float, M> yt;
        bool obs = false;
        float ynext[M];
#pragma unroll
        for (int k = 0; k < M; ++k) ynext[k] = __ldg(y + (int64_t)k * batch + b);
        bool onext = observed_at(0);
        for (int t = 0; t < T; ++t) {
#pragma unroll
            for (int k = 0; k < M; ++k) yt(k) = ynext[k];
            obs = onext;
            if (t + 1 < T) {   // prefetch next step's datum while this step's arithmetic runs
#pragma unroll
                for (int k = 0; k < M; ++k) ynext[k] = __ldg(y + ((int64_t)(t + 1) * M + k) * batch + b);
                onext = observed_at(t + 1);
            }
            if constexpr (LA) {
                if (t == 0 && io.tf) chain_tilt(Lx, want_fe, mu, S, bad, nle);    // the prior state is a source state
            }
            if (t > 0 || io.tf) chain_predict(Ab, Pb, u, NoInput{}, mu, S);
            if (obs) {
                chain_update(B, Q, yt, want_fe, mu, S, bad, nle);
                ++nobs;
            }
            if constexpr (LA) {
                if (t < T - 1) chain_tilt(Lx, want_fe, mu, S, bad, nle);
            }
            // the backward pass starts from the registers: step T-1 is stored only as the final posterior
            if (t < T - 1 || last) {
#pragma unroll
                for (int i = 0; i < D; ++i) mean[((int64_t)t * D + i) * batch + b] = mu(i);
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int j = 0; j < D; ++j)
                        if (t == T - 1 || j <= i) cov[(((int64_t)t * D + i) * D + j) * batch + b] = S(i, j);
            }
        }

        // ---- backward RTS pass, R_q = sum_{observed t} (y_t - B mu_t)(y_t - B mu_t)' + B Sigma_t B' and
        //      R_p = sum_t e e' + cov(x_{t+1} - A x_t | y), e = mu_{t+1} - A mu_t - u (fp64 sums of fp32 step terms)
        double R[M * (M + 1) / 2];
#pragma unroll
        for (int q = 0; q < M * (M + 1) / 2; ++q) R[q] = 0.0;
        auto accumulate = [&](const Vec<float, D>& ms, const Mat<float, D, D>& Sm, const Vec<float, M>& yv) {
            Vec<float, M> e = mulv(B, ms);
            Mat<float, M, M> E;
#pragma unroll
            for (int k = 0; k < M; ++k) e(k) = yv(k) - e(k);
#pragma unroll
            for (int k = 0; k < M; ++k)
#pragma unroll
                for (int l = 0; l < M; ++l) E(k, l) = e(k) * e(l);
            Mat<float, M, D> BS = mul(B, Sm);
            Mat<float, M, M> Rt = sym_mul_nt_add(BS, B, E);
            int q = 0;
#pragma unroll
            for (int k = 0; k < M; ++k)
#pragma unroll
                for (int l = 0; l <= k; ++l) R[q++] += (double)Rt(k, l);
        };
        double Rp[D * (D + 1) / 2];
        if constexpr (LP) {
#pragma unroll
            for (int q = 0; q < D * (D + 1) / 2; ++q) Rp[q] = 0.0;
        }
        double Sxx[LA ? D * (D + 1) / 2 : 1], Sxr[NA];   // LEARN_A: sum E[x_t x_t'] (lower), sum E[x_t r_t']
        if constexpr (LA) {
#pragma unroll
            for (int q = 0; q < D * (D + 1) / 2; ++q) Sxx[q] = 0.0;
#pragma unroll
            for (int q = 0; q < NA; ++q) Sxr[q] = 0.0;
        }
        if constexpr (LQ) {
            if (obs) accumulate(mu, S, yt);
        }
        Vec<float, D> mus = mu;          // smoothed at t+1
        Mat<float, D, D> Ss = S;
        float pm[D], pS[D * (D + 1) / 2], py[M];
        bool po = false;
        auto prefetch = [&](int t) {
#pragma unroll
            for (int i = 0; i < D; ++i) pm[i] = mean[((int64_t)t * D + i) * batch + b];
            int q = 0;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j <= i; ++j) pS[q++] = cov[(((int64_t)t * D + i) * D + j) * batch + b];
#pragma unroll
            for (int k = 0; k < M; ++k) py[k] = __ldg(y + ((int64_t)t * M + k) * batch + b);
            po = observed_at(t);
        };
        if (T >= 2) prefetch(T - 2);
        for (int t = T - 2; t >= 0; --t) {
            Vec<float, D> muf;
            Mat<float, D, D> Sf;
            Vec<float, M> yv;
#pragma unroll
            for (int i = 0; i < D; ++i) muf(i) = pm[i];
            {
                int q = 0;
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int j = 0; j <= i; ++j) { Sf(i, j) = pS[q]; Sf(j, i) = pS[q]; ++q; }
            }
#pragma unroll
            for (int k = 0; k < M; ++k) yv(k) = py[k];
            const bool ob = po;
            if (t > 0) prefetch(t - 1);
            if constexpr (LA || LP) {
                const Vec<float, D> mnext = mus;
                Mat<float, D, D> V, X;
                chain_rts(Ab, Pb, u, NoInput{}, muf, Sf, mus, Ss, bad, PairStats<D, LA, LP>{Ab, V, X});
                accumulate_stats<D, LA, LP>(Rp, Sxx, Sxr, Ab, u, mnext, mus, Ss, V, X);
            } else {
                chain_rts(A, Pb, u, NoInput{}, muf, Sf, mus, Ss, bad);
            }
            if (last) {
#pragma unroll
                for (int i = 0; i < D; ++i) mean[((int64_t)t * D + i) * batch + b] = mus(i);
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int j = 0; j < D; ++j) cov[(((int64_t)t * D + i) * D + j) * batch + b] = Ss(i, j);
            }
            if constexpr (LQ) {
                if (ob) accumulate(mus, Ss, yv);
            }
        }
        if constexpr (LA || LP) {
            // the transition from the prior state (tilted when A is learned) into x[1]: one more RTS step from (m0, S0),
            // not written out
            if (io.tf) {
                Vec<float, D> m0v, mx = mus;
                Mat<float, D, D> S0t, Sx = Ss, V, X;
#pragma unroll
                for (int i = 0; i < D; ++i) m0v(i) = mdl.m0[i];
                if constexpr (LA) {
                    double unused = 0.0;
                    S0t = S0;
                    chain_tilt(Lx, false, m0v, S0t, bad, unused);
                }
                // bound, not copied, when A is known: a copy of S0 changes the learn-P kernels' instruction schedule
                const Mat<float, D, D>& S0b = LA ? S0t : S0;
                chain_rts(Ab, Pb, u, NoInput{}, m0v, S0b, mx, Sx, bad, PairStats<D, LA, LP>{Ab, V, X});
                accumulate_stats<D, LA, LP>(Rp, Sxx, Sxr, Ab, u, mus, mx, Sx, V, X);
            }
        }
        mu = mus;

        // ---- q(w_p), q(w_q) = Wishart(df, inv(Psi)) and the free energy (fp64)
        double fe = nle;
        if constexpr (LA) {   // ---- q(a) with the Wbar_p of this sweep, then R_p at the new E[A]
            Mat<double, D, D> SxxM, SxrM, dR;
            int q = 0;
#pragma unroll
            for (int k = 0; k < D; ++k)
#pragma unroll
                for (int l = 0; l <= k; ++l) { SxxM(k, l) = Sxx[q]; SxxM(l, k) = Sxx[q]; ++q; }
#pragma unroll
            for (int i = 0; i < D * D; ++i) SxrM.a[i] = Sxr[i];
            // the sweep, Sxr and R_p(Abar_old) used the fp32 E[A]: take it as Abar_old, so that D = Abar_new - Abar_old
            // matches them (with the fp64 E[A], D Sxx D' would carry the fp32 rounding of E[A] times |x|^2)
#pragma unroll
            for (int i = 0; i < D * D; ++i) am[i] = (double)Al.a[i];
            double fe_a;
            qa_update<D>(mdl, am, Sa, Lam, Wp, SxxM, SxrM, dR, fe_a, bad);
            fe += fe_a;
#pragma unroll 1
            for (int r = 0; r < NA; ++r) io.a_mean[((int64_t)it * NA + r) * batch + b] = (float)am[r];
#pragma unroll 1
            for (int r = 0; r < NA * NA; ++r) io.a_cov[((int64_t)it * NA * NA + r) * batch + b] = (float)Sa[r];
            if constexpr (LP) {
                q = 0;
#pragma unroll
                for (int k = 0; k < D; ++k)
#pragma unroll
                    for (int l = 0; l <= k; ++l) Rp[q++] += dR(k, l);
            }
            if (want_fe && !LP && !LQ) io.fe[(int64_t)it * batch + b] = fe;
        }
        if constexpr (LP) RXG_WISHART_UPDATE(D, mdl.p, Rp, T - 1 + io.tf, logdet_Wp, Wp, io.df_p, io.inv_scale_p, fe, !LQ)
        if constexpr (LQ) RXG_WISHART_UPDATE(M, mdl.q, R, nobs, logdet_W, Wbar, io.df, io.inv_scale, fe, true)
    }
    if (io.status) {
        bool nan = false;
#pragma unroll
        for (int i = 0; i < D; ++i) nan |= !(mu(i) == mu(i));
        io.status[b] = bad ? RXG_ERR_NOT_SPD : (nan ? RXG_ERR_NAN : RXG_OK);
    }
}

template <int D, int M, int LEARN>
int launch_vmp_wishart(rxg_ctx* ctx, const VmpWishHost& h, const VmpTransIO& io) {
    VmpModel<D, M, LEARN> mdl = {};
    for (int i = 0; i < D * D; ++i) { mdl.A[i] = h.A ? h.A[i] : 0.f; mdl.P[i] = h.P ? h.P[i] : 0.f; mdl.S0[i] = h.S0[i]; }
    for (int i = 0; i < M * D; ++i) mdl.B[i] = h.B[i];
    for (int i = 0; i < D; ++i) { mdl.m0[i] = h.m0[i]; mdl.u[i] = h.u ? h.u[i] : 0.f; }
    for (int i = 0; i < M * M; ++i) { mdl.q.Psi0[i] = h.Psi0[i]; mdl.q.W0[i] = h.W0[i]; }
    mdl.q.nu0 = h.nu0;
    mdl.q.logdet_Psi0 = h.logdet_Psi0;
    if constexpr (LEARN != LEARN_Q) {
        for (int i = 0; i < M * M; ++i) mdl.Q[i] = h.Q ? h.Q[i] : 0.f;
        for (int i = 0; i < D * D; ++i) { mdl.p.Psi0[i] = h.Psi_p0[i]; mdl.p.W0[i] = h.Wp0[i]; }
        mdl.p.nu0 = h.nu_p0;
        mdl.p.logdet_Psi0 = h.logdet_Psi_p0;
    }
    if constexpr ((LEARN & LEARN_A) != 0) {
        constexpr int N = D * D;
        for (int i = 0; i < N; ++i) { mdl.ma0[i] = h.ma0[i]; mdl.ma_init[i] = h.ma_init[i]; }
        for (int i = 0; i < N * N; ++i) { mdl.Va0i[i] = h.Va0i[i]; mdl.Sa_init[i] = h.Sa_init[i]; }
        mdl.logdet_Va0 = h.logdet_Va0;
    }
    const VmpIO<LEARN>& kio = io;
    const int threads = 64;
    if (ctx->profile) { cudaEventRecord(ctx->ev[0], ctx->stream); cudaEventRecord(ctx->ev[1], ctx->stream); }
    lgssm_vmp_wishart_kernel<D, M, LEARN><<<(unsigned)((io.batch + threads - 1) / threads), threads, 0, ctx->stream>>>(mdl, kio);
    if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "lgssm_vmp_wishart_kernel launch");
}

#define RXG_VMP_LAUNCH(PFX, DD, MM, LL) \
    PFX template int launch_vmp_wishart<DD, MM, LL>(rxg_ctx*, const VmpWishHost&, const VmpTransIO&);
#define RXG_VMP_DECL(PFX, DD, MM) \
    RXG_VMP_LAUNCH(PFX, DD, MM, LEARN_Q) RXG_VMP_LAUNCH(PFX, DD, MM, LEARN_P) RXG_VMP_LAUNCH(PFX, DD, MM, LEARN_PQ)
#define RXG_VMP_DECL_A(PFX, DD, MM)                                                                             \
    RXG_VMP_LAUNCH(PFX, DD, MM, LEARN_A) RXG_VMP_LAUNCH(PFX, DD, MM, LEARN_A | LEARN_P)                         \
    RXG_VMP_LAUNCH(PFX, DD, MM, LEARN_A | LEARN_Q) RXG_VMP_LAUNCH(PFX, DD, MM, LEARN_A | LEARN_PQ)

#ifdef RXG_VMP_M
RXG_VMP_DECL(, 1, RXG_VMP_M) RXG_VMP_DECL(, 2, RXG_VMP_M) RXG_VMP_DECL(, 3, RXG_VMP_M)
RXG_VMP_DECL(, 4, RXG_VMP_M) RXG_VMP_DECL(, 5, RXG_VMP_M) RXG_VMP_DECL(, 6, RXG_VMP_M)
RXG_VMP_DECL_A(, 1, RXG_VMP_M) RXG_VMP_DECL_A(, 2, RXG_VMP_M) RXG_VMP_DECL_A(, 3, RXG_VMP_M)
RXG_VMP_DECL_A(, 4, RXG_VMP_M)
}  // namespace rxg
#else

#define RXG_VMP_EXTERN(DECL, DD)                                                                            \
    DECL(extern, DD, 1) DECL(extern, DD, 2) DECL(extern, DD, 3) DECL(extern, DD, 4) DECL(extern, DD, 5)         \
    DECL(extern, DD, 6)
RXG_VMP_EXTERN(RXG_VMP_DECL, 1) RXG_VMP_EXTERN(RXG_VMP_DECL, 2) RXG_VMP_EXTERN(RXG_VMP_DECL, 3)
RXG_VMP_EXTERN(RXG_VMP_DECL, 4) RXG_VMP_EXTERN(RXG_VMP_DECL, 5) RXG_VMP_EXTERN(RXG_VMP_DECL, 6)
RXG_VMP_EXTERN(RXG_VMP_DECL_A, 1) RXG_VMP_EXTERN(RXG_VMP_DECL_A, 2) RXG_VMP_EXTERN(RXG_VMP_DECL_A, 3)
RXG_VMP_EXTERN(RXG_VMP_DECL_A, 4)
#undef RXG_VMP_EXTERN

namespace {
// fp64 Cholesky L L' of the symmetrised (A + A')/2 on the host (n <= 16): false if it is not SPD or not finite; L
// (lower, the rest untouched) and log det on success
bool host_chol(const float* a, int n, double* L, double* logdet) {
    double ld = 0.0;
    for (int j = 0; j < n; ++j) {
        double s = 0.5 * ((double)a[j * n + j] + (double)a[j * n + j]);
        for (int k = 0; k < j; ++k) s -= L[j * n + k] * L[j * n + k];
        if (!(s > 0.0) || !isfinite(s)) return false;
        L[j * n + j] = sqrt(s);
        ld += 2.0 * log(L[j * n + j]);
        for (int i = j + 1; i < n; ++i) {
            double t = 0.5 * ((double)a[i * n + j] + (double)a[j * n + i]);
            for (int k = 0; k < j; ++k) t -= L[i * n + k] * L[j * n + k];
            L[i * n + j] = t / L[j * n + j];
        }
    }
    *logdet = ld;
    return true;
}

// the symmetrised matrix itself, checked to be SPD
bool host_spd(const float* a, int m, double* sym, double* logdet) {
    double L[36];
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < m; ++j) sym[i * m + j] = 0.5 * ((double)a[i * m + j] + (double)a[j * m + i]);
    return host_chol(a, m, L, logdet);
}

// the kernel of (learn, d, m): the instantiations of RXG_VMP_DECL (d = 1..6) and RXG_VMP_DECL_A (d = 1..4)
int dispatch_vmp(rxg_ctx* ctx, int learn, int d, int m, const VmpWishHost& h, const VmpTransIO& io) {
#define RXG_VMP_CASE(LL, DD, MM) case ((LL) * 8 + DD) * 8 + MM: return launch_vmp_wishart<DD, MM, LL>(ctx, h, io);
#define RXG_VMP_ROW(LL, DD) RXG_VMP_CASE(LL, DD, 1) RXG_VMP_CASE(LL, DD, 2) RXG_VMP_CASE(LL, DD, 3) \
                            RXG_VMP_CASE(LL, DD, 4) RXG_VMP_CASE(LL, DD, 5) RXG_VMP_CASE(LL, DD, 6)
#define RXG_VMP_D4(LL) RXG_VMP_ROW(LL, 1) RXG_VMP_ROW(LL, 2) RXG_VMP_ROW(LL, 3) RXG_VMP_ROW(LL, 4)
#define RXG_VMP_D6(LL) RXG_VMP_D4(LL) RXG_VMP_ROW(LL, 5) RXG_VMP_ROW(LL, 6)
    switch ((learn * 8 + d) * 8 + m) {
        RXG_VMP_D6(LEARN_Q) RXG_VMP_D6(LEARN_P) RXG_VMP_D6(LEARN_PQ)
        RXG_VMP_D4(LEARN_A) RXG_VMP_D4(LEARN_A | LEARN_Q) RXG_VMP_D4(LEARN_A | LEARN_P) RXG_VMP_D4(LEARN_A | LEARN_PQ)
        default:     // not reached: vmp_noise() has refused every other combination
            return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_vmp: no kernel for learn=%d, d=%d, m=%d", learn, d, m);
    }
#undef RXG_VMP_D6
#undef RXG_VMP_D4
#undef RXG_VMP_ROW
#undef RXG_VMP_CASE
}

}  // namespace

// fp64 Cholesky of the symmetrised n x n matrix on the host (n <= 16), then its inverse: false if it is not SPD
// (declared in rxg_internal.h: the Gaussian-mixture entry validates its host matrices with it too)
bool host_spd_inv(const float* a, int n, double* inv, double* logdet) {
    double L[256], Li[256] = {};
    if (!host_chol(a, n, L, logdet)) return false;
    for (int j = 0; j < n; ++j) {
        Li[j * n + j] = 1.0 / L[j * n + j];
        for (int i = j + 1; i < n; ++i) {
            double s = 0.0;
            for (int k = j; k < i; ++k) s += L[i * n + k] * Li[k * n + j];
            Li[i * n + j] = -s / L[i * n + i];
        }
    }
    for (int r = 0; r < n; ++r)
        for (int c = 0; c < n; ++c) {
            double s = 0.0;
            for (int k = (r > c ? r : c); k < n; ++k) s += Li[k * n + r] * Li[k * n + c];
            inv[r * n + c] = s;
        }
    return true;
}

namespace {

// the transition matrix of rxg_lgssm_vmp_transition_f32: its Gaussian prior, the initial q(a) and the outputs
struct TransArg {
    const float *mean0, *cov0, *init_mean, *init_cov;
    float *a_mean, *a_cov;
};

// One noise of the call: the known matrix, or the Wishart prior and the initial E[w] when it is learned.
struct NoiseArg {
    char name;                 // 'p' or 'q'
    int k;                     // its dimension (d or m)
    const float *known, *inv_scale0, *init_E_W;
    float nu0;
    float *df, *inv_scale;     // outputs of a learned noise
    bool learned() const { return inv_scale0 || init_E_W; }
};

// argument checks shared by both noises: exactly one of the known matrix and (inv_scale0, init_E_W); the outputs of a
// learned noise and nothing else
int check_noise(rxg_ctx* ctx, const char* who, const NoiseArg& a) {
    if (!a.known == !a.learned())
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: pass exactly one of %c (known) and inv_scale_%c0 / init_E_W%c (learned)", who,
                    a.name - 32, a.name, a.name);
    if (a.learned() && !(a.inv_scale0 && a.init_E_W && a.df && a.inv_scale))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: a learned %c needs inv_scale_%c0, init_E_W%c, df_%c and inv_scale_%c", who,
                    a.name - 32, a.name, a.name, a.name, a.name);
    if (!a.learned() && (a.df || a.inv_scale))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: df_%c / inv_scale_%c must be NULL when %c is known", who, a.name, a.name,
                    a.name - 32);
    return RXG_OK;
}

int prior_of(rxg_ctx* ctx, const char* who, const NoiseArg& a, double* nu0, double* Psi0, double* logdet_Psi0, double* W0) {
    if (!((double)a.nu0 > (double)(a.k - 1)) || !isfinite(a.nu0))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: the prior's degrees of freedom must exceed %s - 1 (nu_%c0=%g, %s=%d)", who,
                    a.name == 'p' ? "d" : "m", a.name, (double)a.nu0, a.name == 'p' ? "d" : "m", a.k);
    *nu0 = (double)a.nu0;
    double ld_w = 0.0;
    if (!host_spd(a.inv_scale0, a.k, Psi0, logdet_Psi0))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: inv_scale_%c0 is not symmetric positive definite", who, a.name);
    if (!host_spd(a.init_E_W, a.k, W0, &ld_w))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: init_E_W%c is not symmetric positive definite", who, a.name);
    return RXG_OK;
}

// the one validation and dispatch path of rxg_lgssm_vmp_wishart_f32, rxg_lgssm_vmp_noise_f32 and (ta non-null: A
// learned, A itself null) rxg_lgssm_vmp_transition_f32
int vmp_noise(rxg_ctx* ctx, const char* who, int d, int m, int T, int64_t batch, int iterations, const float* A,
              const float* B, const float* m0, const float* S0, const float* u, const NoiseArg& np, const NoiseArg& nq,
              const float* y, const uint8_t* ymask, float* post_mean, float* post_cov, double* free_energy, int32_t* status,
              unsigned flags, const TransArg* ta = nullptr) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    const unsigned accepted = RXG_PTR_DEVICE | RXG_TRANSITION_FIRST | RXG_MASK_SHARED | RXG_ASYNC;
    if (flags & ~accepted)
        return fail(ctx, RXG_ERR_UNSUPPORTED, "%s: flags 0x%x are not supported (per-chain models, input sequences and the "
                                              "shared covariance output do not apply: the covariances depend on the chain "
                                              "through w)", who, flags & ~accepted);
    if (!(flags & RXG_PTR_DEVICE)) return fail(ctx, RXG_ERR_UNSUPPORTED, "%s takes device pointers", who);
    if (d < 1 || d > (ta ? 4 : 6) || m < 1 || m > 6)
        return fail(ctx, RXG_ERR_UNSUPPORTED, "%s: d must be in 1..%d and m in 1..6 (got d=%d, m=%d)", who, ta ? 4 : 6, d, m);
    if (T < 1 || batch < 1 || iterations < 1)
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: T, batch and iterations must be >= 1", who);
    if (!(A || ta) || !B || !m0 || !S0 || !y || !post_mean || !post_cov)
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: null pointer argument", who);
    int rc;
    if ((rc = check_noise(ctx, who, np)) != RXG_OK || (rc = check_noise(ctx, who, nq)) != RXG_OK) return rc;
    if (!ta && !np.learned() && !nq.learned())
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: P and Q are both known: that is the plain smoother (rxg_lgssm_smooth_f32)", who);
    VmpWishHost h = {};
    h.A = A; h.B = B; h.m0 = m0; h.S0 = S0; h.u = u; h.P = np.known; h.Q = nq.known;
    if (nq.learned() && (rc = prior_of(ctx, who, nq, &h.nu0, h.Psi0, &h.logdet_Psi0, h.W0)) != RXG_OK) return rc;
    if (np.learned() && (rc = prior_of(ctx, who, np, &h.nu_p0, h.Psi_p0, &h.logdet_Psi_p0, h.Wp0)) != RXG_OK) return rc;
    if (ta) {
        const int n = d * d;
        if (!ta->mean0 || !ta->cov0 || !ta->init_mean || !ta->init_cov)
            return fail(ctx, RXG_ERR_BAD_ARG, "%s: a_mean0, a_cov0, a_init_mean and a_init_cov are required", who);
        if (!ta->a_mean || !ta->a_cov) return fail(ctx, RXG_ERR_BAD_ARG, "%s: the outputs a_mean and a_cov are required", who);
        double ld_init = 0.0;
        if (!host_spd_inv(ta->cov0, n, h.Va0i, &h.logdet_Va0))
            return fail(ctx, RXG_ERR_BAD_ARG, "%s: a_cov0 is not symmetric positive definite", who);
        if (!host_spd_inv(ta->init_cov, n, h.Sa_init, &ld_init))
            return fail(ctx, RXG_ERR_BAD_ARG, "%s: a_init_cov is not symmetric positive definite", who);
        for (int r = 0; r < n; ++r) {   // the initial covariance itself, symmetrised (host_spd_inv checked it)
            h.ma0[r] = (double)ta->mean0[r];
            h.ma_init[r] = (double)ta->init_mean[r];
            if (!isfinite(h.ma0[r]) || !isfinite(h.ma_init[r]))
                return fail(ctx, RXG_ERR_BAD_ARG, "%s: a_mean0 / a_init_mean must be finite", who);
            for (int c = 0; c < n; ++c)
                h.Sa_init[r * n + c] = 0.5 * ((double)ta->init_cov[r * n + c] + (double)ta->init_cov[c * n + r]);
        }
    }
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    VmpTransIO io;
    io.y = y; io.ymask = nullptr; io.tmask = nullptr;
    io.mean = post_mean; io.cov = post_cov; io.df = nq.df; io.inv_scale = nq.inv_scale; io.fe = free_energy;
    io.status = status; io.df_p = np.df; io.inv_scale_p = np.inv_scale;
    io.a_mean = ta ? ta->a_mean : nullptr; io.a_cov = ta ? ta->a_cov : nullptr;
    io.T = T; io.iterations = iterations; io.tf = (flags & RXG_TRANSITION_FIRST) ? 1 : 0;
    io.batch = batch;
    if (ymask) {
        if (flags & RXG_MASK_SHARED) {
            LgssmCall c = {};
            const int rs = stage_shared_mask(ctx, T, ymask, c);
            if (rs != RXG_OK) return rs;
            io.tmask = c.tmask;
        } else {
            io.ymask = ymask;
        }
    }
    const int learn = (ta ? LEARN_A : 0) | (np.learned() ? LEARN_P : 0) | (nq.learned() ? LEARN_Q : 0);
    if ((rc = dispatch_vmp(ctx, learn, d, m, h, io)) != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
}  // namespace

}  // namespace rxg

using namespace rxg;

extern "C" int rxg_lgssm_vmp_wishart_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch, int iterations, const float* A,
                                         const float* B, const float* P, const float* m0, const float* S0, const float* u,
                                         float nu0, const float* inv_scale0, const float* init_E_W, const float* y,
                                         const uint8_t* ymask, float* post_mean, float* post_cov, float* df,
                                         float* inv_scale, double* free_energy, int32_t* status, unsigned flags) {
    const NoiseArg np = {'p', d, P, nullptr, nullptr, 0.f, nullptr, nullptr};
    const NoiseArg nq = {'q', m, nullptr, inv_scale0, init_E_W, nu0, df, inv_scale};
    return vmp_noise(ctx, "lgssm_vmp_wishart", d, m, T, batch, iterations, A, B, m0, S0, u, np, nq, y, ymask, post_mean,
                     post_cov, free_energy, status, flags);
}

extern "C" int rxg_lgssm_vmp_noise_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch, int iterations, const float* A,
                                       const float* B, const float* m0, const float* S0, const float* u, const float* P,
                                       float nu_p0, const float* inv_scale_p0, const float* init_E_Wp, const float* Q,
                                       float nu_q0, const float* inv_scale_q0, const float* init_E_Wq, const float* y,
                                       const uint8_t* ymask, float* post_mean, float* post_cov, float* df_p,
                                       float* inv_scale_p, float* df_q, float* inv_scale_q, double* free_energy,
                                       int32_t* status, unsigned flags) {
    const NoiseArg np = {'p', d, P, inv_scale_p0, init_E_Wp, nu_p0, df_p, inv_scale_p};
    const NoiseArg nq = {'q', m, Q, inv_scale_q0, init_E_Wq, nu_q0, df_q, inv_scale_q};
    return vmp_noise(ctx, "lgssm_vmp_noise", d, m, T, batch, iterations, A, B, m0, S0, u, np, nq, y, ymask, post_mean,
                     post_cov, free_energy, status, flags);
}

extern "C" int rxg_lgssm_vmp_transition_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch, int iterations,
                                            const float* a_mean0, const float* a_cov0, const float* a_init_mean,
                                            const float* a_init_cov, const float* B, const float* m0, const float* S0,
                                            const float* u, const float* P, float nu_p0, const float* inv_scale_p0,
                                            const float* init_E_Wp, const float* Q, float nu_q0, const float* inv_scale_q0,
                                            const float* init_E_Wq, const float* y, const uint8_t* ymask, float* post_mean,
                                            float* post_cov, float* a_mean, float* a_cov, float* df_p, float* inv_scale_p,
                                            float* df_q, float* inv_scale_q, double* free_energy, int32_t* status,
                                            unsigned flags) {
    const NoiseArg np = {'p', d, P, inv_scale_p0, init_E_Wp, nu_p0, df_p, inv_scale_p};
    const NoiseArg nq = {'q', m, Q, inv_scale_q0, init_E_Wq, nu_q0, df_q, inv_scale_q};
    const TransArg ta = {a_mean0, a_cov0, a_init_mean, a_init_cov, a_mean, a_cov};
    return vmp_noise(ctx, "lgssm_vmp_transition", d, m, T, batch, iterations, nullptr, B, m0, S0, u, np, nq, y, ymask,
                     post_mean, post_cov, free_energy, status, flags, &ta);
}

#endif  // RXG_VMP_M
