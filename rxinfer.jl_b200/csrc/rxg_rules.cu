// Batched twins of the reference's per-message @rule bodies for the Gaussian family
// (SURVEY.md section 8a rows 1-9).  One thread = one message; structure-of-arrays I/O with the
// message index innermost, so every global access of a warp is one contiguous 128-byte request.
// All of these are HBM-bound element-wise kernels (plus a d x d Cholesky where the reference
// calls cholinv); they exist so that a host-side ReactiveMP.rule / BayesBase.prod method
// specialised on a batched message type can forward to the GPU one rule at a time
// [ref: rule binding /root/reference/src/model/plugins/reactivemp_inference.jl:509-540;
//  direct invocation test/inference/inference_tests.jl:547-585].
#include "rxg_internal.h"
#include "rxg_linalg.cuh"

namespace rxg {

template <int R, int C>
__device__ __forceinline__ Mat<float, R, C> ld_soa(const float* __restrict__ p, int64_t n, int64_t i) {
    Mat<float, R, C> o;
#pragma unroll
    for (int k = 0; k < R * C; ++k) o.a[k] = __ldg(p + (int64_t)k * n + i);
    return o;
}
template <int R, int C>
__device__ __forceinline__ Mat<float, R, C> ld_mat(const float* __restrict__ p, int shared, int64_t n, int64_t i) {
    Mat<float, R, C> o;
    if (shared) {
#pragma unroll
        for (int k = 0; k < R * C; ++k) o.a[k] = __ldg(p + k);
    } else {
#pragma unroll
        for (int k = 0; k < R * C; ++k) o.a[k] = __ldg(p + (int64_t)k * n + i);
    }
    return o;
}
template <int N>
__device__ __forceinline__ Vec<float, N> ld_vec(const float* __restrict__ p, int64_t n, int64_t i) {
    Vec<float, N> o;
#pragma unroll
    for (int k = 0; k < N; ++k) o.a[k] = __ldg(p + (int64_t)k * n + i);
    return o;
}
template <int R, int C>
__device__ __forceinline__ void st_soa(float* __restrict__ p, int64_t n, int64_t i, const Mat<float, R, C>& A) {
#pragma unroll
    for (int k = 0; k < R * C; ++k) p[(int64_t)k * n + i] = A.a[k];
}
template <int N>
__device__ __forceinline__ void st_vec(float* __restrict__ p, int64_t n, int64_t i, const Vec<float, N>& v) {
#pragma unroll
    for (int k = 0; k < N; ++k) p[(int64_t)k * n + i] = v.a[k];
}

#define RXG_TID                                                            \
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      \
    if (i >= n) return;

// rules #2 / #3: (mu, S + Sigma)
template <int D>
__global__ void k_add_cov(int64_t n, const float* mu_in, const float* S_in, const float* Sigma, int shared,
                          float* mu_out, float* S_out) {
    RXG_TID
    Vec<float, D> mu = ld_vec<D>(mu_in, n, i);
    Mat<float, D, D> S = ld_soa<D, D>(S_in, n, i);
    Mat<float, D, D> Sg = ld_mat<D, D>(Sigma, shared, n, i);
    st_vec<D>(mu_out, n, i, mu);
    st_soa<D, D>(S_out, n, i, add(S, Sg));
}
// rule #3 from data: (y, Sigma)
template <int D>
__global__ void k_from_data(int64_t n, const float* y, const float* Sigma, int shared, float* mu_out, float* S_out) {
    RXG_TID
    st_vec<D>(mu_out, n, i, ld_vec<D>(y, n, i));
    st_soa<D, D>(S_out, n, i, ld_mat<D, D>(Sigma, shared, n, i));
}
// rule #1: (A mu, A S A')
template <int DO, int DI>
__global__ void k_mul_out(int64_t n, const float* A_, int shared, const float* mu_in, const float* S_in,
                          float* mu_out, float* S_out) {
    RXG_TID
    Mat<float, DO, DI> A = ld_mat<DO, DI>(A_, shared, n, i);
    Vec<float, DI> mu = ld_vec<DI>(mu_in, n, i);
    Mat<float, DI, DI> S = ld_soa<DI, DI>(S_in, n, i);
    Mat<float, DO, DI> AS = mul(A, S);
    Mat<float, DO, DO> Z;
#pragma unroll
    for (int k = 0; k < DO * DO; ++k) Z.a[k] = 0.f;
    st_vec<DO>(mu_out, n, i, mulv(A, mu));
    st_soa<DO, DO>(S_out, n, i, sym_mul_nt_add(AS, A, Z));
}
// rule #4: (A' W mu, A' W A), W = cholinv(S_out)
template <int DO, int DI>
__global__ void k_mul_in(int64_t n, const float* A_, int shared, const float* mu_out, const float* S_out,
                         float* xi_in, float* W_in, int32_t* status) {
    RXG_TID
    Mat<float, DO, DI> A = ld_mat<DO, DI>(A_, shared, n, i);
    Vec<float, DO> mu = ld_vec<DO>(mu_out, n, i);
    Mat<float, DO, DO> S = ld_soa<DO, DO>(S_out, n, i);
    bool bad = false;
    Mat<float, DO, DO> W = cholinv(S, bad);
    Vec<float, DO> xo = mulv(W, mu);
    Mat<float, DO, DI> WA = mul(W, A);
    Mat<float, DI, DI> Win = mul_tn(A, WA);
    // symmetrise (A' W A is symmetric up to round-off)
#pragma unroll
    for (int r = 0; r < DI; ++r)
#pragma unroll
        for (int c = 0; c < r; ++c) { float s = 0.5f * (Win(r, c) + Win(c, r)); Win(r, c) = s; Win(c, r) = s; }
    st_vec<DI>(xi_in, n, i, mulv_t(A, xo));
    st_soa<DI, DI>(W_in, n, i, Win);
    if (status) status[i] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
}
// rule #5 / prod: c = a + s*b on (vector, matrix) pairs
template <int D>
__global__ void k_pair_axpy(int64_t n, const float* v1, const float* M1, const float* v2, const float* M2,
                            float sv, float* vo, float* Mo) {
    RXG_TID
    Vec<float, D> a = ld_vec<D>(v1, n, i), b = ld_vec<D>(v2, n, i);
#pragma unroll
    for (int k = 0; k < D; ++k) a.a[k] = __fmaf_rn(sv, b.a[k], a.a[k]);
    st_vec<D>(vo, n, i, a);
    st_soa<D, D>(Mo, n, i, add(ld_soa<D, D>(M1, n, i), ld_soa<D, D>(M2, n, i)));
}
// conversions: (v, M) -> (inv(M) v, inv(M))
template <int D>
__global__ void k_convert(int64_t n, const float* v, const float* M_, float* vo, float* Mo, int32_t* status) {
    RXG_TID
    bool bad = false;
    Mat<float, D, D> Mi = cholinv(ld_soa<D, D>(M_, n, i), bad);
    st_vec<D>(vo, n, i, mulv(Mi, ld_vec<D>(v, n, i)));
    st_soa<D, D>(Mo, n, i, Mi);
    if (status) status[i] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
}
struct PtrList { const float* xi[8]; const float* W[8]; };
template <int D>
__global__ void k_marginal(int64_t n, int k, PtrList pl, float* mu, float* S, int32_t* status) {
    RXG_TID
    Vec<float, D> xi = ld_vec<D>(pl.xi[0], n, i);
    Mat<float, D, D> W = ld_soa<D, D>(pl.W[0], n, i);
    for (int q = 1; q < k; ++q) {           // left-to-right fold, as the reference's MessagesProductFromLeftToRight
        Vec<float, D> x2 = ld_vec<D>(pl.xi[q], n, i);
#pragma unroll
        for (int r = 0; r < D; ++r) xi.a[r] += x2.a[r];
        W = add(W, ld_soa<D, D>(pl.W[q], n, i));
    }
    bool bad = false;
    Mat<float, D, D> Sg = cholinv(W, bad);
    st_vec<D>(mu, n, i, mulv(Sg, xi));
    st_soa<D, D>(S, n, i, Sg);
    if (status) status[i] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
}

__device__ __forceinline__ float digamma_rule(float x) {   // psi(x), x > 0: recurrence up to x >= 6, then the asymptotic series
    float r = 0.f;
    while (x < 6.f) { r -= 1.f / x; x += 1.f; }
    const float i = 1.f / x, i2 = i * i;
    return r + logf(x) - 0.5f * i - i2 * (1.f / 12.f - i2 * (1.f / 120.f - i2 * (1.f / 252.f)));
}

// ---- univariate / Gamma (rows 8-9)
__global__ void k_normal_precision_tau(int64_t n, const float* mo, const float* vo, const float* mm, const float* vm,
                                       float* shape, float* rate) {
    RXG_TID
    const float d = mo[i] - mm[i];
    shape[i] = 1.5f;
    rate[i] = 0.5f * (__fmaf_rn(d, d, vo[i]) + vm[i]);
}
__global__ void k_normal_precision_out(int64_t n, const float* mm, const float* vm, const float* shape,
                                       const float* rate, float* mo, float* vo) {
    RXG_TID
    mo[i] = mm[i];
    vo[i] = vm[i] + rate[i] / shape[i];
}
__global__ void k_prod_gamma(int64_t n, const float* a1, const float* b1, const float* a2, const float* b2,
                             float* a, float* b) {
    RXG_TID
    a[i] = a1[i] + a2[i] - 1.0f;
    b[i] = b1[i] + b2[i];
}
__global__ void k_prod_normal(int64_t n, const float* m1, const float* v1, const float* m2, const float* v2,
                              float* m, float* v) {
    RXG_TID
    const float w1 = 1.0f / v1[i], w2 = 1.0f / v2[i];
    const float w = w1 + w2;
    const float vv = 1.0f / w;
    m[i] = (m1[i] * w1 + m2[i] * w2) * vv;
    v[i] = vv;
}

// structured variant of the tau rule: q(out, mu) jointly Gaussian (m[2][n], V[2][2][n]):
// GammaShapeRate(3/2, 1/2 [V11 + V22 - V12 - V21 + (m1 - m2)^2])
__global__ void k_normal_precision_tau_joint(int64_t n, const float* m, const float* V, float* shape, float* rate) {
    RXG_TID
    const float d = m[i] - m[n + i];
    shape[i] = 1.5f;
    rate[i] = 0.5f * (__fmaf_rn(d, d, V[i] + V[3 * n + i]) - V[n + i] - V[2 * n + i]);
}

// ---- Wishart precision (multivariate twin of the Gamma rules), WishartFast parametrisation (df, inverse scale)
// @rule MvNormalMeanPrecision(:Lambda)(q_out, q_mu) -> Wishart(d + 2, inv(V_out + V_mu + (m_out - m_mu)(m_out - m_mu)'))
template <int D>
__global__ void k_mvn_precision_lambda(int64_t n, const float* mo, const float* Vo, const float* mm, const float* Vm,
                                       float* df, float* invS) {
    RXG_TID
    Vec<float, D> a = ld_vec<D>(mo, n, i), b = ld_vec<D>(mm, n, i);
    Mat<float, D, D> S = add(ld_soa<D, D>(Vo, n, i), ld_soa<D, D>(Vm, n, i));
#pragma unroll
    for (int r = 0; r < D; ++r)
#pragma unroll
        for (int c = 0; c < D; ++c) S(r, c) = __fmaf_rn(a(r) - b(r), a(c) - b(c), S(r, c));
    df[i] = (float)(D + 2);
    st_soa<D, D>(invS, n, i, S);
}
// prod(Wishart(nu1, S1), Wishart(nu2, S2)) = Wishart(nu1 + nu2 - d - 1, inv(inv(S1) + inv(S2))): adds in this parametrisation
template <int D>
__global__ void k_prod_wishart(int64_t n, const float* df1, const float* iS1, const float* df2, const float* iS2,
                               float* df, float* iS) {
    RXG_TID
    df[i] = df1[i] + df2[i] - (float)(D + 1);
    st_soa<D, D>(iS, n, i, add(ld_soa<D, D>(iS1, n, i), ld_soa<D, D>(iS2, n, i)));
}
// mean(Wishart(nu, S)) = nu S = nu inv(invS)
template <int D>
__global__ void k_wishart_mean(int64_t n, const float* df, const float* iS, float* EL, int32_t* status) {
    RXG_TID
    bool bad = false;
    Mat<float, D, D> S = cholinv(ld_soa<D, D>(iS, n, i), bad);
    const float nu = df[i];
#pragma unroll
    for (int k = 0; k < D * D; ++k) S.a[k] *= nu;
    st_soa<D, D>(EL, n, i, S);
    if (status) status[i] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
}

// Fused mean-field VMP of the reference's autoregressive regression model
//   gamma ~ Gamma(a0, b0),  theta ~ MvNormal(0, I / w0),  y[i] ~ Normal(dot(x[i], theta), 1 / gamma),  q(gamma) q(theta)
// with the regressors x[i] = (s[i-1], ..., s[i-p]) taken from the series itself
// [ref: /root/reference/test/models/autoregressive/ar_tests.jl:17-36 (model, constraints, initialisation), :7-15 (lags)].
// One thread = one series: sufficient statistics (sum x x', sum x y, sum y^2) in ONE coalesced pass over s[N][batch] with
// a p-deep sliding window in registers (fp64 accumulators); every VMP iteration is then O(p^3):
//   q(theta): Lambda = w0 I + E[gamma] Sxx,  xi = E[gamma] Sxy                  (dot(:in2) messages, product)
//   q(gamma): Gamma(a0 + n/2, b0 + 1/2 [Syy - 2 m'Sxy + m'Sxx m + tr(Sxx V)])    (NormalMeanPrecision(:tau) messages)
// Bethe free energy per iteration: E[-log p(y | theta, gamma)] + KL(q(theta) || p) + KL(q(gamma) || p).
template <int PMAX>
__global__ void __launch_bounds__(128)
ar_vmp_kernel(const float* __restrict__ series, int N, int64_t batch, int p, int iters, float a0, float b0, float w0,
              float init_a, float init_b, float* __restrict__ th_mean, float* __restrict__ th_cov,
              float* __restrict__ g_shape, float* __restrict__ g_rate, double* __restrict__ fe) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    double Sxx[PMAX][PMAX], Sxy[PMAX], Syy = 0.0;
#pragma unroll
    for (int i = 0; i < PMAX; ++i) {
        Sxy[i] = 0.0;
#pragma unroll
        for (int j = 0; j < PMAX; ++j) Sxx[i][j] = 0.0;
    }
    float win[PMAX];                                    // win[j] = s[k-1-j]
#pragma unroll
    for (int j = 0; j < PMAX; ++j) win[j] = (j < p) ? __ldg(series + (int64_t)(p - 1 - j) * batch + b) : 0.f;
    for (int k = p; k < N; ++k) {
        const float yk = __ldg(series + (int64_t)k * batch + b);
        Syy += (double)yk * (double)yk;
#pragma unroll
        for (int i = 0; i < PMAX; ++i) {
            Sxy[i] += (double)win[i] * (double)yk;
#pragma unroll
            for (int j = 0; j <= i; ++j) Sxx[i][j] += (double)win[i] * (double)win[j];
        }
#pragma unroll
        for (int j = PMAX - 1; j > 0; --j) win[j] = (j < p) ? win[j - 1] : 0.f;
        win[0] = yk;
    }
#pragma unroll
    for (int i = 0; i < PMAX; ++i)
#pragma unroll
        for (int j = i + 1; j < PMAX; ++j) Sxx[i][j] = Sxx[j][i];
    const int n = N - p;
    double ga = (double)init_a, gb = (double)init_b;
    double m[PMAX], V[PMAX][PMAX];
    for (int it = 0; it < iters; ++it) {
        const double Eg = ga / gb;
        // Lambda = w0 I + Eg Sxx = L L' ; V = Lambda^-1 ; m = V (Eg Sxy)
        double L[PMAX][PMAX];
#pragma unroll
        for (int i = 0; i < PMAX; ++i)
#pragma unroll
            for (int j = 0; j < PMAX; ++j) L[i][j] = (i < p && j < p) ? Eg * Sxx[i][j] + (i == j ? (double)w0 : 0.0) : (i == j ? 1.0 : 0.0);
        double logdetL = 0.0;
#pragma unroll
        for (int j = 0; j < PMAX; ++j) {
            double dj = L[j][j];
#pragma unroll
            for (int k = 0; k < j; ++k) dj -= L[j][k] * L[j][k];
            dj = sqrt(dj > 0.0 ? dj : 1e-300);
            L[j][j] = dj;
            logdetL += log(dj);
#pragma unroll
            for (int i = j + 1; i < PMAX; ++i) {
                double sv = L[i][j];
#pragma unroll
                for (int k = 0; k < j; ++k) sv -= L[i][k] * L[j][k];
                L[i][j] = sv / dj;
            }
        }
        // Li = L^-1 (lower), V = Li' Li
        double Li[PMAX][PMAX];
#pragma unroll
        for (int i = 0; i < PMAX; ++i)
#pragma unroll
            for (int j = 0; j < PMAX; ++j) Li[i][j] = 0.0;
#pragma unroll
        for (int j = 0; j < PMAX; ++j) {
            Li[j][j] = 1.0 / L[j][j];
#pragma unroll
            for (int i = j + 1; i < PMAX; ++i) {
                double sv = 0.0;
#pragma unroll
                for (int k = j; k < i; ++k) sv -= L[i][k] * Li[k][j];
                Li[i][j] = sv / L[i][i];
            }
        }
#pragma unroll
        for (int i = 0; i < PMAX; ++i)
#pragma unroll
            for (int j = 0; j < PMAX; ++j) {
                double sv = 0.0;
#pragma unroll
                for (int k = 0; k < PMAX; ++k) sv += Li[k][i] * Li[k][j];
                V[i][j] = sv;
            }
#pragma unroll
        for (int i = 0; i < PMAX; ++i) {
            double sv = 0.0;
#pragma unroll
            for (int j = 0; j < PMAX; ++j) sv += V[i][j] * ((j < p) ? Eg * Sxy[j] : 0.0);
            m[i] = (i < p) ? sv : 0.0;
        }
        // residual: sum_i E(y_i - x_i' theta)^2
        double res = Syy, trSV = 0.0, mm = 0.0, trV = 0.0;
#pragma unroll
        for (int i = 0; i < PMAX; ++i) {
            if (i < p) {
                res -= 2.0 * m[i] * Sxy[i];
                mm += m[i] * m[i];
                trV += V[i][i];
#pragma unroll
                for (int j = 0; j < PMAX; ++j)
                    if (j < p) { res += m[i] * Sxx[i][j] * m[j]; trSV += Sxx[i][j] * V[j][i]; }
            }
        }
        res += trSV;
        ga = (double)a0 + 0.5 * n;
        gb = (double)b0 + 0.5 * res;
        if (fe) {
            double dig = 0.0, xx = ga;                       // psi(x) in fp64: recurrence to x >= 6, then the asymptotic series
            while (xx < 6.0) { dig -= 1.0 / xx; xx += 1.0; }
            { const double i1 = 1.0 / xx, i2 = i1 * i1; dig += log(xx) - 0.5 * i1 - i2 * (1.0 / 12.0 - i2 * (1.0 / 120.0 - i2 * (1.0 / 252.0 - i2 * (1.0 / 240.0)))); }
            const double Elog = dig - log(gb), Egn = ga / gb;
            const double like = 0.5 * n * (1.8378770664093453 - Elog) + 0.5 * Egn * res;
            // KL(N(m, V) || N(0, I / w0)) = 1/2 [w0 (tr V + m'm) - p - p log w0 - log det V],  log det V = -2 log det L
            const double klt = 0.5 * ((double)w0 * (trV + mm) - p - p * log((double)w0) + 2.0 * logdetL);
            const double klg = (ga - a0) * dig - lgamma(ga) + lgamma((double)a0) + a0 * (log(gb) - log((double)b0)) + ga * ((double)b0 - gb) / gb;
            fe[(int64_t)it * batch + b] = like + klt + klg;      // fp64: the reference asserts decreases of 1e-5 on values of 1.4e3
        }
    }
    for (int i = 0; i < p; ++i) {
        th_mean[(int64_t)i * batch + b] = (float)m[i];
        for (int j = 0; j < p; ++j) th_cov[((int64_t)i * p + j) * batch + b] = (float)V[i][j];
    }
    g_shape[b] = (float)ga; g_rate[b] = (float)gb;
}

// Fused mean-field VMP of the multivariate IID model with unknown mean and precision
//   m ~ MvNormal(mu0, Lambda0^-1),  P ~ Wishart(nu0, S0),  y_i ~ MvNormal(m, P^-1),  q(m, P) = q(m) q(P)
// [ref: /root/reference/test/models/iid/mv_iid_precision_tests.jl:10-41].  One thread = one dataset: the sufficient
// statistics (sum y, sum y y') are accumulated in ONE coalesced pass over y[N][d][batch]; every VMP iteration is then
// O(d^3) in registers:   q(m): Lambda = Lambda0 + N E[P],  xi = Lambda0 mu0 + E[P] sum y
//                        q(P): Wishart(nu0 + N, inv(inv(S0) + sum_i [(y_i - m)(y_i - m)' + V_m]))
template <int D>
__global__ void __launch_bounds__(128)
mv_iid_wishart_vmp_kernel(const float* __restrict__ y, int N, int64_t batch, int iters, const float* __restrict__ prior,
                          float* __restrict__ m_out, float* __restrict__ V_out, float* __restrict__ df_out,
                          float* __restrict__ iS_out, int32_t* __restrict__ status) {
    // prior (device, row-major): mu0[D], Lambda0[D*D], nu0, invS0[D*D], E[P] of the initial q(P) [D*D]
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    Vec<double, D> sy;
    Mat<double, D, D> syy;
#pragma unroll
    for (int i = 0; i < D; ++i) sy(i) = 0.0;
#pragma unroll
    for (int i = 0; i < D * D; ++i) syy.a[i] = 0.0;
    for (int t = 0; t < N; ++t) {
        float v[D];
#pragma unroll
        for (int i = 0; i < D; ++i) v[i] = __ldg(y + ((int64_t)t * D + i) * batch + b);
#pragma unroll
        for (int i = 0; i < D; ++i) {
            sy(i) += (double)v[i];
#pragma unroll
            for (int j = 0; j <= i; ++j) syy(i, j) += (double)v[i] * (double)v[j];
        }
    }
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = i + 1; j < D; ++j) syy(i, j) = syy(j, i);
    Vec<double, D> mu0;
    Mat<double, D, D> L0, iS0, EP;
#pragma unroll
    for (int i = 0; i < D; ++i) mu0(i) = (double)prior[i];
#pragma unroll
    for (int i = 0; i < D * D; ++i) { L0.a[i] = (double)prior[D + i]; iS0.a[i] = (double)prior[D + D * D + 1 + i]; EP.a[i] = (double)prior[D + 2 * D * D + 1 + i]; }
    const double nu0 = (double)prior[D + D * D];
    const Vec<double, D> xi0 = mulv(L0, mu0);
    bool bad = false;
    Vec<double, D> m;
    Mat<double, D, D> Vm, iS;
    const double nu = nu0 + (double)N;
    for (int it = 0; it < iters; ++it) {
        // q(m)
        Mat<double, D, D> Lm;
#pragma unroll
        for (int i = 0; i < D * D; ++i) Lm.a[i] = L0.a[i] + (double)N * EP.a[i];
        Vm = cholinv(Lm, bad);
        Vec<double, D> xi = mulv(EP, sy);
#pragma unroll
        for (int i = 0; i < D; ++i) xi(i) += xi0(i);
        m = mulv(Vm, xi);
        // q(P): inverse scale = invS0 + sum (y - m)(y - m)' + N V_m = invS0 + syy - sy m' - m sy' + N (m m' + V_m)
#pragma unroll
        for (int i = 0; i < D; ++i)
#pragma unroll
            for (int j = 0; j < D; ++j)
                iS(i, j) = iS0(i, j) + syy(i, j) - sy(i) * m(j) - m(i) * sy(j) + (double)N * (m(i) * m(j) + Vm(i, j));
        Mat<double, D, D> S = cholinv(iS, bad);
#pragma unroll
        for (int i = 0; i < D * D; ++i) EP.a[i] = nu * S.a[i];
    }
#pragma unroll
    for (int i = 0; i < D; ++i) m_out[(int64_t)i * batch + b] = (float)m(i);
#pragma unroll
    for (int i = 0; i < D * D; ++i) { V_out[(int64_t)i * batch + b] = (float)Vm.a[i]; iS_out[(int64_t)i * batch + b] = (float)iS.a[i]; }
    df_out[b] = (float)nu;
    if (status) status[b] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
}

}  // namespace rxg

using namespace rxg;

static inline unsigned nblk(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

#define RXG_RULE_PROLOGUE(ctx, n)                                                     \
    if (!(ctx)) return RXG_ERR_BAD_ARG;                                               \
    if ((n) < 0) return rxg::fail((ctx), RXG_ERR_BAD_ARG, "n < 0");                   \
    if (!((flags) & RXG_PTR_DEVICE))                                                  \
        return rxg::fail((ctx), RXG_ERR_UNSUPPORTED,                                  \
                         "per-rule kernels take device pointers (set RXG_PTR_DEVICE)"); \
    if ((n) == 0) return RXG_OK;                                                      \
    RXG_CUDA((ctx), cudaSetDevice((ctx)->device));

#define RXG_RULE_EPILOGUE(ctx, what)                                                  \
    (ctx)->launches += 1;                                                             \
    {                                                                                 \
        int _rc = rxg::check_cuda((ctx), cudaGetLastError(), what);                   \
        if (_rc != RXG_OK) return _rc;                                                \
    }                                                                                 \
    if (!(flags & RXG_ASYNC)) RXG_CUDA((ctx), cudaStreamSynchronize((ctx)->stream));  \
    return RXG_OK;

// state sizes without a register-resident instantiation go to csrc/rxg_rules_large.cu (any d <= 64)
#define RXG_LARGE_D(ctx, d, CALL, what)                                                                   \
    if (!rxg::rules_small(d)) {                                                                           \
        if ((d) < 1 || (d) > 64) return rxg::fail((ctx), RXG_ERR_UNSUPPORTED, "rule kernels: d=%d unsupported (1-64)", (d)); \
        { int _rc = (CALL); if (_rc != RXG_OK) return _rc; }                                              \
        (ctx)->launches -= 1;                                                                             \
        RXG_RULE_EPILOGUE(ctx, what)                                                                      \
    }

#define RXG_DISPATCH_D(d, CALL)                                                        \
    switch (d) {                                                                       \
        case 1: { constexpr int D = 1; CALL; } break;                                  \
        case 2: { constexpr int D = 2; CALL; } break;                                  \
        case 3: { constexpr int D = 3; CALL; } break;                                  \
        case 4: { constexpr int D = 4; CALL; } break;                                  \
        case 5: { constexpr int D = 5; CALL; } break;                                  \
        case 6: { constexpr int D = 6; CALL; } break;                                  \
        case 8: { constexpr int D = 8; CALL; } break;                                  \
        default: return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "rule kernels: d=%d unsupported (1-6, 8)", d); \
    }

#define RXG_DISPATCH_DODI(dout, din, CALL)                                             \
    switch ((dout) * 16 + (din)) {                                                     \
        case 1 * 16 + 1: { constexpr int DO = 1, DI = 1; CALL; } break;                \
        case 1 * 16 + 2: { constexpr int DO = 1, DI = 2; CALL; } break;                \
        case 2 * 16 + 2: { constexpr int DO = 2, DI = 2; CALL; } break;                \
        case 3 * 16 + 3: { constexpr int DO = 3, DI = 3; CALL; } break;                \
        case 1 * 16 + 4: { constexpr int DO = 1, DI = 4; CALL; } break;                \
        case 2 * 16 + 4: { constexpr int DO = 2, DI = 4; CALL; } break;                \
        case 4 * 16 + 4: { constexpr int DO = 4, DI = 4; CALL; } break;                \
        case 6 * 16 + 6: { constexpr int DO = 6, DI = 6; CALL; } break;                \
        case 8 * 16 + 8: { constexpr int DO = 8, DI = 8; CALL; } break;                \
        default: return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "rule kernels: A is %dx%d, unsupported", dout, din); \
    }

extern "C" {

int rxg_rule_mvnormal_meancov_out_f32(rxg_ctx* ctx, int64_t n, int d, const float* mu_in, const float* S_in,
                                      const float* Sigma, int M_shared, float* mu_out, float* S_out,
                                      unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_LARGE_D(ctx, d, rxg::rules_large_add_cov(ctx, n, d, mu_in, S_in, Sigma, M_shared, mu_out, S_out), "rules_large_add_cov")
    RXG_DISPATCH_D(d, (k_add_cov<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, mu_in, S_in, Sigma, M_shared, mu_out, S_out)))
    RXG_RULE_EPILOGUE(ctx, "k_add_cov")
}
int rxg_rule_mvnormal_meancov_mean_f32(rxg_ctx* ctx, int64_t n, int d, const float* mu_in, const float* S_in,
                                       const float* Sigma, int M_shared, float* mu_out, float* S_out,
                                       unsigned flags) {
    return rxg_rule_mvnormal_meancov_out_f32(ctx, n, d, mu_in, S_in, Sigma, M_shared, mu_out, S_out, flags);
}
int rxg_rule_mvnormal_meancov_mean_data_f32(rxg_ctx* ctx, int64_t n, int d, const float* y, const float* Sigma,
                                            int M_shared, float* mu_out, float* S_out, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_LARGE_D(ctx, d, rxg::rules_large_add_cov(ctx, n, d, y, nullptr, Sigma, M_shared, mu_out, S_out), "rules_large_from_data")
    RXG_DISPATCH_D(d, (k_from_data<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, y, Sigma, M_shared, mu_out, S_out)))
    RXG_RULE_EPILOGUE(ctx, "k_from_data")
}
int rxg_rule_mul_out_f32(rxg_ctx* ctx, int64_t n, int d_out, int d_in, const float* A, int M_shared,
                         const float* mu_in, const float* S_in, float* mu_out, float* S_out, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    if (!rxg::rules_small2(d_out, d_in)) {
        if (d_out < 1 || d_out > 64 || d_in < 1 || d_in > 64) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "mul_out: A is %dx%d, unsupported (1-64)", d_out, d_in);
        if (!M_shared) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "mul_out: a per-message A needs one of the register-resident shapes (A %dx%d)", d_out, d_in);
        { int _rc = rxg::rules_large_mul_out(ctx, n, d_out, d_in, A, mu_in, S_in, mu_out, S_out); if (_rc != RXG_OK) return _rc; }
        ctx->launches -= 1;
        RXG_RULE_EPILOGUE(ctx, "rules_large_mul_out")
    }
    RXG_DISPATCH_DODI(d_out, d_in, (k_mul_out<DO, DI><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, A, M_shared, mu_in, S_in, mu_out, S_out)))
    RXG_RULE_EPILOGUE(ctx, "k_mul_out")
}
int rxg_rule_mul_in_f32(rxg_ctx* ctx, int64_t n, int d_out, int d_in, const float* A, int M_shared,
                        const float* mu_out, const float* S_out, float* xi_in, float* W_in, int32_t* status,
                        unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    if (!rxg::rules_small2(d_out, d_in)) {
        if (d_out < 1 || d_out > 64 || d_in < 1 || d_in > 64) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "mul_in: A is %dx%d, unsupported (1-64)", d_out, d_in);
        if (!M_shared) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "mul_in: a per-message A needs one of the register-resident shapes (A %dx%d)", d_out, d_in);
        { int _rc = rxg::rules_large_mul_in(ctx, n, d_out, d_in, A, mu_out, S_out, xi_in, W_in, status); if (_rc != RXG_OK) return _rc; }
        ctx->launches -= 1;
        RXG_RULE_EPILOGUE(ctx, "rules_large_mul_in")
    }
    RXG_DISPATCH_DODI(d_out, d_in, (k_mul_in<DO, DI><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, A, M_shared, mu_out, S_out, xi_in, W_in, status)))
    RXG_RULE_EPILOGUE(ctx, "k_mul_in")
}
int rxg_rule_add_out_f32(rxg_ctx* ctx, int64_t n, int d, const float* mu1, const float* S1, const float* mu2,
                         const float* S2, float* mu_out, float* S_out, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_LARGE_D(ctx, d, rxg::rules_large_pair_axpy(ctx, n, d, mu1, S1, mu2, S2, 1.0f, mu_out, S_out), "rules_large_add_out")
    RXG_DISPATCH_D(d, (k_pair_axpy<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, mu1, S1, mu2, S2, 1.0f, mu_out, S_out)))
    RXG_RULE_EPILOGUE(ctx, "k_pair_axpy(add_out)")
}
int rxg_rule_add_in_f32(rxg_ctx* ctx, int64_t n, int d, const float* mu_out, const float* S_out,
                        const float* mu_other, const float* S_other, float* mu_in, float* S_in, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_LARGE_D(ctx, d, rxg::rules_large_pair_axpy(ctx, n, d, mu_out, S_out, mu_other, S_other, -1.0f, mu_in, S_in), "rules_large_add_in")
    RXG_DISPATCH_D(d, (k_pair_axpy<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, mu_out, S_out, mu_other, S_other, -1.0f, mu_in, S_in)))
    RXG_RULE_EPILOGUE(ctx, "k_pair_axpy(add_in)")
}
int rxg_prod_gaussian_f32(rxg_ctx* ctx, int64_t n, int d, const float* xi1, const float* W1, const float* xi2,
                          const float* W2, float* xi, float* W, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_LARGE_D(ctx, d, rxg::rules_large_pair_axpy(ctx, n, d, xi1, W1, xi2, W2, 1.0f, xi, W), "rules_large_prod")
    RXG_DISPATCH_D(d, (k_pair_axpy<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, xi1, W1, xi2, W2, 1.0f, xi, W)))
    RXG_RULE_EPILOGUE(ctx, "k_pair_axpy(prod)")
}
int rxg_meancov_to_wmp_f32(rxg_ctx* ctx, int64_t n, int d, const float* mu, const float* S, float* xi, float* W,
                           int32_t* status, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_LARGE_D(ctx, d, rxg::rules_large_convert(ctx, n, d, 1, &mu, &S, xi, W, status), "rules_large_convert")
    RXG_DISPATCH_D(d, (k_convert<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, mu, S, xi, W, status)))
    RXG_RULE_EPILOGUE(ctx, "k_convert")
}
int rxg_wmp_to_meancov_f32(rxg_ctx* ctx, int64_t n, int d, const float* xi, const float* W, float* mu, float* S,
                           int32_t* status, unsigned flags) {
    return rxg_meancov_to_wmp_f32(ctx, n, d, xi, W, mu, S, status, flags);
}
int rxg_marginal_gaussian_f32(rxg_ctx* ctx, int64_t n, int d, int k, const float* const* xi_list,
                              const float* const* W_list, float* mu, float* S, int32_t* status, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    if (k < 1 || k > 8) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "marginal: k=%d must be in 1..8", k);
    RXG_LARGE_D(ctx, d, rxg::rules_large_convert(ctx, n, d, k, xi_list, W_list, mu, S, status), "rules_large_marginal")
    PtrList pl = {};
    for (int q = 0; q < k; ++q) { pl.xi[q] = xi_list[q]; pl.W[q] = W_list[q]; }
    RXG_DISPATCH_D(d, (k_marginal<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, k, pl, mu, S, status)))
    RXG_RULE_EPILOGUE(ctx, "k_marginal")
}
int rxg_rule_normal_precision_tau_f32(rxg_ctx* ctx, int64_t n, const float* m_out, const float* v_out,
                                      const float* m_mu, const float* v_mu, float* shape, float* rate,
                                      unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    k_normal_precision_tau<<<nblk(n, 256), 256, 0, ctx->stream>>>(n, m_out, v_out, m_mu, v_mu, shape, rate);
    RXG_RULE_EPILOGUE(ctx, "k_normal_precision_tau")
}
int rxg_rule_normal_precision_out_f32(rxg_ctx* ctx, int64_t n, const float* m_mu, const float* v_mu,
                                      const float* shape, const float* rate, float* m_out, float* v_out,
                                      unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    k_normal_precision_out<<<nblk(n, 256), 256, 0, ctx->stream>>>(n, m_mu, v_mu, shape, rate, m_out, v_out);
    RXG_RULE_EPILOGUE(ctx, "k_normal_precision_out")
}
int rxg_prod_gamma_f32(rxg_ctx* ctx, int64_t n, const float* a1, const float* b1, const float* a2, const float* b2,
                       float* a, float* b, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    k_prod_gamma<<<nblk(n, 256), 256, 0, ctx->stream>>>(n, a1, b1, a2, b2, a, b);
    RXG_RULE_EPILOGUE(ctx, "k_prod_gamma")
}
int rxg_rule_normal_precision_tau_joint_f32(rxg_ctx* ctx, int64_t n, const float* m_joint, const float* V_joint,
                                            float* shape, float* rate, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    k_normal_precision_tau_joint<<<nblk(n, 256), 256, 0, ctx->stream>>>(n, m_joint, V_joint, shape, rate);
    RXG_RULE_EPILOGUE(ctx, "k_normal_precision_tau_joint")
}
int rxg_rule_mvnormal_precision_lambda_f32(rxg_ctx* ctx, int64_t n, int d, const float* m_out, const float* V_out,
                                           const float* m_mu, const float* V_mu, float* df, float* inv_scale,
                                           unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_DISPATCH_D(d, (k_mvn_precision_lambda<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, m_out, V_out, m_mu, V_mu, df, inv_scale)))
    RXG_RULE_EPILOGUE(ctx, "k_mvn_precision_lambda")
}
int rxg_prod_wishart_f32(rxg_ctx* ctx, int64_t n, int d, const float* df1, const float* inv_scale1, const float* df2,
                         const float* inv_scale2, float* df, float* inv_scale, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_DISPATCH_D(d, (k_prod_wishart<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, df1, inv_scale1, df2, inv_scale2, df, inv_scale)))
    RXG_RULE_EPILOGUE(ctx, "k_prod_wishart")
}
int rxg_wishart_mean_f32(rxg_ctx* ctx, int64_t n, int d, const float* df, const float* inv_scale, float* mean,
                         int32_t* status, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    RXG_DISPATCH_D(d, (k_wishart_mean<D><<<nblk(n, 128), 128, 0, ctx->stream>>>(n, df, inv_scale, mean, status)))
    RXG_RULE_EPILOGUE(ctx, "k_wishart_mean")
}
int rxg_mv_iid_wishart_vmp_f32(rxg_ctx* ctx, int d, int N, int64_t batch, int iterations, const float* mu0,
                               const float* Lambda0, float nu0, const float* inv_scale0, const float* init_E_P,
                               const float* y, float* m_mean, float* m_cov, float* df, float* inv_scale,
                               int32_t* status, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "mv_iid_wishart_vmp takes device pointers");
    if (d < 1 || N < 1 || batch < 1 || iterations < 1 || !mu0 || !Lambda0 || !inv_scale0 || !init_E_P || !y || !m_mean ||
        !m_cov || !df || !inv_scale)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "mv_iid_wishart_vmp: bad argument");
    if (d > 6) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "mv_iid_wishart_vmp: d=%d unsupported (1-6)", d);
    if (!(nu0 > (float)(d - 1)))                        // a proper Wishart prior, as the LGSSM Wishart entries require
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "mv_iid_wishart_vmp: nu0 must exceed d - 1");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    // prior block (host) -> device workspace: mu0[d], Lambda0[d*d], nu0, invS0[d*d], E[P]_init[d*d]
    const int dd = d * d;
    float hp[6 + 3 * 36 + 1];
    for (int i = 0; i < d; ++i) hp[i] = mu0[i];
    for (int i = 0; i < dd; ++i) { hp[d + i] = Lambda0[i]; hp[d + dd + 1 + i] = inv_scale0[i]; hp[d + 2 * dd + 1 + i] = init_E_P[i]; }
    hp[d + dd] = nu0;
    float* dp = (float*)rxg::workspace(ctx, sizeof(hp));
    if (!dp) return RXG_ERR_CUDA;
    RXG_CUDA(ctx, cudaMemcpyAsync(dp, hp, (size_t)(d + 3 * dd + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    const unsigned grid = (unsigned)((batch + 127) / 128);
    switch (d) {
#define RXG_WISH(DD) case DD: mv_iid_wishart_vmp_kernel<DD><<<grid, 128, 0, ctx->stream>>>(y, N, batch, iterations, dp, m_mean, m_cov, df, inv_scale, status); break;
        RXG_WISH(1) RXG_WISH(2) RXG_WISH(3) RXG_WISH(4) RXG_WISH(5) RXG_WISH(6)
#undef RXG_WISH
    }
    RXG_RULE_EPILOGUE(ctx, "mv_iid_wishart_vmp_kernel")
}
int rxg_ar_vmp_f32(rxg_ctx* ctx, int order, int N, int64_t batch, int iterations, float a0, float b0, float theta_prior_precision,
                   float init_shape, float init_rate, const float* series, float* theta_mean, float* theta_cov,
                   float* gamma_shape, float* gamma_rate, double* free_energy, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "ar_vmp takes device pointers");
    if (order < 1 || order > 8) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "ar_vmp: order=%d unsupported (1-8)", order);
    if (N <= order || batch < 1 || iterations < 1 || !series || !theta_mean || !theta_cov || !gamma_shape || !gamma_rate ||
        !(a0 > 0.f) || !(b0 > 0.f) || !(theta_prior_precision > 0.f) || !(init_shape > 0.f) || !(init_rate > 0.f))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "ar_vmp: bad argument");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const unsigned grid = (unsigned)((batch + 127) / 128);
    if (order <= 4)
        ar_vmp_kernel<4><<<grid, 128, 0, ctx->stream>>>(series, N, batch, order, iterations, a0, b0, theta_prior_precision, init_shape,
                                                        init_rate, theta_mean, theta_cov, gamma_shape, gamma_rate, free_energy);
    else
        ar_vmp_kernel<8><<<grid, 128, 0, ctx->stream>>>(series, N, batch, order, iterations, a0, b0, theta_prior_precision, init_shape,
                                                        init_rate, theta_mean, theta_cov, gamma_shape, gamma_rate, free_energy);
    RXG_RULE_EPILOGUE(ctx, "ar_vmp_kernel")
}
int rxg_prod_normal_f32(rxg_ctx* ctx, int64_t n, const float* m1, const float* v1, const float* m2, const float* v2,
                        float* m, float* v, unsigned flags) {
    RXG_RULE_PROLOGUE(ctx, n)
    k_prod_normal<<<nblk(n, 256), 256, 0, ctx->stream>>>(n, m1, v1, m2, v2, m, v);
    RXG_RULE_EPILOGUE(ctx, "k_prod_normal")
}

}  // extern "C"
