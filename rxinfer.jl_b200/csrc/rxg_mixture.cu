// Fused mean-field VMP of the Gaussian mixture model, `batch` independent data sets, all iterations in one launch
// [ref: test/models/mixtures/gmm_multivariate_tests.jl:4-24 (K = 3, d = 2) and gmm_univariate_tests.jl:6-20 (K = 2,
// d = 1, the Beta / Bernoulli / Gamma spelling of the same model)]:
//   s ~ Dirichlet(alpha0);  m[k] ~ MvNormal(mu0[k], V0[k]);  W[k] ~ Wishart(nu0[k], S0[k]);
//   z[i] ~ Categorical(s);  y[i] ~ NormalMixture(z[i], m, W);  q = q(s) prod q(m[k]) prod q(W[k]) prod q(z[i]).
// One thread = one data set.  Every iteration is one coalesced pass over y[N][d][batch] (batch innermost): the
// responsibilities r[i][k] from the previous q(s), q(m), q(W), then the per-component statistics N_k, sum r (y - c_k),
// sum r (y - c_k)(y - c_k)' accumulated in fp64 around c_k = the previous E[m_k] (the points sit near their cluster's
// mean, so nothing cancels when the data are far from the origin), then the O(K d^3) conjugate updates in fp64 in the
// order q(m) (previous E[W]), q(W) (new q(m)), q(s) (DESIGN 3.17), then the Bethe free energy in fp64.
// Shared memory per thread, laid out [slot][thread]: the fp64 accumulators and the fp32 per-component constants the
// data pass reads (centre, packed E[W], log-weight offset).  At K = 8, d = 4 that is 120 + 120 slots.
#include <cfloat>
#include <cmath>

#include "rxg_internal.h"
#include "rxg_linalg.cuh"

namespace rxg {
namespace gmm {

constexpr int TPB = 64;                       // threads (chains) per block
constexpr double LOG2PI = 1.8378770664093453;
constexpr double LOGPI = 1.1447298858494002;

__host__ __device__ constexpr int packed(int d) { return d * (d + 1) / 2; }
__host__ __device__ constexpr int acc_slots(int d) { return 1 + d + packed(d); }      // N_k, b_k, C_k (lower)
__host__ __device__ constexpr int st_slots(int d) { return d + packed(d) + 1; }       // c_k, E[W_k] (lower), cst_k

// fp64 host constants, per component k (block of blk(d) doubles), then two global values
struct Layout {
    int mu0, V0i, xi0, ldV0, S0i, ldS0, nu0, a0, lgd0, ai, mi, Vi, nui, iSi, blk;
};
__host__ __device__ constexpr Layout layout(int d) {
    const int dd = d * d;
    return Layout{0, d, d + dd, 2 * d + dd, 2 * d + dd + 1, 2 * d + 2 * dd + 1, 2 * d + 2 * dd + 2, 2 * d + 2 * dd + 3,
                  2 * d + 2 * dd + 4, 2 * d + 2 * dd + 5, 2 * d + 2 * dd + 6, 3 * d + 2 * dd + 6, 3 * d + 3 * dd + 6,
                  3 * d + 3 * dd + 7, 3 * d + 4 * dd + 7};
}
// after the K blocks: sum(alpha0), lgamma(sum alpha0) - sum lgamma(alpha0)

__device__ __forceinline__ double digamma(double x) {      // psi(x), x > 0: recurrence up to x >= 10, asymptotic series
    double r = 0.0;
    while (x < 10.0) { r -= 1.0 / x; x += 1.0; }
    const double i = 1.0 / x, i2 = i * i;
    return r + log(x) - 0.5 * i - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252 - i2 * (1.0 / 240 - i2 * (1.0 / 132)))));
}
template <int D>
__host__ __device__ inline double lgamma_mv(double a) {   // log Gamma_D(a)
    double s = 0.25 * D * (D - 1) * LOGPI;
    for (int i = 0; i < D; ++i) s += lgamma(a - 0.5 * i);
    return s;
}

struct Out {
    float *alpha, *m_mean, *m_cov, *w_df, *w_inv_scale;
    double* free_energy;
    float* z_prob;
    float *h_alpha, *h_m_mean, *h_m_cov, *h_w_df, *h_w_inv_scale;
    int32_t* status;
};

// inv(A) and log|A| of an SPD matrix from one Cholesky factorisation (cholinv's inverse, rxg_linalg.cuh)
template <int D>
__device__ __forceinline__ Mat<double, D, D> inv_logdet(const Mat<double, D, D>& A, double& logdet, bool& bad) {
    const Chol<double, D> c = cholesky<double, D, true>(A, bad);
    logdet = -2.0 * c.neg_half_logdet;
    Mat<double, D, D> Li;                                   // L^-1 (lower), column by column
#pragma unroll
    for (int i = 0; i < D * D; ++i) Li.a[i] = 0.0;
#pragma unroll
    for (int j = 0; j < D; ++j) {
        Li(j, j) = c.L(j, j);
#pragma unroll
        for (int i = j + 1; i < D; ++i) {
            double s = 0.0;
#pragma unroll
            for (int k = j; k < i; ++k) s = fma(-c.L(i, k), Li(k, j), s);
            Li(i, j) = s * c.L(i, i);
        }
    }
    Mat<double, D, D> o;                                    // L^-T L^-1
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) {
            double s = 0.0;
#pragma unroll
            for (int k = i; k < D; ++k) s = fma(Li(k, i), Li(k, j), s);
            o(i, j) = s;
            o(j, i) = s;
        }
    return o;
}

// From q(m_k) = N(m, Vm) and q(W_k) = Wishart(nu, inv(iS)): the fp32 constants of the data pass (without the
// E[log s_k] term, added once every alpha is known); returns E[log|W_k|].
template <int D>
__device__ __forceinline__ double derive(const Vec<double, D>& m, const Mat<double, D, D>& Vm, double nu,
                                         const Mat<double, D, D>& iS, float* st, int tid, bool& bad,
                                         Mat<double, D, D>& EW) {
    double ldiS;
    const Mat<double, D, D> S = inv_logdet(iS, ldiS, bad);
    double elog = D * 0.6931471805599453 - ldiS;                              // log|S| = -log|iS|
    for (int i = 0; i < D; ++i) elog += digamma(0.5 * (nu - i));
    double tr = 0.0;
#pragma unroll
    for (int i = 0; i < D * D; ++i) { EW.a[i] = nu * S.a[i]; tr += EW.a[i] * Vm.a[i]; }
#pragma unroll
    for (int i = 0; i < D; ++i) st[i * TPB + tid] = (float)m(i);
    int p = D;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j, ++p) st[p * TPB + tid] = (float)((i == j ? 1.0 : 2.0) * EW(i, j));   // off-diagonal doubled
    st[p * TPB + tid] = (float)(0.5 * elog - 0.5 * D * LOG2PI - 0.5 * tr);
    return elog;
}

template <int D, int K>
__global__ void __launch_bounds__(TPB)
gmm_vmp_kernel(const float* __restrict__ y, int N, int64_t batch, int iters, const double* __restrict__ prm, Out o) {
    constexpr int P = packed(D), SA = acc_slots(D), SS = st_slots(D);
    constexpr Layout LY = layout(D);
    extern __shared__ double smem[];
    double* acc = smem;                                        // [K * SA][TPB]
    float* st = reinterpret_cast<float*>(smem + K * SA * TPB); // [K * SS][TPB]
    const int tid = threadIdx.x;
    const int64_t b = (int64_t)blockIdx.x * TPB + tid;
    if (b >= batch) return;
    bool bad = false;
    const double sum_a0 = prm[K * LY.blk], lg_dir0 = prm[K * LY.blk + 1];

    // initial q(s), q(m), q(W) -> constants of the first data pass
    {
        double sa = 0.0;
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            const double* pk = prm + k * LY.blk;
            Vec<double, D> m;
            Mat<double, D, D> Vm, iS, EW;
            for (int i = 0; i < D; ++i) m(i) = pk[LY.mi + i];
            for (int i = 0; i < D * D; ++i) { Vm.a[i] = pk[LY.Vi + i]; iS.a[i] = pk[LY.iSi + i]; }
            derive<D>(m, Vm, pk[LY.nui], iS, st + k * SS * TPB, tid, bad, EW);
            sa += pk[LY.ai];
        }
        const double psa = digamma(sa);
#pragma unroll 1
        for (int k = 0; k < K; ++k)
            st[(k * SS + SS - 1) * TPB + tid] += (float)(digamma(prm[k * LY.blk + LY.ai]) - psa);
    }

    for (int it = 0; it < iters; ++it) {
        const bool last = it == iters - 1;
#pragma unroll
        for (int j = 0; j < K * SA; ++j) acc[j * TPB + tid] = 0.0;
        double Hz = 0.0;                                       // sum_i H[q(z_i)]
        // ---- q(z): one pass over the data
        for (int t = 0; t < N; ++t) {
            float v[D];
#pragma unroll
            for (int i = 0; i < D; ++i) v[i] = __ldg(y + ((int64_t)t * D + i) * batch + b);
            float lr[K], dl[K][D];
            float mx = -FLT_MAX;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const float* sk = st + k * SS * TPB + tid;
#pragma unroll
                for (int i = 0; i < D; ++i) dl[k][i] = v[i] - sk[i * TPB];
                float q = 0.f;
                int p = D;
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    float row = 0.f;
#pragma unroll
                    for (int j = 0; j <= i; ++j, ++p) row = __fmaf_rn(sk[p * TPB], dl[k][j], row);
                    q = __fmaf_rn(row, dl[k][i], q);
                }
                lr[k] = __fmaf_rn(-0.5f, q, sk[(SS - 1) * TPB]);
                mx = fmaxf(mx, lr[k]);
            }
            float se = 0.f;
#pragma unroll
            for (int k = 0; k < K; ++k) { lr[k] -= mx; se += expf(lr[k]); }
            const float lse = logf(se);
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const float lrk = lr[k] - lse;
                const float r = expf(lrk);
                if (last && o.z_prob) o.z_prob[((int64_t)t * K + k) * batch + b] = r;
                if (r > 0.f) Hz -= (double)r * (double)lrk;
                double* ak = acc + k * SA * TPB + tid;
                ak[0] += (double)r;
                int p = 1 + D;
#pragma unroll
                for (int i = 0; i < D; ++i) {
                    const double rd = (double)r * (double)dl[k][i];
                    ak[(1 + i) * TPB] += rd;
#pragma unroll
                    for (int j = 0; j <= i; ++j, ++p) ak[p * TPB] = fma(rd, (double)dl[k][j], ak[p * TPB]);
                }
            }
        }
        // ---- q(m_k), q(W_k) per component, then q(s); the free energy with the new marginals
        double fe = -Hz, sa = sum_a0;
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            const double* pk = prm + k * LY.blk;
            const double* ak = acc + k * SA * TPB + tid;
            float* sk = st + k * SS * TPB;
            const double Nk = ak[0];
            sa += Nk;
            Vec<double, D> c, bk;
            Mat<double, D, D> EW, Ck;
#pragma unroll
            for (int i = 0; i < D; ++i) { c(i) = (double)sk[i * TPB + tid]; bk(i) = ak[(1 + i) * TPB]; }
            int p = D, pc = 1 + D;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j <= i; ++j, ++p, ++pc) {
                    const double w = (double)sk[p * TPB + tid] * (i == j ? 1.0 : 0.5);
                    EW(i, j) = w; EW(j, i) = w;
                    Ck(i, j) = ak[pc * TPB]; Ck(j, i) = Ck(i, j);
                }
            // q(m_k): precision V0^-1 + N_k E[W_k], weighted mean V0^-1 mu0 + E[W_k] sum_i r_ik y_i.  E[W_k] and the centre
            // c_k are the fp32 constants the data pass used: c_k exactly (the statistics are taken around it), E[W_k]
            // rounded to fp32 (relative 6e-8, DESIGN 3.17)
            Mat<double, D, D> Lm;
            Vec<double, D> sy;
#pragma unroll
            for (int i = 0; i < D * D; ++i) Lm.a[i] = pk[LY.V0i + i] + Nk * EW.a[i];
#pragma unroll
            for (int i = 0; i < D; ++i) sy(i) = bk(i) + Nk * c(i);
            double ldL;
            const Mat<double, D, D> Vm = inv_logdet(Lm, ldL, bad);
            Vec<double, D> xi = mulv(EW, sy);
#pragma unroll
            for (int i = 0; i < D; ++i) xi(i) += pk[LY.xi0 + i];
            const Vec<double, D> m = mulv(Vm, xi);
            // q(W_k): nu0 + N_k, inverse scale inv(S0) + R_k + N_k V_m, R_k = sum_i r_ik (y_i - m)(y_i - m)'
            Vec<double, D> dm;
#pragma unroll
            for (int i = 0; i < D; ++i) dm(i) = m(i) - c(i);
            Mat<double, D, D> R, iS;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j < D; ++j) {
                    R(i, j) = Ck(i, j) - bk(i) * dm(j) - dm(i) * bk(j) + Nk * dm(i) * dm(j);
                    iS(i, j) = pk[LY.S0i + i * D + j] + R(i, j) + Nk * Vm(i, j);
                }
            const double nu = pk[LY.nu0] + Nk;
            Mat<double, D, D> EWn;
            const double elog = derive<D>(m, Vm, nu, iS, sk, tid, bad, EWn);
            // free energy: KL(q(m_k) || prior), KL(q(W_k) || prior), the NormalMixture's average energy on component k
            double trV = 0.0, quad = 0.0, trS = 0.0, trR = 0.0;
            Vec<double, D> e;
#pragma unroll
            for (int i = 0; i < D; ++i) e(i) = m(i) - pk[LY.mu0 + i];
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j < D; ++j) {
                    const double v0i = pk[LY.V0i + i * D + j];
                    trV += v0i * Vm(j, i);
                    quad += e(i) * v0i * e(j);
                    trS += pk[LY.S0i + i * D + j] * EWn(j, i);                 // nu tr(inv(S0) S)
                    trR += EWn(i, j) * (R(j, i) + Nk * Vm(j, i));
                }
            const double nu0 = pk[LY.nu0];
            double psum = 0.0;
            for (int i = 0; i < D; ++i) psum += digamma(0.5 * (nu - i));
            const double logdetS = elog - D * 0.6931471805599453 - psum;            // log|S| of the new q(W_k)
            const double kl_m = 0.5 * (trV + quad - D + pk[LY.ldV0] + ldL);
            const double kl_w = 0.5 * (nu - nu0) * elog - 0.5 * nu * D + 0.5 * trS - 0.5 * (nu - nu0) * D * 0.6931471805599453
                                - 0.5 * nu * logdetS + 0.5 * nu0 * pk[LY.ldS0] - lgamma_mv<D>(0.5 * nu) + pk[LY.lgd0];
            fe += kl_m + kl_w + Nk * (0.5 * D * LOG2PI - 0.5 * elog) + 0.5 * trR;
            // outputs
            const double ak_new = pk[LY.a0] + Nk;
            if (o.h_alpha) o.h_alpha[((int64_t)it * K + k) * batch + b] = (float)ak_new;
            if (o.h_w_df) o.h_w_df[((int64_t)it * K + k) * batch + b] = (float)nu;
#pragma unroll
            for (int i = 0; i < D; ++i)
                if (o.h_m_mean) o.h_m_mean[(((int64_t)it * K + k) * D + i) * batch + b] = (float)m(i);
#pragma unroll
            for (int i = 0; i < D * D; ++i) {
                if (o.h_m_cov) o.h_m_cov[(((int64_t)it * K + k) * D * D + i) * batch + b] = (float)Vm.a[i];
                if (o.h_w_inv_scale) o.h_w_inv_scale[(((int64_t)it * K + k) * D * D + i) * batch + b] = (float)iS.a[i];
            }
            if (last) {
                o.alpha[(int64_t)k * batch + b] = (float)ak_new;
                o.w_df[(int64_t)k * batch + b] = (float)nu;
#pragma unroll
                for (int i = 0; i < D; ++i) o.m_mean[((int64_t)k * D + i) * batch + b] = (float)m(i);
#pragma unroll
                for (int i = 0; i < D * D; ++i) {
                    o.m_cov[((int64_t)k * D * D + i) * batch + b] = (float)Vm.a[i];
                    o.w_inv_scale[((int64_t)k * D * D + i) * batch + b] = (float)iS.a[i];
                }
            }
        }
        // q(s) = Dirichlet(alpha0 + N); E[log s_k] into the next pass's constants.  KL(q(s) || prior) carries
        // sum_k (alpha_k - alpha0_k) E[log s_k] = sum_k N_k E[log s_k], which cancels the Categorical nodes' average
        // energy -sum_k N_k E[log s_k]: the two add up to the log-normaliser difference alone.
        const double psa = digamma(sa);
        double lg = lgamma(sa) - lg_dir0;
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            const double a = prm[k * LY.blk + LY.a0] + acc[k * SA * TPB + tid];
            st[(k * SS + SS - 1) * TPB + tid] += (float)(digamma(a) - psa);
            lg -= lgamma(a);
        }
        fe += lg;
        if (o.free_energy) o.free_energy[(int64_t)it * batch + b] = fe;
    }
    if (o.status) o.status[b] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
}

}  // namespace gmm
}  // namespace rxg

namespace {

template <int D, int K>
int launch(rxg_ctx* ctx, const float* y, int N, int64_t batch, int iterations, const double* dp, const rxg::gmm::Out& o) {
    using namespace rxg::gmm;
    const size_t shm = (size_t)K * TPB * (acc_slots(D) * sizeof(double) + st_slots(D) * sizeof(float));
    RXG_CUDA(ctx, cudaFuncSetAttribute(gmm_vmp_kernel<D, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    const unsigned grid = (unsigned)((batch + TPB - 1) / TPB);
    gmm_vmp_kernel<D, K><<<grid, TPB, shm, ctx->stream>>>(y, N, batch, iterations, dp, o);
    return RXG_OK;
}

template <int D>
int launch_k(rxg_ctx* ctx, int K, const float* y, int N, int64_t batch, int iterations, const double* dp,
             const rxg::gmm::Out& o) {
    switch (K) {
        case 2: return launch<D, 2>(ctx, y, N, batch, iterations, dp, o);
        case 3: return launch<D, 3>(ctx, y, N, batch, iterations, dp, o);
        case 4: return launch<D, 4>(ctx, y, N, batch, iterations, dp, o);
        case 5: return launch<D, 5>(ctx, y, N, batch, iterations, dp, o);
        case 6: return launch<D, 6>(ctx, y, N, batch, iterations, dp, o);
        case 7: return launch<D, 7>(ctx, y, N, batch, iterations, dp, o);
        default: return launch<D, 8>(ctx, y, N, batch, iterations, dp, o);
    }
}

}  // namespace

extern "C" int rxg_gmm_vmp_f32(rxg_ctx* ctx, int d, int K, int N, int64_t batch, int iterations, const float* alpha0,
                               const float* mu0, const float* V0, const float* nu0, const float* S0,
                               const float* alpha_init, const float* m_init, const float* Vm_init, const float* nu_init,
                               const float* S_init, const float* y, float* alpha, float* m_mean, float* m_cov, float* w_df,
                               float* w_inv_scale, double* free_energy, float* z_prob, float* hist_alpha,
                               float* hist_m_mean, float* hist_m_cov, float* hist_w_df, float* hist_w_inv_scale,
                               int32_t* status, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "gmm_vmp takes device pointers");
    if (d < 1 || d > 4 || K < 2 || K > 8)
        return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "gmm_vmp: d=%d, K=%d unsupported (d 1-4, K 2-8)", d, K);
    if (N < 1 || batch < 1 || iterations < 1 || !alpha0 || !mu0 || !V0 || !nu0 || !S0 || !alpha_init || !m_init ||
        !Vm_init || !nu_init || !S_init || !y || !alpha || !m_mean || !m_cov || !w_df || !w_inv_scale)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: bad argument");
    const rxg::gmm::Layout LY = rxg::gmm::layout(d);
    const int dd = d * d;
    double hp[8 * (3 * 4 + 4 * 16 + 7) + 2];
    double sa0 = 0.0, slg0 = 0.0;
    for (int k = 0; k < K; ++k) {
        double* pk = hp + k * LY.blk;
        if (!(alpha0[k] > 0.f) || !(alpha_init[k] > 0.f) || !std::isfinite(alpha0[k]) || !std::isfinite(alpha_init[k]))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: alpha0 and alpha_init must be positive (component %d)", k);
        if (!(nu0[k] > (float)(d - 1)) || !(nu_init[k] > (float)(d - 1)) || !std::isfinite(nu0[k]) || !std::isfinite(nu_init[k]))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: nu0 and nu_init must exceed d - 1 (component %d)", k);
        for (int i = 0; i < d; ++i)
            if (!std::isfinite(mu0[k * d + i]) || !std::isfinite(m_init[k * d + i]))
                return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: mu0 and m_init must be finite (component %d)", k);
        double ld, tmp[16];
        if (!rxg::host_spd_inv(V0 + k * dd, d, pk + LY.V0i, &ld))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: V0[%d] is not SPD", k);
        pk[LY.ldV0] = ld;
        if (!rxg::host_spd_inv(S0 + k * dd, d, pk + LY.S0i, &ld))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: S0[%d] is not SPD", k);
        pk[LY.ldS0] = ld;
        if (!rxg::host_spd_inv(Vm_init + k * dd, d, tmp, &ld))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: Vm_init[%d] is not SPD", k);
        for (int i = 0; i < d; ++i)              // symmetrised, as every host matrix is validated
            for (int j = 0; j < d; ++j) pk[LY.Vi + i * d + j] = 0.5 * ((double)Vm_init[k * dd + i * d + j] + (double)Vm_init[k * dd + j * d + i]);
        if (!rxg::host_spd_inv(S_init + k * dd, d, pk + LY.iSi, &ld))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: S_init[%d] is not SPD", k);
        for (int i = 0; i < d; ++i) {
            pk[LY.mu0 + i] = mu0[k * d + i];
            pk[LY.mi + i] = m_init[k * d + i];
        }
        for (int i = 0; i < d; ++i) {
            double s = 0.0;
            for (int j = 0; j < d; ++j) s += pk[LY.V0i + i * d + j] * (double)mu0[k * d + j];
            pk[LY.xi0 + i] = s;
        }
        pk[LY.nu0] = nu0[k];
        pk[LY.a0] = alpha0[k];
        pk[LY.ai] = alpha_init[k];
        pk[LY.nui] = nu_init[k];
        double lgd = 0.25 * d * (d - 1) * rxg::gmm::LOGPI;
        for (int i = 0; i < d; ++i) lgd += std::lgamma(0.5 * ((double)nu0[k] - i));
        pk[LY.lgd0] = lgd;
        sa0 += alpha0[k];
        slg0 += std::lgamma((double)alpha0[k]);
    }
    hp[K * LY.blk] = sa0;
    hp[K * LY.blk + 1] = std::lgamma(sa0) - slg0;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nbytes = (size_t)(K * LY.blk + 2) * sizeof(double);
    double* dp = (double*)rxg::workspace(ctx, nbytes);
    if (!dp) return RXG_ERR_CUDA;
    RXG_CUDA(ctx, cudaMemcpyAsync(dp, hp, nbytes, cudaMemcpyHostToDevice, ctx->stream));
    const rxg::gmm::Out o{alpha, m_mean, m_cov, w_df, w_inv_scale, free_energy, z_prob, hist_alpha, hist_m_mean,
                          hist_m_cov, hist_w_df, hist_w_inv_scale, status};
    int rc;
    switch (d) {
        case 1: rc = launch_k<1>(ctx, K, y, N, batch, iterations, dp, o); break;
        case 2: rc = launch_k<2>(ctx, K, y, N, batch, iterations, dp, o); break;
        case 3: rc = launch_k<3>(ctx, K, y, N, batch, iterations, dp, o); break;
        default: rc = launch_k<4>(ctx, K, y, N, batch, iterations, dp, o); break;
    }
    if (rc != RXG_OK) return rc;
    ctx->launches += 1;
    rc = rxg::check_cuda(ctx, cudaGetLastError(), "gmm_vmp_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
