// Variational message passing around the per-chain smoother with an unknown observation precision MATRIX, one per
// chain: the multivariate twin of vmp_gamma_kernel (rxg_hgf.cu).
//
//   w ~ Wishart(nu0, inv(Psi0));  x[1] ~ N(m0, S0) (or one transition earlier, RXG_TRANSITION_FIRST);
//   x[t] ~ N(A x[t-1] + u, P);    y[t] ~ N(B x[t], inv(w));    q(x) q(w)
// [ref: docs/src/manuals/model-specification.md:265-271, constraints q(x, w) = q(x)q(w)].
//
// One iteration k, per chain:
//   q(x)  exact Kalman filter + RTS smoother with Q = inv(Wbar), Wbar = E[w] under q_{k-1}(w) (init_E_W at k = 0): the
//         average energy of the y node under q(w) is N(y | Bx, inv(E[w])) up to constants.
//   q(w)  = prior x prod_t MvNormalMeanPrecision(:Lambda)(q_out = PointMass(y_t), q_mu = N(B mu_t, B Sigma_t B')), i.e.
//         df = nu0 + N_b, Psi = Psi0 + R_b, R_b = sum_{observed t} (y_t - B mu_t)(y_t - B mu_t)' + B Sigma_t B'.
//   F_k   = NLE(Wbar) + N_b/2 (log det Wbar - E log det w) + 1/2 tr((E w - Wbar) R_b) + KL(q_k(w) || prior)   (fp64)
//         with q(x) the exact chain posterior under Wbar (its Gaussian part collapses to the filter's evidence).
// One thread = one chain, all iterations in one launch; every array is [..][batch] (coalesced).  post_mean / post_cov are
// the forward->backward stash of every iteration; only the last iteration writes the smoothed q(x) over it.  The Kalman and
// RTS step bodies are lgssm_chain_kernel's (rxg_chain_step.cuh).
//
// This translation unit is compiled once per Wishart dimension m (-DRXG_VMP_M=m: d = 1..6 of that m) and once without it
// for the C entry below.  m is compiled exactly: padding y would add dummy coordinates to w and change the answer.
#include <math.h>

#include "rxg_chain_step.cuh"
#include "rxg_internal.h"

namespace rxg {

struct VmpWishHost {        // host-side model of one call (fp64 where the kernel works in fp64)
    const float *A, *B, *P, *m0, *S0, *u;
    double nu0, logdet_Psi0;
    double Psi0[36], W0[36];   // [m][m], symmetrised
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

template <int D, int M>
struct VmpWishModel {
    float A[D * D], B[M * D], P[D * D], m0[D], S0[D * D], u[D];
    double nu0, logdet_Psi0, Psi0[M * M], W0[M * M];
};

__device__ __forceinline__ double digamma_d(double x) {      // psi(x), x > 0: recurrence up to x >= 10, asymptotic series
    double r = 0.0;
    while (x < 10.0) { r -= 1.0 / x; x += 1.0; }
    const double i = 1.0 / x, i2 = i * i;
    return r + log(x) - 0.5 * i - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 * (1.0 / 252 - i2 * (1.0 / 240 - i2 * (1.0 / 132)))));
}

template <int D, int M>
__global__ void __launch_bounds__(128)
lgssm_vmp_wishart_kernel(const __grid_constant__ VmpWishModel<D, M> mdl, const VmpWishIO io) {
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
    for (int i = 0; i < M * M; ++i) Wbar.a[i] = mdl.W0[i];
    bool bad = false;
    const bool want_fe = io.fe != nullptr;
    Vec<float, D> mu;

    for (int it = 0; it < io.iterations; ++it) {
        const bool last = it == io.iterations - 1;
        // ---- q(x) under Q = inv(Wbar)
        const double logdet_W = -2.0 * cholesky<double, M, true>(Wbar, bad).neg_half_logdet;
        const Mat<float, M, M> Q = convert<float>(cholinv(Wbar, bad));
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
            if (t > 0 || io.tf) chain_predict(A, P, u, NoInput{}, mu, S);
            if (obs) {
                chain_update(B, Q, yt, want_fe, mu, S, bad, nle);
                ++nobs;
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

        // ---- backward RTS pass and R_b = sum_{observed t} (y_t - B mu_t)(y_t - B mu_t)' + B Sigma_t B' (fp64)
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
        if (obs) accumulate(mu, S, yt);
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
            chain_rts(A, P, u, NoInput{}, muf, Sf, mus, Ss, bad);
            if (last) {
#pragma unroll
                for (int i = 0; i < D; ++i) mean[((int64_t)t * D + i) * batch + b] = mus(i);
#pragma unroll
                for (int i = 0; i < D; ++i)
#pragma unroll
                    for (int j = 0; j < D; ++j) cov[(((int64_t)t * D + i) * D + j) * batch + b] = Ss(i, j);
            }
            if (ob) accumulate(mus, Ss, yv);
        }
        mu = mus;

        // ---- q(w) = Wishart(df, inv(Psi)) and the free energy (fp64)
        const double df = mdl.nu0 + (double)nobs;
        Mat<double, M, M> Psi;
        {
            int q = 0;
#pragma unroll
            for (int k = 0; k < M; ++k)
#pragma unroll
                for (int l = 0; l <= k; ++l) {
                    Psi(k, l) = mdl.Psi0[k * M + l] + R[q];
                    Psi(l, k) = Psi(k, l);
                    ++q;
                }
        }
        const Mat<double, M, M> Pinv = cholinv(Psi, bad);
        io.df[(int64_t)it * batch + b] = (float)df;
#pragma unroll
        for (int k = 0; k < M; ++k)
#pragma unroll
            for (int l = 0; l < M; ++l) io.inv_scale[(((int64_t)it * M + k) * M + l) * batch + b] = (float)Psi(k, l);
        Mat<double, M, M> Wn;
#pragma unroll
        for (int i = 0; i < M * M; ++i) Wn.a[i] = df * Pinv.a[i];
        if (want_fe) {
            const double logdet_Psi = -2.0 * cholesky<double, M, true>(Psi, bad).neg_half_logdet;
            double psi_m = 0.0, lg = 0.0;      // sum_i psi((df - i)/2), sum_i [lgamma((nu0 - i)/2) - lgamma((df - i)/2)]
#pragma unroll
            for (int i = 0; i < M; ++i) {
                psi_m += digamma_d(0.5 * (df - i));
                lg += lgamma(0.5 * (mdl.nu0 - i)) - lgamma(0.5 * (df - i));
            }
            const double Elogdet = psi_m + M * 0.69314718055994530942 - logdet_Psi;
            double trR = 0.0, trP = 0.0;        // tr((E w - Wbar) R), tr(Psi0 inv(Psi))
            {
                int q = 0;
#pragma unroll
                for (int k = 0; k < M; ++k)
#pragma unroll
                    for (int l = 0; l <= k; ++l) {
                        const double f = (k == l) ? 1.0 : 2.0;
                        trR += f * (Wn(k, l) - Wbar(k, l)) * R[q++];
                        trP += f * mdl.Psi0[k * M + l] * Pinv(k, l);
                    }
            }
            const double kl = -0.5 * mdl.nu0 * (mdl.logdet_Psi0 - logdet_Psi) + 0.5 * df * (trP - M) + lg +
                              0.5 * (df - mdl.nu0) * psi_m;
            io.fe[(int64_t)it * batch + b] = nle + 0.5 * nobs * (logdet_W - Elogdet) + 0.5 * trR + kl;
        }
        Wbar = Wn;
    }
    if (io.status) {
        bool nan = false;
#pragma unroll
        for (int i = 0; i < D; ++i) nan |= !(mu(i) == mu(i));
        io.status[b] = bad ? RXG_ERR_NOT_SPD : (nan ? RXG_ERR_NAN : RXG_OK);
    }
}

template <int D, int M>
int launch_vmp_wishart(rxg_ctx* ctx, const VmpWishHost& h, const VmpWishIO& io) {
    VmpWishModel<D, M> mdl = {};
    for (int i = 0; i < D * D; ++i) { mdl.A[i] = h.A[i]; mdl.P[i] = h.P[i]; mdl.S0[i] = h.S0[i]; }
    for (int i = 0; i < M * D; ++i) mdl.B[i] = h.B[i];
    for (int i = 0; i < D; ++i) { mdl.m0[i] = h.m0[i]; mdl.u[i] = h.u ? h.u[i] : 0.f; }
    for (int i = 0; i < M * M; ++i) { mdl.Psi0[i] = h.Psi0[i]; mdl.W0[i] = h.W0[i]; }
    mdl.nu0 = h.nu0;
    mdl.logdet_Psi0 = h.logdet_Psi0;
    const int threads = 64;
    if (ctx->profile) { cudaEventRecord(ctx->ev[0], ctx->stream); cudaEventRecord(ctx->ev[1], ctx->stream); }
    lgssm_vmp_wishart_kernel<D, M><<<(unsigned)((io.batch + threads - 1) / threads), threads, 0, ctx->stream>>>(mdl, io);
    if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "lgssm_vmp_wishart_kernel launch");
}

#ifdef RXG_VMP_M
template int launch_vmp_wishart<1, RXG_VMP_M>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);
template int launch_vmp_wishart<2, RXG_VMP_M>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);
template int launch_vmp_wishart<3, RXG_VMP_M>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);
template int launch_vmp_wishart<4, RXG_VMP_M>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);
template int launch_vmp_wishart<5, RXG_VMP_M>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);
template int launch_vmp_wishart<6, RXG_VMP_M>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);
}  // namespace rxg
#else

namespace {
// fp64 Cholesky of the symmetrised (A + A')/2 on the host: false if it is not SPD; log det on success
bool host_spd(const float* a, int m, double* sym, double* logdet) {
    double L[36] = {};
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < m; ++j) sym[i * m + j] = 0.5 * ((double)a[i * m + j] + (double)a[j * m + i]);
    double ld = 0.0;
    for (int j = 0; j < m; ++j) {
        double s = sym[j * m + j];
        for (int k = 0; k < j; ++k) s -= L[j * m + k] * L[j * m + k];
        if (!(s > 0.0) || !isfinite(s)) return false;
        L[j * m + j] = sqrt(s);
        ld += 2.0 * log(L[j * m + j]);
        for (int i = j + 1; i < m; ++i) {
            double t = sym[i * m + j];
            for (int k = 0; k < j; ++k) t -= L[i * m + k] * L[j * m + k];
            L[i * m + j] = t / L[j * m + j];
        }
    }
    *logdet = ld;
    return true;
}

int dispatch(rxg_ctx* ctx, int d, int m, const VmpWishHost& h, const VmpWishIO& io) {
#define RXG_VMP_CASE(DD, MM) case DD * 16 + MM: return launch_vmp_wishart<DD, MM>(ctx, h, io);
#define RXG_VMP_ROW(DD) RXG_VMP_CASE(DD, 1) RXG_VMP_CASE(DD, 2) RXG_VMP_CASE(DD, 3) RXG_VMP_CASE(DD, 4) \
                        RXG_VMP_CASE(DD, 5) RXG_VMP_CASE(DD, 6)
    switch (d * 16 + m) {
        RXG_VMP_ROW(1) RXG_VMP_ROW(2) RXG_VMP_ROW(3) RXG_VMP_ROW(4) RXG_VMP_ROW(5) RXG_VMP_ROW(6)
        default: return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_vmp_wishart: d and m must be in 1..6 (got d=%d, m=%d)", d, m);
    }
#undef RXG_VMP_ROW
#undef RXG_VMP_CASE
}
}  // namespace

#define RXG_VMP_EXTERN(DD)                                                                                  \
    extern template int launch_vmp_wishart<DD, 1>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);          \
    extern template int launch_vmp_wishart<DD, 2>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);          \
    extern template int launch_vmp_wishart<DD, 3>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);          \
    extern template int launch_vmp_wishart<DD, 4>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);          \
    extern template int launch_vmp_wishart<DD, 5>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);          \
    extern template int launch_vmp_wishart<DD, 6>(rxg_ctx*, const VmpWishHost&, const VmpWishIO&);
RXG_VMP_EXTERN(1) RXG_VMP_EXTERN(2) RXG_VMP_EXTERN(3) RXG_VMP_EXTERN(4) RXG_VMP_EXTERN(5) RXG_VMP_EXTERN(6)
#undef RXG_VMP_EXTERN

}  // namespace rxg

using namespace rxg;

extern "C" int rxg_lgssm_vmp_wishart_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch, int iterations, const float* A,
                                         const float* B, const float* P, const float* m0, const float* S0, const float* u,
                                         float nu0, const float* inv_scale0, const float* init_E_W, const float* y,
                                         const uint8_t* ymask, float* post_mean, float* post_cov, float* df,
                                         float* inv_scale, double* free_energy, int32_t* status, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    const unsigned accepted = RXG_PTR_DEVICE | RXG_TRANSITION_FIRST | RXG_MASK_SHARED | RXG_ASYNC;
    if (flags & ~accepted)
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_vmp_wishart: flags 0x%x are not supported (per-chain models, input "
                                              "sequences and the shared covariance output do not apply: the covariances "
                                              "depend on the chain through w)", flags & ~accepted);
    if (!(flags & RXG_PTR_DEVICE)) return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_vmp_wishart takes device pointers");
    if (d < 1 || d > 6 || m < 1 || m > 6)
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_vmp_wishart: d and m must be in 1..6 (got d=%d, m=%d)", d, m);
    if (T < 1 || batch < 1 || iterations < 1)
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_vmp_wishart: T, batch and iterations must be >= 1");
    if (!A || !B || !P || !m0 || !S0 || !inv_scale0 || !init_E_W || !y || !post_mean || !post_cov || !df || !inv_scale)
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_vmp_wishart: null pointer argument");
    if (!((double)nu0 > (double)(m - 1)) || !isfinite(nu0))
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_vmp_wishart: the prior's degrees of freedom must exceed m - 1 (nu0=%g, m=%d)",
                    (double)nu0, m);
    VmpWishHost h;
    h.A = A; h.B = B; h.P = P; h.m0 = m0; h.S0 = S0; h.u = u;
    h.nu0 = (double)nu0;
    double ld_w = 0.0;
    if (!host_spd(inv_scale0, m, h.Psi0, &h.logdet_Psi0))
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_vmp_wishart: inv_scale0 is not symmetric positive definite");
    if (!host_spd(init_E_W, m, h.W0, &ld_w))
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_vmp_wishart: init_E_W is not symmetric positive definite");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    VmpWishIO io;
    io.y = y; io.ymask = nullptr; io.tmask = nullptr;
    io.mean = post_mean; io.cov = post_cov; io.df = df; io.inv_scale = inv_scale; io.fe = free_energy; io.status = status;
    io.T = T; io.iterations = iterations; io.tf = (flags & RXG_TRANSITION_FIRST) ? 1 : 0;
    io.batch = batch;
    if (ymask) {
        if (flags & RXG_MASK_SHARED) {
            LgssmCall c = {};
            const int rc = stage_shared_mask(ctx, T, ymask, c);
            if (rc != RXG_OK) return rc;
            io.tmask = c.tmask;
        } else {
            io.ymask = ymask;
        }
    }
    const int rc = dispatch(ctx, d, m, h, io);
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

#endif  // RXG_VMP_M
