// Fused mean-field VMP of the Gaussian mixture model, `batch` independent data sets, all iterations in one launch
// [ref: test/models/mixtures/gmm_multivariate_tests.jl:4-24 (K = 3, d = 2) and gmm_univariate_tests.jl:6-20 (K = 2,
// d = 1, the Beta / Bernoulli / Gamma spelling of the same model)]:
//   s ~ Dirichlet(alpha0);  m[k] ~ MvNormal(mu0[k], V0[k]);  W[k] ~ Wishart(nu0[k], S0[k]);
//   z[i] ~ Categorical(s);  y[i] ~ NormalMixture(z[i], m, W);  q = q(s) prod q(m[k]) prod q(W[k]) prod q(z[i]).
// One thread = one data set.  Every iteration is one coalesced pass over y[N][d][batch] (batch innermost): the
// responsibilities r[i][k] from the previous q(s), q(m), q(W), then the per-component statistics N_k, sum r (y - c_k),
// sum r (y - c_k)(y - c_k)' accumulated in fp64 around c_k = the previous E[m_k] (the points sit near their cluster's
// mean, so nothing cancels when the data are far from the origin), then the O(K d^3) conjugate updates in fp64 in the
// order q(m) (previous E[W]), q(W) (new q(m)) (rxg_normal_wishart.cuh), q(s) (DESIGN 3.17), then the Bethe free energy
// in fp64.
// Shared memory per thread, laid out [slot][thread]: the fp64 accumulators and the fp32 per-component constants the
// data pass reads (centre, packed E[W], log-weight offset).  At K = 8, d = 4 that is 120 + 120 slots.
#include <cfloat>
#include <cmath>

#include "rxg_internal.h"
#include "rxg_normal_wishart.cuh"

namespace rxg {
namespace gmm {

constexpr int TPB = 64;                       // threads (chains) per block
using namespace nw;                           // the component: layout, derive, update, store, digamma

// fp64 host constants: one nw::Layout block per component, then alpha0[K], alpha_init[K], sum(alpha0),
// lgamma(sum alpha0) - sum lgamma(alpha0)
inline int n_params(int K, int d) { return K * layout(d).blk + 2 * K + 2; }

struct Out {
    float *alpha, *m_mean, *m_cov, *w_df, *w_inv_scale;
    double* free_energy;
    float* z_prob;
    float *h_alpha, *h_m_mean, *h_m_cov, *h_w_df, *h_w_inv_scale;
    int32_t* status;
};

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
    // Status: RXG_ERR_NOT_SPD from the first non-positive pivot on, else RXG_OK.  At d = 1 it is written when a pivot
    // fails, since a flag kept through the kernel is spilled there around the fp64 slow-path calls of the updates; the
    // other sizes keep the flag, which at d = 4, K = 8 keeps the data pass faster (82 against 90 ms, DESIGN 3.17).
    constexpr bool EAGER = D == 1;
    bool bad = false, bk = false;
    if (EAGER && o.status) o.status[b] = RXG_OK;
    const double* a0 = prm + K * LY.blk;                       // alpha0[K], alpha_init[K], sum(alpha0), normaliser

    // initial q(s), q(m), q(W) -> constants of the first data pass
    {
        double sa = 0.0;
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            const double* pk = prm + k * LY.blk;
            double EW[D * D];
            derive<D>(pk + LY.mi, pk + LY.Vi, pk[LY.nui], pk + LY.iSi, st + k * SS * TPB + tid, TPB, EAGER ? bk : bad, EW);
            if (EAGER && bk && o.status) o.status[b] = RXG_ERR_NOT_SPD;
            sa += a0[K + k];
        }
        const double psa = digamma(sa);
#pragma unroll 1
        for (int k = 0; k < K; ++k) st[(k * SS + SS - 1) * TPB + tid] += (float)(digamma(a0[K + k]) - psa);
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
        double fe = -Hz, sa = a0[2 * K];
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            const double Nk = acc[k * SA * TPB + tid];
            sa += Nk;
            double m[D], Vm[D * D], nu, iS[D * D];
            fe += update<D>(prm + k * LY.blk, acc + k * SA * TPB + tid, st + k * SS * TPB + tid, TPB, EAGER ? bk : bad, m, Vm,
                            nu, iS);
            if (EAGER && bk && o.status) o.status[b] = RXG_ERR_NOT_SPD;
            const double ak_new = a0[k] + Nk;
            if (o.h_alpha) o.h_alpha[((int64_t)it * K + k) * batch + b] = (float)ak_new;
            store<D>((int64_t)it * K + k, batch, b, m, Vm, nu, iS, o.h_m_mean, o.h_m_cov, o.h_w_df, o.h_w_inv_scale);
            if (last) {
                o.alpha[(int64_t)k * batch + b] = (float)ak_new;
                store<D>(k, batch, b, m, Vm, nu, iS, o.m_mean, o.m_cov, o.w_df, o.w_inv_scale);
            }
        }
        // q(s) = Dirichlet(alpha0 + N); E[log s_k] into the next pass's constants.  KL(q(s) || prior) carries
        // sum_k (alpha_k - alpha0_k) E[log s_k] = sum_k N_k E[log s_k], which cancels the Categorical nodes' average
        // energy -sum_k N_k E[log s_k]: the two add up to the log-normaliser difference alone.
        const double psa = digamma(sa);
        double lg = lgamma(sa) - a0[2 * K + 1];
#pragma unroll 1
        for (int k = 0; k < K; ++k) {
            const double a = a0[k] + acc[k * SA * TPB + tid];
            st[(k * SS + SS - 1) * TPB + tid] += (float)(digamma(a) - psa);
            lg -= lgamma(a);
        }
        fe += lg;
        if (o.free_energy) o.free_energy[(int64_t)it * batch + b] = fe;
    }
    if (!EAGER && o.status) o.status[b] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
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
    const int blk = rxg::nw::layout(d).blk;
    double hp[8 * (3 * 4 + 4 * 16 + 5) + 2 * 8 + 2];
    double *a0 = hp + K * blk, *ai = a0 + K;
    double sa0 = 0.0, slg0 = 0.0;
    for (int k = 0; k < K; ++k) {
        if (!(alpha0[k] > 0.f) || !(alpha_init[k] > 0.f) || !std::isfinite(alpha0[k]) || !std::isfinite(alpha_init[k]))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gmm_vmp: alpha0 and alpha_init must be positive (component %d)", k);
        if (int rc = rxg::nw::pack(ctx, "gmm_vmp", "component", k, d, mu0, V0, nu0, S0, m_init, Vm_init, nu_init, S_init,
                                   hp + k * blk))
            return rc;
        a0[k] = alpha0[k];
        ai[k] = alpha_init[k];
        sa0 += alpha0[k];
        slg0 += std::lgamma((double)alpha0[k]);
    }
    a0[2 * K] = sa0;
    a0[2 * K + 1] = std::lgamma(sa0) - slg0;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nbytes = (size_t)rxg::gmm::n_params(K, d) * sizeof(double);
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
