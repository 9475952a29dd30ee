// rxg_hmm_gauss_vmp_f32: the hidden Markov model with Gaussian (NormalMixture) emissions as one launch over a batch of
// chains (kernel body: rxg_hmm_gauss.cuh).  One thread per chain, d = 1..4 x K = 2..8 compiled.  Shared memory per thread,
// laid out [slot][thread]: the transition counts [K][K] and the Gaussian statistics [K][1 + d + d(d+1)/2] (fp64), then
// the sweep constants [K][d + d(d+1)/2 + 1] (fp32): 1.95 KB at K = 8, d = 4.
#include <cmath>

#include "rxg_internal.h"
#include "rxg_hmm_gauss.cuh"

namespace rxg {
namespace hmmg {

constexpr int TPB = 32;     // threads (chains) per block: small blocks, since shared memory bounds the chains per SM

inline size_t smem_bytes(int d, int K) {
    return (size_t)TPB * ((K * K + K * acc_slots(d)) * sizeof(double) + f_slots(d, K) * sizeof(float));
}

template <int D, int K>
__global__ void __launch_bounds__(TPB) hmm_gauss_vmp_kernel(Args a, int32_t* __restrict__ status) {
    extern __shared__ double smem[];
    const int tid = threadIdx.x;
    const int64_t b = (int64_t)blockIdx.x * TPB + tid;
    if (b >= a.batch) return;
    double* dsh = smem + tid;                                                          // [K (K + SA)][TPB]
    float* fsh = reinterpret_cast<float*>(smem + (K * K + K * acc_slots(D)) * TPB) + tid;   // [f_slots][TPB]
    const int st = chain<D, K>(b, a, fsh, dsh, TPB);
    if (status) status[b] = st;
}

}  // namespace hmmg
}  // namespace rxg

namespace {

template <int D, int K>
int launch(rxg_ctx* ctx, const rxg::hmmg::Args& a, int32_t* status) {
    using namespace rxg::hmmg;
    const size_t shm = smem_bytes(D, K);
    RXG_CUDA(ctx, cudaFuncSetAttribute(hmm_gauss_vmp_kernel<D, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    const unsigned grid = (unsigned)((a.batch + TPB - 1) / TPB);
    hmm_gauss_vmp_kernel<D, K><<<grid, TPB, shm, ctx->stream>>>(a, status);
    return RXG_OK;
}

template <int D>
int launch_k(rxg_ctx* ctx, int K, const rxg::hmmg::Args& a, int32_t* status) {
    switch (K) {
        case 2: return launch<D, 2>(ctx, a, status);
        case 3: return launch<D, 3>(ctx, a, status);
        case 4: return launch<D, 4>(ctx, a, status);
        case 5: return launch<D, 5>(ctx, a, status);
        case 6: return launch<D, 6>(ctx, a, status);
        case 7: return launch<D, 7>(ctx, a, status);
        default: return launch<D, 8>(ctx, a, status);
    }
}

}  // namespace

extern "C" int rxg_hmm_gauss_vmp_f32(rxg_ctx* ctx, int d, int K, int T, int64_t batch, int iterations, const float* p0,
                                     const float* A_prior, const float* A_init, const float* A_known, const float* mu0,
                                     const float* V0, const float* nu0, const float* S0, const float* m_init,
                                     const float* Vm_init, const float* nu_init, const float* S_init, const float* y,
                                     float* s_prob, float* s0_prob, float* A_alpha, float* m_mean, float* m_cov,
                                     float* w_df, float* w_inv_scale, double* free_energy, float* hist_s, float* hist_A,
                                     float* hist_m_mean, float* hist_m_cov, float* hist_w_df, float* hist_w_inv_scale,
                                     int32_t* status, unsigned flags) {
    using namespace rxg::hmmg;
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "hmm_gauss_vmp takes device pointers");
    if (d < 1 || d > 4 || K < 2 || K > 8)
        return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "hmm_gauss_vmp: d=%d, K=%d unsupported (d 1-4, K 2-8)", d, K);
    if (T < 1 || batch < 1 || iterations < 1 || !p0 || !mu0 || !V0 || !nu0 || !S0 || !m_init || !Vm_init || !nu_init ||
        !S_init || !y || !s_prob)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hmm_gauss_vmp: bad argument");
    const bool learn_A = A_prior || A_init;
    if (learn_A == (A_known != nullptr) || (learn_A && !(A_prior && A_init)))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hmm_gauss_vmp: pass either A_prior and A_init (A learned) or A_known");
    if (!rxg::stochastic_columns(p0, K, 1))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hmm_gauss_vmp: p0 is not a probability vector");
    if (learn_A ? !(rxg::positive(A_prior, K * K) && rxg::positive(A_init, K * K)) : !rxg::stochastic_columns(A_known, K, K))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, learn_A ? "hmm_gauss_vmp: A_prior and A_init must be positive"
                                                        : "hmm_gauss_vmp: the columns of A_known must be probability vectors");
    const int blk = layout(d).blk;
    double hp[8 + 2 * 64 + 8 * (3 * 4 + 4 * 16 + 5)];
    for (int i = 0; i < K; ++i) hp[i] = p0[i];
    for (int q = 0; q < K * K; ++q) {
        hp[K + q] = learn_A ? A_prior[q] : A_known[q];
        hp[K + K * K + q] = learn_A ? A_init[q] : 0.0;
    }
    for (int k = 0; k < K; ++k)
        if (int rc = pack(ctx, "hmm_gauss_vmp", "state", k, d, mu0, V0, nu0, S0, m_init, Vm_init, nu_init, S_init,
                          hp + off_states(K) + k * blk))
            return rc;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nbytes = (size_t)n_params(K, d) * sizeof(double);
    double* dp = (double*)rxg::workspace(ctx, nbytes);
    if (!dp) return RXG_ERR_CUDA;
    RXG_CUDA(ctx, cudaMemcpyAsync(dp, hp, nbytes, cudaMemcpyHostToDevice, ctx->stream));
    Args a{T, iterations, batch, learn_A, dp, y, s_prob, s0_prob, learn_A ? A_alpha : nullptr, m_mean, m_cov, w_df,
           w_inv_scale, free_energy, hist_s, learn_A ? hist_A : nullptr, hist_m_mean, hist_m_cov, hist_w_df,
           hist_w_inv_scale};
    int rc;
    switch (d) {
        case 1: rc = launch_k<1>(ctx, K, a, status); break;
        case 2: rc = launch_k<2>(ctx, K, a, status); break;
        case 3: rc = launch_k<3>(ctx, K, a, status); break;
        default: rc = launch_k<4>(ctx, K, a, status); break;
    }
    if (rc != RXG_OK) return rc;
    ctx->launches += 1;
    rc = rxg::check_cuda(ctx, cudaGetLastError(), "hmm_gauss_vmp_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
