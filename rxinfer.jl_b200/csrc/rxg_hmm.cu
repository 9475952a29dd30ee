// rxg_hmm_vmp_f32: the hidden Markov model of test/models/statespace/hmm_tests.jl as one launch over a batch of chains
// (kernel body: rxg_hmm.cuh).  One thread per chain, K = 2..8 compiled, M <= 16 at run time.  Shared memory per thread,
// laid out [slot][thread]: B~ [M][K] (fp32), the transition counts [K][K] and the emission counts [M][K] (fp64).
#include <cmath>

#include "rxg_internal.h"
#include "rxg_hmm.cuh"

namespace rxg {
namespace hmm {

constexpr int TPB = 32;     // threads (chains) per block: small blocks, since shared memory bounds the chains per SM

inline size_t smem_bytes(int K, int M) { return (size_t)TPB * (M * K * sizeof(float) + (K * K + M * K) * sizeof(double)); }

template <int K>
__global__ void __launch_bounds__(TPB) hmm_vmp_kernel(Args a, int32_t* __restrict__ status) {
    extern __shared__ double smem[];
    const int tid = threadIdx.x;
    const int64_t b = (int64_t)blockIdx.x * TPB + tid;
    if (b >= a.batch) return;
    double* dsh = smem + tid;                                                     // [(K + M) K][TPB]
    float* fsh = reinterpret_cast<float*>(smem + (K * K + a.M * K) * TPB) + tid;  // [M K][TPB]
    const int st = chain<K>(b, a, fsh, dsh, TPB);
    if (status) status[b] = st;
}

}  // namespace hmm
}  // namespace rxg

namespace {

template <int K>
int launch(rxg_ctx* ctx, const rxg::hmm::Args& a, int32_t* status) {
    using namespace rxg::hmm;
    const size_t shm = smem_bytes(K, a.M);
    RXG_CUDA(ctx, cudaFuncSetAttribute(hmm_vmp_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    const unsigned grid = (unsigned)((a.batch + TPB - 1) / TPB);
    hmm_vmp_kernel<K><<<grid, TPB, shm, ctx->stream>>>(a, status);
    return RXG_OK;
}

}  // namespace

namespace rxg {

// columns of a [rows][K] matrix each a probability vector (non-negative, finite, sum 1 within 1e-5)
bool stochastic_columns(const float* p, int rows, int K) {
    for (int j = 0; j < K; ++j) {
        double s = 0.0;
        for (int i = 0; i < rows; ++i) {
            const float v = p[i * K + j];
            if (!(v >= 0.f) || !std::isfinite(v)) return false;
            s += v;
        }
        if (std::fabs(s - 1.0) > 1e-5) return false;
    }
    return true;
}

bool positive(const float* p, int n) {
    for (int i = 0; i < n; ++i)
        if (!(p[i] > 0.f) || !std::isfinite(p[i])) return false;
    return true;
}

}  // namespace rxg

extern "C" int rxg_hmm_vmp_f32(rxg_ctx* ctx, int K, int M, int T, int64_t batch, int iterations, const float* p0,
                               const float* A_prior, const float* A_init, const float* A_known, const float* B_prior,
                               const float* B_init, const float* B_known, const uint8_t* x, float* s_prob,
                               float* s0_prob, float* A_alpha, float* B_alpha, double* free_energy, float* hist_s,
                               float* hist_A, float* hist_B, int32_t* status, unsigned flags) {
    using namespace rxg::hmm;
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "hmm_vmp takes device pointers");
    if (K < 2 || K > 8 || M < 2 || M > MAX_M)
        return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "hmm_vmp: K=%d, M=%d unsupported (K 2-8, M 2-16)", K, M);
    if (T < 1 || batch < 1 || iterations < 1 || !p0 || !x || !s_prob)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hmm_vmp: bad argument");
    const bool learn_A = A_prior || A_init, learn_B = B_prior || B_init;
    if (learn_A == (A_known != nullptr) || (learn_A && !(A_prior && A_init)))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hmm_vmp: pass either A_prior and A_init (A learned) or A_known");
    if (learn_B == (B_known != nullptr) || (learn_B && !(B_prior && B_init)))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hmm_vmp: pass either B_prior and B_init (B learned) or B_known");
    if (!rxg::stochastic_columns(p0, K, 1)) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hmm_vmp: p0 is not a probability vector");
    if (learn_A ? !(rxg::positive(A_prior, K * K) && rxg::positive(A_init, K * K)) : !rxg::stochastic_columns(A_known, K, K))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, learn_A ? "hmm_vmp: A_prior and A_init must be positive"
                                                        : "hmm_vmp: the columns of A_known must be probability vectors");
    if (learn_B ? !(rxg::positive(B_prior, M * K) && rxg::positive(B_init, M * K)) : !rxg::stochastic_columns(B_known, M, K))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, learn_B ? "hmm_vmp: B_prior and B_init must be positive"
                                                        : "hmm_vmp: the columns of B_known must be probability vectors");
    double hp[8 + 2 * 64 + 2 * MAX_M * 8];
    for (int i = 0; i < K; ++i) hp[i] = p0[i];
    for (int q = 0; q < K * K; ++q) {
        hp[off_A(K) + q] = learn_A ? A_prior[q] : A_known[q];
        hp[off_Ai(K) + q] = learn_A ? A_init[q] : 0.0;
    }
    for (int q = 0; q < M * K; ++q) {
        hp[off_B(K) + q] = learn_B ? B_prior[q] : B_known[q];
        hp[off_Bi(K, M) + q] = learn_B ? B_init[q] : 0.0;
    }
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nbytes = (size_t)n_params(K, M) * sizeof(double);
    double* dp = (double*)rxg::workspace(ctx, nbytes);
    if (!dp) return RXG_ERR_CUDA;
    RXG_CUDA(ctx, cudaMemcpyAsync(dp, hp, nbytes, cudaMemcpyHostToDevice, ctx->stream));
    Args a{T, M, iterations, batch, learn_A, learn_B, dp, x, s_prob, s0_prob,
           learn_A ? A_alpha : nullptr, learn_B ? B_alpha : nullptr, free_energy, hist_s,
           learn_A ? hist_A : nullptr, learn_B ? hist_B : nullptr};
    int rc;
    switch (K) {
        case 2: rc = launch<2>(ctx, a, status); break;
        case 3: rc = launch<3>(ctx, a, status); break;
        case 4: rc = launch<4>(ctx, a, status); break;
        case 5: rc = launch<5>(ctx, a, status); break;
        case 6: rc = launch<6>(ctx, a, status); break;
        case 7: rc = launch<7>(ctx, a, status); break;
        default: rc = launch<8>(ctx, a, status); break;
    }
    if (rc != RXG_OK) return rc;
    ctx->launches += 1;
    rc = rxg::check_cuda(ctx, cudaGetLastError(), "hmm_vmp_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
