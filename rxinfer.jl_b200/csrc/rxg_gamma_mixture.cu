// Fused mean-field VMP of the Gamma mixture model with point-mass shapes, `batch` independent data sets, all iterations
// in one launch (rxg_gamma_mixture.cuh has the model, the updates and the free energy; DESIGN 3.24).  One thread = one
// data set; every iteration reads y[N][batch] once, coalesced (batch innermost), with log y formed on the fly.  The
// pass keeps its per-component constants and fp64 accumulators in registers; the per-chain fp64 state the component
// loop indexes by k lives in shared memory, laid out [slot][thread].
#include <cmath>

#include "rxg_gamma_mixture.cuh"
#include "rxg_internal.h"

namespace rxg {
namespace gamix {

constexpr int TPB = 64;                       // threads (data sets) per block

template <int K>
__global__ void __launch_bounds__(TPB) gamma_mixture_vmp_kernel(Args a, int32_t* status) {
    extern __shared__ double smem[];          // [N_SLOTS * K][TPB]
    const int64_t b = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (b >= a.batch) return;
    const int st = chain<K>(b, a, smem + threadIdx.x, TPB);
    if (status) status[b] = st;
}

}  // namespace gamix
}  // namespace rxg

namespace {

template <int K>
void launch(rxg_ctx* ctx, const rxg::gamix::Args& a, int32_t* status) {
    using namespace rxg::gamix;
    const size_t shm = (size_t)N_SLOTS * K * TPB * sizeof(double);
    const unsigned grid = (unsigned)((a.batch + TPB - 1) / TPB);
    gamma_mixture_vmp_kernel<K><<<grid, TPB, shm, ctx->stream>>>(a, status);
}

}  // namespace

extern "C" int rxg_gamma_mixture_vmp_f32(rxg_ctx* ctx, int K, int N, int64_t batch, int iterations, const float* alpha_s,
                                         const float* a_shape0, const float* a_rate0, const float* b_shape0,
                                         const float* b_rate0, const float* alpha_init, const float* b_shape_init,
                                         const float* b_rate_init, const float* a_start, const float* y, float* alpha,
                                         float* a_hat, float* b_shape, float* b_rate, double* free_energy, float* z_prob,
                                         float* hist_a, float* hist_b_shape, float* hist_b_rate, int32_t* status,
                                         unsigned flags) {
    using namespace rxg::gamix;
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "gamma_mixture_vmp takes device pointers");
    if (K < 2 || K > MAX_K) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "gamma_mixture_vmp: K=%d unsupported (2-8)", K);
    const float* host[N_BLOCKS] = {a_shape0, a_rate0, b_shape0, b_rate0, alpha_s, alpha_init, b_shape_init, b_rate_init,
                                   a_start};
    bool null_host = false;
    for (const float* h : host) null_host |= !h;
    if (N < 1 || batch < 1 || iterations < 1 || null_host || !y || !alpha || !a_hat || !b_shape || !b_rate)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gamma_mixture_vmp: bad argument");
    static const char* names[N_BLOCKS] = {"a_shape0", "a_rate0", "b_shape0", "b_rate0", "alpha_s", "alpha_init",
                                          "b_shape_init", "b_rate_init", "a_start"};
    double hp[N_BLOCKS * MAX_K + 2];
    double sa = 0.0, slg = 0.0;
    for (int j = 0; j < N_BLOCKS; ++j)
        for (int k = 0; k < K; ++k) {
            const float v = host[j][k];
            if (!(v > 0.f) || !std::isfinite(v))
                return rxg::fail(ctx, RXG_ERR_BAD_ARG, "gamma_mixture_vmp: %s must be positive and finite (component %d)",
                                 names[j], k);
            hp[j * K + k] = v;
        }
    for (int k = 0; k < K; ++k) {
        // a shape prior below 1 makes the shape objective non-concave near 0: its maximiser need not be unique
        if (a_shape0[k] < 1.f)
            return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "gamma_mixture_vmp: a_shape0 must be >= 1 (component %d: %g)", k,
                             (double)a_shape0[k]);
        sa += alpha_s[k];
        slg += std::lgamma((double)alpha_s[k]);
    }
    hp[N_BLOCKS * K] = sa;
    hp[N_BLOCKS * K + 1] = std::lgamma(sa) - slg;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nbytes = (size_t)n_params(K) * sizeof(double);
    double* dp = (double*)rxg::workspace(ctx, nbytes);
    if (!dp) return RXG_ERR_CUDA;
    RXG_CUDA(ctx, cudaMemcpyAsync(dp, hp, nbytes, cudaMemcpyHostToDevice, ctx->stream));
    const Args a{K, N, iterations, batch, dp, y, alpha, a_hat, b_shape, b_rate, free_energy, z_prob, hist_a,
                 hist_b_shape, hist_b_rate};
    switch (K) {
        case 2: launch<2>(ctx, a, status); break;
        case 3: launch<3>(ctx, a, status); break;
        case 4: launch<4>(ctx, a, status); break;
        case 5: launch<5>(ctx, a, status); break;
        case 6: launch<6>(ctx, a, status); break;
        case 7: launch<7>(ctx, a, status); break;
        default: launch<8>(ctx, a, status); break;
    }
    ctx->launches += 1;
    int rc = rxg::check_cuda(ctx, cudaGetLastError(), "gamma_mixture_vmp_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
