// rxg_hgf_vmp_learn_f32: the HGF with learned kappa and omega per series (kernel body: rxg_hgf_learn.cuh).  One thread per
// chain, every iteration in one launch.  The unit keeps its own Gauss-Hermite table in constant memory, filled by the
// host routine of rxg_hgf.cu.
#include <cmath>

#include "rxg_internal.h"
#include "rxg_hgf_learn.cuh"

namespace rxg {
namespace hgfl {

constexpr int TPB = 64;

__constant__ GH c_gh;

// The fp64 fold sums and, with the free energy, the old marginals of the previous iteration need more than the 128
// registers at which 65 536 chains would fit the 132 SMs in one wave; below 168 the free-energy variant spills.
template <bool FE>
__global__ void __maxnreg__(168) hgf_learn_kernel(Args a, int32_t* __restrict__ status) {
    const int64_t b = (int64_t)blockIdx.x * TPB + threadIdx.x;
    if (b >= a.batch) return;
    const int st = chain<FE>(b, a, c_gh);
    if (status) status[b] = st;
}

int ensure_tables(rxg_ctx* ctx) {
    if (ctx->gh_learn_ready) return RXG_OK;
    double t[NGH], w[NGH];
    gauss_hermite_31(t, w);
    GH h;
    for (int i = 0; i < NGH; ++i) { h.t[i] = (float)t[i]; h.lw2[i] = (float)std::log2(w[i]); }
    fill_vfix(h);
    RXG_CUDA(ctx, cudaMemcpyToSymbol(c_gh, &h, sizeof(h)));
    ctx->gh_learn_ready = true;
    return RXG_OK;
}

}  // namespace hgfl
}  // namespace rxg

namespace {

bool positive(float v) { return v > 0.f && std::isfinite(v); }

}  // namespace

extern "C" int rxg_hgf_vmp_learn_f32(rxg_ctx* ctx, int T, int64_t batch, int iterations, const float prior[8],
                                     float z_precision, float y_variance, const float init[8], const float* y, float* x0,
                                     float* xz, float* kw, float* hist_kw, double* free_energy, int32_t* status,
                                     unsigned flags) {
    using namespace rxg::hgfl;
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (T < 1 || batch < 1 || iterations < 1 || !prior || !init || !y || !xz || !kw)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hgf_vmp_learn: bad argument");
    for (int i = 0; i < 8; ++i)
        if (!std::isfinite(prior[i]) || !std::isfinite(init[i]))
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hgf_vmp_learn: prior and init must be finite");
    if (!positive(prior[1]) || !positive(prior[3]) || !positive(prior[5]) || !positive(prior[7]) || !positive(z_precision) ||
        !positive(y_variance))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hgf_vmp_learn: prior variances, z_precision and y_variance must be positive");
    if (!positive(init[1]) || !positive(init[3]) || !positive(init[5]) || !positive(init[7]))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "hgf_vmp_learn: initial variances must be positive");
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "hgf_vmp_learn takes device pointers");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = ensure_tables(ctx);
    if (rc != RXG_OK) return rc;
    Args a{T, iterations, batch,
           Prm{prior[0], prior[1], prior[2], prior[3], prior[4], prior[5], prior[6], prior[7], z_precision, y_variance,
               init[0], init[1], init[2], init[3], init[4], init[5], init[6], init[7]},
           y, x0, xz, kw, hist_kw, free_energy};
    const unsigned grid = (unsigned)((batch + TPB - 1) / TPB);
    if (free_energy)
        hgf_learn_kernel<true><<<grid, TPB, 0, ctx->stream>>>(a, status);
    else
        hgf_learn_kernel<false><<<grid, TPB, 0, ctx->stream>>>(a, status);
    ctx->launches += 1;
    rc = rxg::check_cuda(ctx, cudaGetLastError(), "hgf_learn_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
