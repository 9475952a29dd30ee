// rxg_binomial_polya_vmp_f32: Bayesian binomial / logistic regression of test/models/regression/binomialreg_tests.jl as one
// launch over a batch of chains (kernel body: rxg_polya.cuh, DESIGN 3.21).  Two kernels, p = 1..8 compiled:
//   polya_thread_kernel: one thread per chain; lane = chain, so each warp load of a feature is one 128-byte row;
//   polya_group_kernel:  GROUP consecutive chains per CTA, SLOTS threads per chain striding over its samples; per pass the
//                        sums are reduced per chain (shuffles, then shared memory in warp order), one thread per chain
//                        makes the new q and shares it with the others.  A chain's reduction order depends only on N.
// RXG_OPT_POLYA_PATH forces one of them; by default select_path() picks.
#include <cmath>

#include "rxg_internal.h"
#include "rxg_polya.cuh"

namespace rxg {
namespace polya {

constexpr int THREAD_TPB = 128;

template <int P>
__global__ void __launch_bounds__(THREAD_TPB) polya_thread_kernel(Args a, Prior pr, int32_t* __restrict__ status) {
    const int64_t b = (int64_t)blockIdx.x * THREAD_TPB + threadIdx.x;
    if (b >= a.batch) return;
    const int st = chain<P>(b, a, pr);
    if (status) status[b] = st;
}

template <int P>
__global__ void __launch_bounds__(GROUP_THREADS, 1) polya_group_kernel(Args a, Prior pr, int32_t* __restrict__ status) {
    constexpr int NL = nw::packed(P), NR = NL + P + 2;       // reduced per chain: L, then (first pass) xi_d, lc; g
    constexpr int WARPS = GROUP_THREADS / 32;
    __shared__ double red[WARPS][GROUP][NR];
    __shared__ double first_sums[GROUP][P + 1];                // xi_d, lc of the first pass
    __shared__ Q<P> qs[GROUP];
    __shared__ int sbad[GROUP];
    const int tid = threadIdx.x, c = tid % GROUP, slot = tid / GROUP, lane = tid & 31, warp = tid >> 5;
    const int64_t b = (int64_t)blockIdx.x * GROUP + c;
    const bool valid = b < a.batch;
    if (tid < GROUP) sbad[tid] = 0;
    __syncthreads();
    Q<P> q;
    init_q<P>(pr, q);
    Acc<P> acc;
#pragma unroll
    for (int j = 0; j < P; ++j) acc.xi[j] = 0.0;
    acc.lc = 0.0;
    acc.bad = false;
    double fk = 0.0;
    int st = 0;
    const int np = passes(a);
    for (int k = 0; k < np; ++k) {
        zero_pass<P>(acc);
        const bool first = k == 0, want_g = a.fe && k >= 1, want_lc = a.fe != nullptr;
        if (valid && slot < a.N) {
            float x[P], xn[P];
            int y, n, yn = 0, nn = 0;
            load<P>(a, slot, b, x, y, n);
            for (int i = slot; i < a.N; i += SLOTS) {
                if (i + SLOTS < a.N) load<P>(a, i + SLOTS, b, xn, yn, nn);
                sample<P>(x, y, n, q, acc, first, want_lc, want_g);
#pragma unroll
                for (int j = 0; j < P; ++j) x[j] = xn[j];
                y = yn;
                n = nn;
            }
        }
        if (first && acc.bad) atomicOr(&sbad[c], 1);
        // lanes c, c + 8, c + 16, c + 24 of a warp hold chain c: two butterfly steps, then the warps in order
        auto put = [&](int r, double v) {
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            if (lane < GROUP) red[warp][lane][r] = v;
        };
#pragma unroll
        for (int t = 0; t < NL; ++t) put(t, acc.L[t]);
        put(NR - 1, acc.g);
        if (first) {
#pragma unroll
            for (int j = 0; j < P; ++j) put(NL + j, acc.xi[j]);
            put(NL + P, acc.lc);
        }
        __syncthreads();
        if (tid < GROUP) {
            Acc<P> tot;
            zero_pass<P>(tot);
#pragma unroll
            for (int w = 0; w < WARPS; ++w) {
#pragma unroll
                for (int t = 0; t < NL; ++t) tot.L[t] += red[w][c][t];
                tot.g += red[w][c][NR - 1];
            }
            if (first)
#pragma unroll
                for (int j = 0; j <= P; ++j) {
                    double s = 0.0;
#pragma unroll
                    for (int w = 0; w < WARPS; ++w) s += red[w][c][NL + j];
                    first_sums[c][j] = s;
                }
#pragma unroll
            for (int j = 0; j < P; ++j) tot.xi[j] = first_sums[c][j];
            tot.lc = first_sums[c][P];
            tot.bad = sbad[c] != 0;
            if (valid) end_pass<P>(k, b, a, pr, tot, q, fk, st);
            qs[c] = q;
        }
        __syncthreads();
        q = qs[c];
    }
    if (tid < GROUP && valid && status) status[b] = st;
}

template <int P>
void launch(cudaStream_t s, int path, const Args& a, const Prior& pr, int32_t* status) {
    if (path == PATH_GROUP)
        polya_group_kernel<P><<<(unsigned)((a.batch + GROUP - 1) / GROUP), GROUP_THREADS, 0, s>>>(a, pr, status);
    else
        polya_thread_kernel<P><<<(unsigned)((a.batch + THREAD_TPB - 1) / THREAD_TPB), THREAD_TPB, 0, s>>>(a, pr, status);
}

}  // namespace polya
}  // namespace rxg

extern "C" int rxg_binomial_polya_vmp_f32(rxg_ctx* ctx, int p, int N, int64_t batch, int iterations, const float* xi0,
                                          const float* W0, const float* X, const int32_t* y, const int32_t* ntrials,
                                          float* beta_mean, float* beta_cov, double* free_energy, float* hist_mean,
                                          float* hist_cov, int32_t* status, unsigned flags) {
    using namespace rxg::polya;
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "binomial_polya_vmp takes device pointers");
    if (p < 1 || p > MAX_P) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "binomial_polya_vmp: p=%d unsupported (1-8)", p);
    if (N < 1 || batch < 1 || iterations < 1 || !xi0 || !W0 || !X || !y || !beta_mean)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "binomial_polya_vmp: bad argument");
    const long long opt = ctx->opt[RXG_OPT_POLYA_PATH];
    if (opt < PATH_AUTO || opt > PATH_GROUP)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "binomial_polya_vmp: RXG_OPT_POLYA_PATH=%lld (0 auto, 1 thread, 2 group)", opt);
    Prior pr{};
    for (int i = 0; i < p; ++i) {
        if (!std::isfinite(xi0[i])) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "binomial_polya_vmp: xi0 must be finite");
        for (int j = 0; j < p; ++j) {
            const double u = W0[i * p + j], v = W0[j * p + i];
            if (!(std::fabs(u - v) <= 1e-6 * (std::fabs(u) + std::fabs(v))))
                return rxg::fail(ctx, RXG_ERR_BAD_ARG, "binomial_polya_vmp: W0 is not symmetric");
            pr.W0[i * MAX_P + j] = u;
        }
        pr.xi0[i] = xi0[i];
    }
    double S0[MAX_P * MAX_P];
    if (!rxg::host_spd_inv(W0, p, S0, &pr.logdetW0))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "binomial_polya_vmp: W0 is not symmetric positive definite");
    pr.quad0 = 0.0;
    for (int i = 0; i < p; ++i) {
        double t = 0.0;
        for (int j = 0; j < p; ++j) {
            pr.S0[i * MAX_P + j] = S0[i * p + j];
            t += S0[i * p + j] * pr.xi0[j];
        }
        pr.m0[i] = t;
        pr.quad0 += pr.xi0[i] * t;
    }
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const Args a{N, iterations, batch, X, y, ntrials, beta_mean, beta_cov, free_energy, hist_mean, hist_cov};
    const int path = opt != PATH_AUTO ? (int)opt : select_path(batch, N, p, ctx->sm_count);
    switch (p) {
        case 1: launch<1>(ctx->stream, path, a, pr, status); break;
        case 2: launch<2>(ctx->stream, path, a, pr, status); break;
        case 3: launch<3>(ctx->stream, path, a, pr, status); break;
        case 4: launch<4>(ctx->stream, path, a, pr, status); break;
        case 5: launch<5>(ctx->stream, path, a, pr, status); break;
        case 6: launch<6>(ctx->stream, path, a, pr, status); break;
        case 7: launch<7>(ctx->stream, path, a, pr, status); break;
        default: launch<8>(ctx->stream, path, a, pr, status); break;
    }
    ctx->launches += 1;
    const int rc = rxg::check_cuda(ctx, cudaGetLastError(), path == PATH_GROUP ? "polya_group_kernel" : "polya_thread_kernel");
    if (rc != RXG_OK) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
