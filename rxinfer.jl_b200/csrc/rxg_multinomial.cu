// rxg_multinomial_polya_vmp_f32 / rxg_multinomial_polya_online_f32: Bayesian multinomial regression of
// test/models/regression/multinomialreg_tests.jl over a batch of chains (step and chain bodies: rxg_multinomial.cuh,
// DESIGN 3.22).  Three kernels, 2 <= K <= 64:
//   mnp_data_kernel:   whole data sets, read once: 32 consecutive chains per CTA (one 128-byte row per category and
//                      sample) x 8 sample slots; per-category totals and the log-coefficient sum, reduced over the slots
//                      in slot order, become each chain's message (b, n, lc) in the workspace;
//   mnp_vmp_kernel:    whole data sets, every iteration: one warp per chain, its q in fp64 shared memory, the prior
//                      shared by the CTA;
//   mnp_online_kernel: datum by datum: one warp per chain, base and q in fp64 shared memory, the carry in and out fp64.
#include <algorithm>
#include <cmath>
#include <vector>

#include "rxg_internal.h"
#include "rxg_multinomial.cuh"

namespace rxg {
namespace mnp {

constexpr int DATA_CHAINS = 32, DATA_SLOTS = 8;
constexpr int MAX_WARPS = 8;
constexpr size_t SMEM_SOFT = 48 * 1024;        // warps per CTA: as many as fit here, at least one

__device__ void fill_log_fact(double* lf, int tid, int nthreads) {
    for (int i = tid; i < LF_N; i += nthreads) lf[i] = lgamma(i + 1.0);
}

// stats[2D + 2][B]: b[D], n[D], lc, bad
template <int KB>
__global__ void __launch_bounds__(DATA_CHAINS* DATA_SLOTS) mnp_data_kernel(int K, int n_samples, int64_t B,
                                                                          const int32_t* __restrict__ y,
                                                                          double* __restrict__ stats) {
    __shared__ double lf[LF_N];
    __shared__ double red[DATA_SLOTS][DATA_CHAINS];
    const int cx = threadIdx.x, slot = threadIdx.y, tid = slot * DATA_CHAINS + cx;
    fill_log_fact(lf, tid, DATA_CHAINS * DATA_SLOTS);
    __syncthreads();
    const int64_t c = (int64_t)blockIdx.x * DATA_CHAINS + cx;
    double Y[KB], lcoef = 0.0, bad = 0.0;
#pragma unroll
    for (int k = 0; k < KB; ++k) Y[k] = 0.0;
    if (c < B)
        for (int i = slot; i < n_samples; i += DATA_SLOTS) {
            int32_t v[KB];
#pragma unroll
            for (int k = 0; k < KB; ++k) v[k] = k < K ? __ldg(y + ((int64_t)i * K + k) * B + c) : 0;
            if (!add_sample<KB>(K, v, lf, Y, lcoef)) bad = 1.0;
        }
    auto reduce = [&](double& v) {
        red[slot][cx] = v;
        __syncthreads();
        if (slot == 0) {
            double s = red[0][cx];
#pragma unroll
            for (int q = 1; q < DATA_SLOTS; ++q) s += red[q][cx];
            v = s;
        }
        __syncthreads();
    };
#pragma unroll
    for (int k = 0; k < KB; ++k)
        if (k < K) reduce(Y[k]);
    reduce(lcoef);
    reduce(bad);
    if (slot == 0 && c < B) {
        const int D = K - 1;
        const double lc = suffix_totals<KB>(K, Y, lcoef);
#pragma unroll
        for (int k = 0; k < KB - 1; ++k)
            if (k < D) {
                stats[(int64_t)k * B + c] = (Y[k] - Y[k + 1]) - 0.5 * Y[k];
                stats[(int64_t)(D + k) * B + c] = Y[k];
            }
        stats[(int64_t)(2 * D) * B + c] = lc;
        stats[(int64_t)(2 * D + 1) * B + c] = bad;
    }
}

// per warp: S [D][D], then m, d, u, r, b, n [D]
__host__ __device__ constexpr size_t vmp_warp_doubles(int D) { return (size_t)D * D + 6 * D; }

__global__ void mnp_vmp_kernel(int D, int iters, const double* __restrict__ prior, const double* __restrict__ stats,
                               Out o, int32_t* __restrict__ status) {
    extern __shared__ double sm[];
    const int W = blockDim.x / 32, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* m0 = sm;                 // the prior, shared: m0 [D], S0 [D][D]
    double* S0 = sm + D;
    for (int i = threadIdx.x; i < D + D * D; i += blockDim.x) sm[i] = prior[i];
    double* p = sm + D + D * D + warp * vmp_warp_doubles(D);
    const Work w{p, p + D * D, p + D * D + D, p + D * D + 2 * D, p + D * D + 3 * D};
    double *b = p + D * D + 4 * D, *n = p + D * D + 5 * D;
    const int64_t B = o.batch, c = (int64_t)blockIdx.x * W + warp;
    __syncthreads();
    if (c >= B) return;
    for (int k = lane; k < D; k += 32) {
        b[k] = stats[(int64_t)k * B + c];
        n[k] = stats[(int64_t)(D + k) * B + c];
    }
    const double lc = stats[(int64_t)(2 * D) * B + c];
    int st = stats[(int64_t)(2 * D + 1) * B + c] != 0.0 ? ST_BAD : 0;
    __syncwarp();
    offline(lane, 32, D, iters, m0, S0, b, n, lc, w, o, c, st);
    if (lane == 0 && status) status[c] = st;
}

// per warp: base S, q S [D][D], then base m, q m, d, u, r, b, n [D], then the counts (MAX_K int32 = MAX_K / 2 doubles)
__host__ __device__ constexpr size_t online_warp_doubles(int D) { return 2 * (size_t)D * D + 7 * D + MAX_K / 2; }

__global__ void mnp_online_kernel(int K, int T, int iters, const double* __restrict__ prior, const double* m_in,
                                  const double* S_in, const int32_t* __restrict__ y, double* m_out, double* S_out, Out o,
                                  int32_t* __restrict__ status) {
    extern __shared__ double sm[];
    const int D = K - 1, W = blockDim.x / 32, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* lf = sm;
    fill_log_fact(lf, threadIdx.x, blockDim.x);
    double* p = sm + LF_N + warp * online_warp_doubles(D);
    const int DD = D * D;
    Work base{p, p + 2 * DD, p + 2 * DD + 2 * D, p + 2 * DD + 3 * D, p + 2 * DD + 4 * D};
    Work w{p + DD, p + 2 * DD + D, base.d, base.u, base.r};
    double *b = p + 2 * DD + 5 * D, *n = p + 2 * DD + 6 * D;
    int32_t* cnt = (int32_t*)(p + 2 * DD + 7 * D);
    const int64_t B = o.batch, c = (int64_t)blockIdx.x * W + warp;
    __syncthreads();
    if (c >= B) return;
    for (int j = lane; j < D; j += 32) {
        base.m[j] = m_in ? m_in[(int64_t)j * B + c] : prior[j];
        for (int i = 0; i < D; ++i) base.S[i * D + j] = S_in ? S_in[((int64_t)i * D + j) * B + c] : prior[D + i * D + j];
    }
    __syncwarp();
    int st = 0;
    online<(MAX_K + 31) / 32>(lane, 32, K, T, iters, y, c, lf, base, w, cnt, b, n, o, st);
    for (int j = lane; j < D; j += 32) {
        m_out[(int64_t)j * B + c] = base.m[j];
        for (int i = 0; i < D; ++i) S_out[((int64_t)i * D + j) * B + c] = base.S[i * D + j];
    }
    if (lane == 0 && status) status[c] = st;
}

// warps per CTA and dynamic shared bytes for per-warp and per-CTA fp64 counts
void shape(size_t per_warp, size_t per_cta, int* warps, size_t* bytes) {
    const size_t pw = per_warp * sizeof(double), pc = per_cta * sizeof(double);
    int W = SMEM_SOFT > pc + pw ? (int)((SMEM_SOFT - pc) / pw) : 1;
    W = std::max(1, std::min(W, MAX_WARPS));
    *warps = W;
    *bytes = pc + W * pw;
}

template <class Kernel>
int set_smem(rxg_ctx* ctx, Kernel k, size_t bytes) {
    if (bytes > SMEM_SOFT) RXG_CUDA(ctx, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return RXG_OK;
}

// The prior block shared by every chain, m0 = W0^-1 xi0 [D] then S0 = W0^-1 [D][D], fp64 from one Cholesky of the
// symmetrised W0; false if W0 is not symmetric positive definite (or not finite).
bool prior_block(const float* xi0, const float* W0, int D, double* out) {
    std::vector<double> L((size_t)D * D, 0.0), Li((size_t)D * D, 0.0);
    for (int i = 0; i < D; ++i) {
        if (!std::isfinite(xi0[i])) return false;
        for (int j = 0; j <= i; ++j) {
            double s = 0.5 * ((double)W0[i * D + j] + (double)W0[j * D + i]);
            for (int k = 0; k < j; ++k) s -= L[i * D + k] * L[j * D + k];
            if (i == j) {
                if (!(s > 0.0) || !std::isfinite(s)) return false;
                L[i * D + i] = std::sqrt(s);
            } else {
                L[i * D + j] = s / L[j * D + j];
            }
        }
    }
    for (int j = 0; j < D; ++j) {            // Li = L^-1, lower
        Li[j * D + j] = 1.0 / L[j * D + j];
        for (int i = j + 1; i < D; ++i) {
            double s = 0.0;
            for (int k = j; k < i; ++k) s -= L[i * D + k] * Li[k * D + j];
            Li[i * D + j] = s / L[i * D + i];
        }
    }
    double* m0 = out;
    double* S0 = out + D;
    for (int i = 0; i < D; ++i)
        for (int j = 0; j < D; ++j) {
            double s = 0.0;
            for (int k = std::max(i, j); k < D; ++k) s += Li[k * D + i] * Li[k * D + j];
            S0[i * D + j] = s;
        }
    for (int i = 0; i < D; ++i) {
        double s = 0.0;
        for (int j = 0; j < D; ++j) s += S0[i * D + j] * (double)xi0[j];
        m0[i] = s;
    }
    return true;
}

bool symmetric(const float* W0, int D) {
    for (int i = 0; i < D; ++i)
        for (int j = 0; j < i; ++j) {
            const double u = W0[i * D + j], v = W0[j * D + i];
            if (!(std::fabs(u - v) <= 1e-6 * (std::fabs(u) + std::fabs(v)))) return false;
        }
    return true;
}

int check_prior(rxg_ctx* ctx, const char* who, const float* xi0, const float* W0, int D, double* block) {
    if (!symmetric(W0, D)) return fail(ctx, RXG_ERR_BAD_ARG, "%s: W0 is not symmetric", who);
    if (!prior_block(xi0, W0, D, block))
        return fail(ctx, RXG_ERR_BAD_ARG, "%s: xi0 must be finite and W0 symmetric positive definite", who);
    return RXG_OK;
}

}  // namespace mnp
}  // namespace rxg

extern "C" int rxg_multinomial_polya_vmp_f32(rxg_ctx* ctx, int K, int n, int64_t batch, int iterations, const float* xi0,
                                             const float* W0, const int32_t* y, float* psi_mean, float* psi_cov,
                                             double* free_energy, float* hist_mean, float* hist_cov, int32_t* status,
                                             unsigned flags) {
    using namespace rxg::mnp;
    const char* who = "multinomial_polya_vmp";
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "%s takes device pointers", who);
    if (K < 2 || K > MAX_K) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "%s: K=%d unsupported (2-64)", who, K);
    if (n < 1 || batch < 1 || iterations < 1 || !xi0 || !W0 || !y || !psi_mean)
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "%s: bad argument", who);
    const int D = K - 1;
    std::vector<double> block((size_t)D + (size_t)D * D);
    if (int rc = check_prior(ctx, who, xi0, W0, D, block.data())) return rc;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const size_t nprior = block.size(), nstats = (size_t)(2 * D + 2) * (size_t)batch;
    double* ws = (double*)rxg::workspace(ctx, (nprior + nstats) * sizeof(double));
    if (!ws) return RXG_ERR_CUDA;
    double* stats = ws + nprior;
    RXG_CUDA(ctx, cudaMemcpyAsync(ws, block.data(), nprior * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    const dim3 dgrid((unsigned)((batch + DATA_CHAINS - 1) / DATA_CHAINS)), dblock(DATA_CHAINS, DATA_SLOTS);
    if (K <= 8) mnp_data_kernel<8><<<dgrid, dblock, 0, ctx->stream>>>(K, n, batch, y, stats);
    else if (K <= 16) mnp_data_kernel<16><<<dgrid, dblock, 0, ctx->stream>>>(K, n, batch, y, stats);
    else if (K <= 32) mnp_data_kernel<32><<<dgrid, dblock, 0, ctx->stream>>>(K, n, batch, y, stats);
    else mnp_data_kernel<64><<<dgrid, dblock, 0, ctx->stream>>>(K, n, batch, y, stats);
    ctx->launches += 1;
    if (int rc = rxg::check_cuda(ctx, cudaGetLastError(), "mnp_data_kernel")) return rc;
    int W;
    size_t bytes;
    shape(vmp_warp_doubles(D), nprior, &W, &bytes);
    if (int rc = set_smem(ctx, mnp_vmp_kernel, bytes)) return rc;
    const Out o{batch, psi_mean, psi_cov, hist_mean, hist_cov, free_energy};
    mnp_vmp_kernel<<<(unsigned)((batch + W - 1) / W), 32 * W, bytes, ctx->stream>>>(D, iterations, ws, stats, o, status);
    ctx->launches += 1;
    if (int rc = rxg::check_cuda(ctx, cudaGetLastError(), "mnp_vmp_kernel")) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

extern "C" int rxg_multinomial_polya_online_f32(rxg_ctx* ctx, int K, int T, int64_t batch, int iterations,
                                                const float* xi0, const float* W0, const double* m_in, const double* S_in,
                                                const int32_t* y, double* m_out, double* S_out, float* hist_mean,
                                                float* hist_cov, double* free_energy, int32_t* status, unsigned flags) {
    using namespace rxg::mnp;
    const char* who = "multinomial_polya_online";
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "%s takes device pointers", who);
    if (K < 2 || K > MAX_K) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "%s: K=%d unsupported (2-64)", who, K);
    if (T < 1 || batch < 1 || iterations < 1 || !xi0 || !W0 || !y || !m_out || !S_out || (!m_in != !S_in))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "%s: bad argument (m_in and S_in are given together or not at all)", who);
    const int D = K - 1;
    std::vector<double> block((size_t)D + (size_t)D * D);
    if (int rc = check_prior(ctx, who, xi0, W0, D, block.data())) return rc;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    double* ws = (double*)rxg::workspace(ctx, block.size() * sizeof(double));
    if (!ws) return RXG_ERR_CUDA;
    RXG_CUDA(ctx, cudaMemcpyAsync(ws, block.data(), block.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    int W;
    size_t bytes;
    shape(online_warp_doubles(D), LF_N, &W, &bytes);
    if (int rc = set_smem(ctx, mnp_online_kernel, bytes)) return rc;
    const Out o{batch, nullptr, nullptr, hist_mean, hist_cov, free_energy};
    mnp_online_kernel<<<(unsigned)((batch + W - 1) / W), 32 * W, bytes, ctx->stream>>>(K, T, iterations, ws, m_in, S_in, y,
                                                                                      m_out, S_out, o, status);
    ctx->launches += 1;
    if (int rc = rxg::check_cuda(ctx, cudaGetLastError(), "mnp_online_kernel")) return rc;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
