// lgssm_generic_chain_kernel: the full (mu, Sigma) recursion of ONE chain per CTA for any state / observation
// size up to 64, runtime d and m.  This is the general-shape member of the per-chain family
// (lgssm_chain_kernel keeps d <= 6 in registers, one thread per chain): per-chain models
// (RXG_MODEL_PER_CHAIN), missing data (ymask), transition offsets and RXG_PATH_PER_CHAIN for d, m that the
// register-resident kernels do not cover -- the reference has no restriction on d and m
// [ref: /root/reference/test/models/statespace/mlgssm_test.jl:8-17 (any-size MvNormal chain);
//  missing data docs/src/manuals/inference/static.md:98-125].
//
// Same message algebra as lgssm_chain_kernel (Kalman-gain / RTS form of rules #1-#4, #3', #4 and the products,
// one Cholesky per direction).  All matrices live in shared memory (row-major, leading dimension n + 1), every
// operation is block-cooperative over 256 threads; the filtered (mu, Sigma) are stashed in the output buffers and
// overwritten by the smoothed ones on the way back.  fp32 storage and arithmetic like the register kernels.
// Throughput is that of a CUDA-core fallback: ~800 barrier-separated phases per step with little work each; a variant
// with block-parallel triangular solves (two barriers per row) was slower.
// The shared-model gain-table families remain the fast path; a tensor-core per-chain recursion is the open item.
#include <math.h>

#include "rxg_internal.h"

namespace rxg {

namespace {

struct GenArgs {
    int d, m, T;
    int64_t batch;
    int per_chain;                       // model arrays carry a trailing [batch] axis
    const float *A, *B, *P, *Q, *m0, *S0, *u;     // device pointers (shared: row-major; per chain: [..][batch])
    const float* mean0_chain;            // [d][batch] or null
    const float* useq;                   // per-step inputs (replace u): row t at useq + t * d * ustride (+ b if uchain)
    int64_t ustride;
    int uchain;
    const float* y;
    const uint8_t* mask;
    float *mean, *cov, *nle;
    int32_t* status;
    int smooth, transition_first;
};

// C (r x c) = X (r x k) * Y (k x c)  [+ Add];  all row-major with leading dimension ld
__device__ void g_mul_nn(float* C, const float* X, const float* Y, const float* Add, int r, int c, int k, int ld) {
    for (int e = threadIdx.x; e < r * c; e += blockDim.x) {
        const int i = e / c, j = e % c;
        float s = Add ? Add[i * ld + j] : 0.f;
        for (int q = 0; q < k; ++q) s = __fmaf_rn(X[i * ld + q], Y[q * ld + j], s);
        C[i * ld + j] = s;
    }
    __syncthreads();
}
// C (r x c) = X (r x k) * Y' (Y is c x k)  [+ Add]
__device__ void g_mul_nt(float* C, const float* X, const float* Y, const float* Add, int r, int c, int k, int ld) {
    for (int e = threadIdx.x; e < r * c; e += blockDim.x) {
        const int i = e / c, j = e % c;
        float s = Add ? Add[i * ld + j] : 0.f;
        for (int q = 0; q < k; ++q) s = __fmaf_rn(X[i * ld + q], Y[j * ld + q], s);
        C[i * ld + j] = s;
    }
    __syncthreads();
}
// symmetric C (n x n) = X (n x k) * Y' + Add, computed on the lower triangle and mirrored (exactly symmetric)
__device__ void g_sym_nt(float* C, const float* X, const float* Y, const float* Add, int n, int k, int ld) {
    for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
        const int i = e / n, j = e % n;
        if (j > i) continue;
        float s = Add ? Add[i * ld + j] : 0.f;
        for (int q = 0; q < k; ++q) s = __fmaf_rn(X[i * ld + q], Y[j * ld + q], s);
        C[i * ld + j] = s;
        C[j * ld + i] = s;
    }
    __syncthreads();
}
// S (n x n, symmetric) -= V' V with V (k x n): lower triangle + mirror
__device__ void g_downdate_tn(float* S, const float* V, int n, int k, int ld) {
    for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
        const int i = e / n, j = e % n;
        if (j > i) continue;
        float s = S[i * ld + j];
        for (int q = 0; q < k; ++q) s = __fmaf_rn(-V[q * ld + i], V[q * ld + j], s);
        S[i * ld + j] = s;
        S[j * ld + i] = s;
    }
    __syncthreads();
}
// in-place lower Cholesky of the n x n matrix A (right-looking, one column per round); returns false on a
// non-positive pivot (the pivot is clamped so that the sweep finishes; the chain is flagged)
__device__ bool g_chol(float* A, int n, int ld, float* s_scal) {
    bool ok = true;
    for (int j = 0; j < n; ++j) {
        if (threadIdx.x == 0) {
            float dj = A[j * ld + j];
            if (!(dj > 0.f)) { dj = 1e-30f; s_scal[1] = 1.f; }
            s_scal[0] = sqrtf(dj);
        }
        __syncthreads();
        const float ljj = s_scal[0], inv = 1.0f / ljj;
        if (threadIdx.x == 0) A[j * ld + j] = ljj;
        for (int i = j + 1 + threadIdx.x; i < n; i += blockDim.x) A[i * ld + j] *= inv;
        __syncthreads();
        // trailing update of the lower triangle: A[i][k] -= A[i][j] A[k][j], j < k <= i
        const int rem = n - j - 1;
        for (int e = threadIdx.x; e < rem * rem; e += blockDim.x) {
            const int i = j + 1 + e / rem, k = j + 1 + e % rem;
            if (k <= i) A[i * ld + k] = __fmaf_rn(-A[i * ld + j], A[k * ld + j], A[i * ld + k]);
        }
        __syncthreads();
    }
    if (s_scal[1] != 0.f) ok = false;
    return ok;
}
// X (n x c) <- L^-1 X, one thread per column (forward substitution)
__device__ void g_trsm_lower(const float* L, float* X, int n, int c, int ld) {
    for (int col = threadIdx.x; col < c; col += blockDim.x)
        for (int i = 0; i < n; ++i) {
            float s = X[i * ld + col];
            for (int k = 0; k < i; ++k) s = __fmaf_rn(-L[i * ld + k], X[k * ld + col], s);
            X[i * ld + col] = s / L[i * ld + i];
        }
    __syncthreads();
}
// X (n x c) <- L^-T X (backward substitution)
__device__ void g_trsm_lower_t(const float* L, float* X, int n, int c, int ld) {
    for (int col = threadIdx.x; col < c; col += blockDim.x)
        for (int i = n - 1; i >= 0; --i) {
            float s = X[i * ld + col];
            for (int k = i + 1; k < n; ++k) s = __fmaf_rn(-L[k * ld + i], X[k * ld + col], s);
            X[i * ld + col] = s / L[i * ld + i];
        }
    __syncthreads();
}
// out (r) = X (r x k) v  [+ add];   out' = X' v variant below
__device__ void g_mulv(float* out, const float* X, const float* v, const float* add, int r, int k, int ld, float sign = 1.f) {
    for (int i = threadIdx.x; i < r; i += blockDim.x) {
        float s = 0.f;
        for (int q = 0; q < k; ++q) s = __fmaf_rn(X[i * ld + q], v[q], s);
        out[i] = (add ? add[i] : 0.f) + sign * s;
    }
    __syncthreads();
}
__device__ void g_mulv_t(float* out, const float* X, const float* v, const float* add, int r, int k, int ld) {   // out (r) = X' v, X is k x r
    for (int i = threadIdx.x; i < r; i += blockDim.x) {
        float s = 0.f;
        for (int q = 0; q < k; ++q) s = __fmaf_rn(X[q * ld + i], v[q], s);
        out[i] = (add ? add[i] : 0.f) + s;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(256) lgssm_generic_chain_kernel(GenArgs g) {
    extern __shared__ float sm[];
    const int d = g.d, m = g.m, n = d > m ? d : m, ld = n + 1;
    const size_t msz = (size_t)n * ld;
    float* sA = sm;                 // d x d
    float* sB = sA + msz;           // m x d      (backward: C = Sf - U'U)
    float* sP = sB + msz;           // d x d
    float* sQ = sP + msz;           // m x m      (backward: T3 = Ss+ G')
    float* sS = sQ + msz;           // current covariance
    float* sT = sS + msz;           // scratch
    float* sL = sT + msz;           // Cholesky factor
    float* sX = sL + msz;           // smoothed covariance of the next step (backward)
    float* v_mu = sX + msz;         // d
    float* v_e = v_mu + n;          // m (innovation / whitened innovation), d in the backward pass
    float* v_t = v_e + n;           // scratch
    float* v_u = v_t + n;           // offset
    float* v_ms = v_u + n;          // smoothed mean of the next step
    float* s_scal = v_ms + n;       // [0] pivot, [1] failure flag

    for (int64_t b = blockIdx.x; b < g.batch; b += gridDim.x) {
        // ---- model into shared memory
        const int64_t st = g.per_chain ? g.batch : 1;
        const int64_t ob = g.per_chain ? b : 0;
        for (int e = threadIdx.x; e < d * d; e += blockDim.x) {
            const int i = e / d, j = e % d;
            sA[i * ld + j] = g.A[(int64_t)e * st + ob];
            sP[i * ld + j] = g.P[(int64_t)e * st + ob];
            sS[i * ld + j] = g.S0[(int64_t)e * st + ob];
        }
        for (int e = threadIdx.x; e < m * d; e += blockDim.x) sB[(e / d) * ld + e % d] = g.B[(int64_t)e * st + ob];
        for (int e = threadIdx.x; e < m * m; e += blockDim.x) sQ[(e / m) * ld + e % m] = g.Q[(int64_t)e * st + ob];
        for (int i = threadIdx.x; i < d; i += blockDim.x) {
            v_mu[i] = g.mean0_chain ? g.mean0_chain[(int64_t)i * g.batch + b] : g.m0[(int64_t)i * st + ob];
            v_u[i] = g.u ? g.u[(int64_t)i * st + ob] : 0.f;
        }
        if (threadIdx.x == 0) s_scal[1] = 0.f;
        __syncthreads();
        double acc = 0.0;                        // evidence (thread 0)
        // ---------------------------------------------------------------- forward
        for (int t = 0; t < g.T; ++t) {
            if (t > 0 || g.transition_first) {
                if (g.useq) {
                    for (int i = threadIdx.x; i < d; i += blockDim.x) v_u[i] = g.useq[((int64_t)t * d + i) * g.ustride + b * g.uchain];
                    __syncthreads();
                }
                g_mulv(v_t, sA, v_mu, v_u, d, d, ld);                 // mu <- A mu + u
                for (int i = threadIdx.x; i < d; i += blockDim.x) v_mu[i] = v_t[i];
                g_mul_nn(sT, sA, sS, nullptr, d, d, d, ld);           // T = A S
                g_sym_nt(sS, sT, sA, sP, d, d, ld);                   // S = T A' + P
            }
            const bool observed = g.mask ? (g.mask[(int64_t)t * g.batch + b] != 0) : true;
            if (observed) {
                g_mul_nn(sT, sB, sS, nullptr, m, d, d, ld);           // T = B S            (m x d)
                g_sym_nt(sL, sT, sB, sQ, m, d, ld);                   // L = T B' + Q       (m x m)
                g_chol(sL, m, ld, s_scal);
                g_trsm_lower(sL, sT, m, d, ld);                       // T = L^-1 B S  =: V' (m x d)
                for (int k = threadIdx.x; k < m; k += blockDim.x) {   // e = y - B mu
                    float s = g.y[((int64_t)t * m + k) * g.batch + b];
                    for (int q = 0; q < d; ++q) s = __fmaf_rn(-sB[k * ld + q], v_mu[q], s);
                    v_e[k] = s;
                }
                __syncthreads();
                if (threadIdx.x == 0) {                               // z = L^-1 e (sequential: m <= 64)
                    float q2 = 0.f, ldet = 0.f;
                    for (int i = 0; i < m; ++i) {
                        float s = v_e[i];
                        for (int k = 0; k < i; ++k) s = __fmaf_rn(-sL[i * ld + k], v_e[k], s);
                        s /= sL[i * ld + i];
                        v_e[i] = s;
                        q2 = __fmaf_rn(s, s, q2);
                        ldet += logf(sL[i * ld + i]);
                    }
                    acc += (double)(0.5f * q2 + ldet) + m * 0.91893853320467274178;
                }
                __syncthreads();
                g_mulv_t(v_t, sT, v_e, v_mu, d, m, ld);               // mu += V z
                for (int i = threadIdx.x; i < d; i += blockDim.x) v_mu[i] = v_t[i];
                g_downdate_tn(sS, sT, d, m, ld);                      // S -= V V'
            }
            // filtered (mu, Sigma): the filter's output, the smoother's stash
            for (int i = threadIdx.x; i < d; i += blockDim.x) g.mean[((int64_t)t * d + i) * g.batch + b] = v_mu[i];
            for (int e = threadIdx.x; e < d * d; e += blockDim.x)
                g.cov[((int64_t)t * d * d + e) * g.batch + b] = sS[(e / d) * ld + e % d];
            __syncthreads();
        }
        if (g.nle && threadIdx.x == 0) g.nle[b] = (float)acc;
        // ---------------------------------------------------------------- backward (RTS, PSD-sum form)
        if (g.smooth) {
            for (int e = threadIdx.x; e < d * d; e += blockDim.x) sX[(e / d) * ld + e % d] = sS[(e / d) * ld + e % d];
            for (int i = threadIdx.x; i < d; i += blockDim.x) v_ms[i] = v_mu[i];
            __syncthreads();
            float* sC = sB;      // the observation model is not needed any more
            float* sT3 = sQ;
            for (int t = g.T - 2; t >= 0; --t) {
                for (int e = threadIdx.x; e < d * d; e += blockDim.x)
                    sS[(e / d) * ld + e % d] = g.cov[((int64_t)t * d * d + e) * g.batch + b];
                for (int i = threadIdx.x; i < d; i += blockDim.x) v_mu[i] = g.mean[((int64_t)t * d + i) * g.batch + b];
                if (g.useq)       // the transition into x[t+1]
                    for (int i = threadIdx.x; i < d; i += blockDim.x) v_u[i] = g.useq[((int64_t)(t + 1) * d + i) * g.ustride + b * g.uchain];
                __syncthreads();
                g_mul_nn(sT, sA, sS, nullptr, d, d, d, ld);           // T = A Sf
                g_sym_nt(sL, sT, sA, sP, d, d, ld);                   // L = A Sf A' + P = Sp(t+1)
                g_chol(sL, d, ld, s_scal);
                g_trsm_lower(sL, sT, d, d, ld);                       // T = L^-1 A Sf =: U'
                for (int e = threadIdx.x; e < d * d; e += blockDim.x) sC[(e / d) * ld + e % d] = sS[(e / d) * ld + e % d];
                __syncthreads();
                g_downdate_tn(sC, sT, d, d, ld);                      // C = Sf - U U'   (cov(x_t | x_t+1))
                g_trsm_lower_t(sL, sT, d, d, ld);                     // T = L^-T U' = G'
                g_mul_nn(sT3, sX, sT, nullptr, d, d, d, ld);          // T3 = Ss+ G'
                // Ss = C + G T3 = C + (G')' T3 : symmetric
                for (int e = threadIdx.x; e < d * d; e += blockDim.x) {
                    const int i = e / d, j = e % d;
                    if (j > i) continue;
                    float s = sC[i * ld + j];
                    for (int q = 0; q < d; ++q) s = __fmaf_rn(sT[q * ld + i], sT3[q * ld + j], s);
                    sS[i * ld + j] = s;
                    sS[j * ld + i] = s;
                }
                __syncthreads();
                // mu_s = mu_f + G (mu_s+ - A mu_f - u)
                g_mulv(v_t, sA, v_mu, v_u, d, d, ld);
                for (int i = threadIdx.x; i < d; i += blockDim.x) v_e[i] = v_ms[i] - v_t[i];
                __syncthreads();
                g_mulv_t(v_t, sT, v_e, v_mu, d, d, ld);               // (G')' v = G v
                for (int i = threadIdx.x; i < d; i += blockDim.x) {
                    v_ms[i] = v_t[i];
                    g.mean[((int64_t)t * d + i) * g.batch + b] = v_t[i];
                }
                for (int e = threadIdx.x; e < d * d; e += blockDim.x) {
                    const float v = sS[(e / d) * ld + e % d];
                    sX[(e / d) * ld + e % d] = v;
                    g.cov[((int64_t)t * d * d + e) * g.batch + b] = v;
                }
                __syncthreads();
            }
        }
        if (g.status && threadIdx.x == 0) {
            bool nan = false;
            for (int i = 0; i < d; ++i) nan |= !(v_ms[i] == v_ms[i]) && g.smooth;
            for (int i = 0; i < d; ++i) nan |= !(v_mu[i] == v_mu[i]);
            g.status[b] = (s_scal[1] != 0.f) ? RXG_ERR_NOT_SPD : (nan ? RXG_ERR_NAN : RXG_OK);
        }
        __syncthreads();
    }
}

}  // namespace

// Shared models arrive as host arrays: they are staged into the ctx workspace first.
int lgssm_generic_chain(rxg_ctx* ctx, const LgssmCall& c) {
    const int d = c.d, m = c.m;
    if (d < 1 || m < 1 || d > 64 || m > 64)
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm: d, m must be in 1..64 (got d=%d, m=%d)", d, m);
    if (!c.cov) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: post_cov is required on the per-chain path (it is the stash)");
    GenArgs g = {};
    g.d = d; g.m = m; g.T = c.T; g.batch = c.batch;
    g.per_chain = (c.flags & RXG_MODEL_PER_CHAIN) ? 1 : 0;
    if (g.per_chain) {
        g.A = c.A; g.B = c.B; g.P = c.P; g.Q = c.Q; g.m0 = c.m0; g.S0 = c.S0; g.u = c.u;
    } else {
        const size_t nA = (size_t)d * d, nB = (size_t)m * d, nQ = (size_t)m * m;
        const size_t tot = 3 * nA + nB + nQ + 2 * (size_t)d;
        float* dev = (float*)workspace(ctx, tot * 4);
        if (!dev) return RXG_ERR_CUDA;
        float *dA = dev, *dB = dA + nA, *dP = dB + nB, *dQ = dP + nA, *dS0 = dQ + nQ, *dm0 = dS0 + nA, *du = dm0 + d;
        RXG_CUDA(ctx, cudaMemcpyAsync(dA, c.A, nA * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(dB, c.B, nB * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(dP, c.P, nA * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(dQ, c.Q, nQ * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(dS0, c.S0, nA * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(dm0, c.m0, (size_t)d * 4, cudaMemcpyHostToDevice, ctx->stream));
        if (c.u) RXG_CUDA(ctx, cudaMemcpyAsync(du, c.u, (size_t)d * 4, cudaMemcpyHostToDevice, ctx->stream));
        g.A = dA; g.B = dB; g.P = dP; g.Q = dQ; g.S0 = dS0; g.m0 = dm0; g.u = c.u ? du : nullptr;
    }
    g.mean0_chain = c.mean0_chain;
    g.useq = c.useq; g.ustride = c.useq_chain ? c.batch : 1; g.uchain = c.useq_chain ? 1 : 0;
    g.y = c.y; g.mask = c.ymask; g.mean = c.mean; g.cov = c.cov; g.nle = c.nle; g.status = c.status;
    g.smooth = c.smooth ? 1 : 0;
    g.transition_first = (c.flags & RXG_TRANSITION_FIRST) ? 1 : 0;
    const int n = d > m ? d : m;
    const size_t smem = ((size_t)8 * n * (n + 1) + 5 * (size_t)n + 4) * 4;
    RXG_CUDA(ctx, cudaFuncSetAttribute(lgssm_generic_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = (int)(220 * 1024 / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 4) per_sm = 4;
    int64_t grid = (int64_t)ctx->sm_count * per_sm;
    if (grid > c.batch) grid = c.batch;
    if (ctx->profile) { cudaEventRecord(ctx->ev[0], ctx->stream); cudaEventRecord(ctx->ev[1], ctx->stream); }
    lgssm_generic_chain_kernel<<<(unsigned)grid, 256, smem, ctx->stream>>>(g);
    if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "lgssm_generic_chain_kernel");
}

}  // namespace rxg
