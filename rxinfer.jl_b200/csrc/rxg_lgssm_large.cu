// Large-state family of the shared-model LGSSM sweeps (d = m in {8, 16, 32, 64}; BASELINE
// configs[2] is d = 64, T = 1000, batch = 4096).  Same decomposition as the small-state path
// (rxg_lgssm_shared.cuh): with shared (A, B, P, Q, S0) every covariance-valued message of the
// reference schedule [ref: /root/reference/benchmarks/...Benchmark.ipynb:95-105;
// src/inference/batch.jl:391-430] is chain independent, so
//   1. the gain tables come from block-cooperative fp64 kernels working on d x d matrices in
//      shared memory (large_riccati_seq: sequential in t; large_gain_tables: one CTA per t;
//      large_smooth_seq: sequential in t), and
//   2. every chain runs only the mean recursions.  Across a tile of NB chains those are small
//      GEMMs per step,  X <- [F_t | K_t] [X ; Y_t]  and  X <- [E_t | G_t] [mu_f,t ; X],
//      executed by lgssm_block_sweep with the per-step gain block streamed through shared memory
//      (cp.async, double buffered) and a 4 x 2 register tile per thread.
// For d >= 16 the mean recursions run on the tensor cores (rxg_umma_sweep.cu: wgmma tf32, 3xTF32 split,
// register accumulators, TMA bulk copies of the gain records); lgssm_block_sweep is the d = 8 path and the
// RXG_OPT_NO_UMMA cross-check.  The family also produces neg_log_evidence (large_evidence_kernel).
#include <math.h>

#include <stdlib.h>

#include "rxg_internal.h"
#include "rxg_umma.cuh"

namespace rxg {

// ------------------------------------------------------------------------------------------------
// block-cooperative fp64 linear algebra on shared-memory matrices (row-major, leading dim LD)
// ------------------------------------------------------------------------------------------------
// C(i,j) = beta * Add(i,j) + sum_k a(i,k) b(k,j); accessors are functors so that transposes are free.
template <int R, int C, int K, class FA, class FB, class FC>
__device__ __forceinline__ void bgemm(FA a, FB b, FC store) {
    constexpr int TR = 4, TC = 4;
    constexpr int NTR = (R + TR - 1) / TR, NTC = (C + TC - 1) / TC;
    for (int tile = threadIdx.x; tile < NTR * NTC; tile += blockDim.x) {
        const int i0 = (tile / NTC) * TR, j0 = (tile % NTC) * TC;
        double acc[TR][TC];
#pragma unroll
        for (int r = 0; r < TR; ++r)
#pragma unroll
            for (int c = 0; c < TC; ++c) acc[r][c] = 0.0;
        for (int k = 0; k < K; ++k) {
            double av[TR], bv[TC];
#pragma unroll
            for (int r = 0; r < TR; ++r) av[r] = (i0 + r < R) ? a(i0 + r, k) : 0.0;
#pragma unroll
            for (int c = 0; c < TC; ++c) bv[c] = (j0 + c < C) ? b(k, j0 + c) : 0.0;
#pragma unroll
            for (int r = 0; r < TR; ++r)
#pragma unroll
                for (int c = 0; c < TC; ++c) acc[r][c] = fma(av[r], bv[c], acc[r][c]);
        }
#pragma unroll
        for (int r = 0; r < TR; ++r)
#pragma unroll
            for (int c = 0; c < TC; ++c)
                if (i0 + r < R && j0 + c < C) store(i0 + r, j0 + c, acc[r][c]);
    }
}

// in-place lower Cholesky (left-looking), blockDim.x == 256: P = 256 / N threads share the dot
// product of one row and reduce with shuffles; two barriers per column.  Only the lower triangle
// is written / meaningful afterwards.
template <int N, int LD>
__device__ void bchol(double* A, int* flag) {
    constexpr int P = (256 / N) > 32 ? 32 : (256 / N);
    const int row = threadIdx.x / P, part = threadIdx.x % P;
    __syncthreads();
    for (int j = 0; j < N; ++j) {
        double s = 0.0;
        if (row < N && row >= j)
            for (int k = part; k < j; k += P) s = fma(A[row * LD + k], A[j * LD + k], s);
#pragma unroll
        for (int o = P / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (row == j && part == 0) {
            double d = A[j * LD + j] - s;
            if (!(d > 0.0)) { *flag = 1; d = 1e-300; }
            A[j * LD + j] = sqrt(d);
        }
        __syncthreads();
        if (row > j && row < N && part == 0) A[row * LD + j] = (A[row * LD + j] - s) / A[j * LD + j];
        __syncthreads();
    }
}
// X <- L^-1 X  (X is N x C): P = 256 / C threads per column split each dot product
template <int N, int C, int LD>
__device__ void btrsm_lower(const double* L, double* X) {
    constexpr int P = (256 / C) > 32 ? 32 : (256 / C);
    const int col = threadIdx.x / P, part = threadIdx.x % P;
    if (col < C) {
        for (int i = 0; i < N; ++i) {
            double s = 0.0;
            for (int k = part; k < i; k += P) s = fma(L[i * LD + k], X[k * LD + col], s);
#pragma unroll
            for (int o = P / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (part == 0) X[i * LD + col] = (X[i * LD + col] - s) / L[i * LD + i];
            __syncwarp();
        }
    }
    __syncthreads();
}
// X <- L^-T X
template <int N, int C, int LD>
__device__ void btrsm_lower_t(const double* L, double* X) {
    constexpr int P = (256 / C) > 32 ? 32 : (256 / C);
    const int col = threadIdx.x / P, part = threadIdx.x % P;
    if (col < C) {
        for (int i = N - 1; i >= 0; --i) {
            double s = 0.0;
            for (int k = i + 1 + part; k < N; k += P) s = fma(L[k * LD + i], X[k * LD + col], s);
#pragma unroll
            for (int o = P / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (part == 0) X[i * LD + col] = (X[i * LD + col] - s) / L[i * LD + i];
            __syncwarp();
        }
    }
    __syncthreads();
}

struct LargeWs {
    const double *A, *B, *P, *Q, *S0, *BA;   // fp64 copies of the model (global)
    double *Sp, *Sf, *Cc, *Gd;               // [T][D*D]
    float *fwdT;                             // [T][(D+M)][D]   [F_t | K_t] transposed (k-major)
    float *bwdT;                             // [T][2D][D]      [E_t | G_t] transposed
    float *ss, *sf;                          // [T][D*D] smoothed / filtered covariance (fp32)
    int* flag;
    int b_identity;                          // B == I: skip the two B products
    // tensor-core sweep (rxg_umma_sweep.cu): per-step gain blocks split tf32 hi | lo in the canonical
    // K-major layout (K = D), or null:  recFE[t] = [F_t ; E_{t-1}] (2D x D),  recG[t] = G_t,  recK[t] = K_t (D x D)
    float *recFE, *recG, *recK;
    // evidence (optional): evT[t][(D+M)][M] = [-(L_t^-1 B A) | L_t^-1]' (k-major, like fwdT) with S_t = L_t L_t',
    // evc[t] = M/2 log 2pi + sum_i log L_t(i,i); null when the caller did not ask for neg_log_evidence
    float* evT;
    double* evc;
};

template <int D> struct LD_ { static constexpr int v = D + 1; };   // padded leading dim: no bank conflicts on transposed reads

// Phase 1: Riccati recursion, sequential in t, one CTA.
template <int D, int M>
__global__ void __launch_bounds__(256) large_riccati_seq(LargeWs w, int T, int transition_first) {
    constexpr int LD = LD_<D>::v;
    extern __shared__ double sm[];
    double* S = sm;                 // D x D   current covariance
    double* T1 = S + D * LD;        // scratch
    double* T2 = T1 + D * LD;       // scratch (innovation covariance / its Cholesky factor)
    double* As = T2 + D * LD;       // A staged in shared memory
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
        S[(i / D) * LD + i % D] = w.S0[i];
        As[(i / D) * LD + i % D] = w.A[i];
    }
    __syncthreads();
    for (int t = 0; t < T; ++t) {
        if (t > 0 || transition_first) {
            bgemm<D, D, D>([&](int i, int k) { return As[i * LD + k]; }, [&](int k, int j) { return S[k * LD + j]; },
                           [&](int i, int j, double v) { T1[i * LD + j] = v; });
            __syncthreads();
            bgemm<D, D, D>([&](int i, int k) { return T1[i * LD + k]; }, [&](int k, int j) { return As[j * LD + k]; },
                           [&](int i, int j, double v) { S[i * LD + j] = v + w.P[i * D + j]; });
            __syncthreads();
        }
        for (int i = threadIdx.x; i < D * D; i += blockDim.x) w.Sp[(size_t)t * D * D + i] = S[(i / D) * LD + i % D];
        if (w.b_identity && M == D) {
            for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
                const int i = idx / D, j = idx % D;
                const double v = S[i * LD + j];
                T1[i * LD + j] = v;
                T2[i * LD + j] = v + w.Q[i * M + j];
            }
        } else {
            // T1 = B S (M x D); T2 = T1 B' + Q (M x M)
            bgemm<M, D, D>([&](int i, int k) { return w.B[i * D + k]; }, [&](int k, int j) { return S[k * LD + j]; },
                           [&](int i, int j, double v) { T1[i * LD + j] = v; });
            __syncthreads();
            bgemm<M, M, D>([&](int i, int k) { return T1[i * LD + k]; }, [&](int k, int j) { return w.B[j * D + k]; },
                           [&](int i, int j, double v) { T2[i * LD + j] = v + w.Q[i * M + j]; });
        }
        bchol<M, LD>(T2, w.flag);
        btrsm_lower<M, D, LD>(T2, T1);                 // W = L^-1 B S   (M x D)
        // S <- S - W' W
        bgemm<D, D, M>([&](int i, int k) { return T1[k * LD + i]; }, [&](int k, int j) { return T1[k * LD + j]; },
                       [&](int i, int j, double v) { S[i * LD + j] -= v; });
        __syncthreads();
        // symmetrise (round-off) and publish
        for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
            const int i = idx / D, j = idx % D;
            if (j < i) { const double s = 0.5 * (S[i * LD + j] + S[j * LD + i]); T2[i * LD + j] = s; }
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
            const int i = idx / D, j = idx % D;
            if (j < i) { S[i * LD + j] = T2[i * LD + j]; S[j * LD + i] = T2[i * LD + j]; }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < D * D; i += blockDim.x) w.Sf[(size_t)t * D * D + i] = S[(i / D) * LD + i % D];
    }
}

// Phase 2: one CTA per time step: Kalman gain, F = (I - K B) A, RTS gain, E = I - G A, conditional cov.
template <int D, int M>
__global__ void __launch_bounds__(256) large_gain_tables(LargeWs w, int T, int transition_first) {
    constexpr int LD = LD_<D>::v;
    extern __shared__ double sm[];
    // three D x D fp64 buffers (100 KB at d = 64: two CTAs per SM).  A is read from global memory in the forward part
    // (one element-wise use) and staged into X1 -- free by then -- for the products of the backward part.
    double* X0 = sm;
    double* X1 = X0 + D * LD;
    double* X2 = X1 + D * LD;
    const int t = blockIdx.x;
    const double* Sp = w.Sp + (size_t)t * D * D;
    const double* Sf = w.Sf + (size_t)t * D * D;
    // ---- forward gain: X1 = B Sp; X2 = X1 B' + Q = L L'; X1 <- L^-T L^-1 X1 = K'  (M x D)
    if (w.b_identity && M == D) {
        for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
            const int i = idx / D, j = idx % D;
            const double v = Sp[idx];
            X1[i * LD + j] = v;
            X2[i * LD + j] = v + w.Q[i * M + j];
        }
    } else {
        bgemm<M, D, D>([&](int i, int k) { return w.B[i * D + k]; }, [&](int k, int j) { return Sp[k * D + j]; },
                       [&](int i, int j, double v) { X1[i * LD + j] = v; });
        __syncthreads();
        bgemm<M, M, D>([&](int i, int k) { return X1[i * LD + k]; }, [&](int k, int j) { return w.B[j * D + k]; },
                       [&](int i, int j, double v) { X2[i * LD + j] = v + w.Q[i * M + j]; });
    }
    bchol<M, LD>(X2, w.flag);
    btrsm_lower<M, D, LD>(X2, X1);
    btrsm_lower_t<M, D, LD>(X2, X1);                   // X1 = K' (M x D): K(r, k) = X1[k][r]
    float* ft = w.fwdT + (size_t)t * (D + M) * D;
    const bool pred = (t > 0) || transition_first;
    // tensor-core sweep: emit a D x D block W(r, k) = srcT[k][r] into rows [row0, row0 + D) of a record whose hi part
    // starts at rec_hi and lo part at rec_lo (canonical K-major layout with K = D, rxg_umma.cuh)
    auto emit_umma = [&](float* rec_hi, float* rec_lo, const float* srcT, int row0) {
        for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
            const int k = idx / D, r = idx % D;
            float hi, lo;
            umma::split_tf32(srcT[k * D + r], hi, lo);
            const uint32_t off = umma::elem_off(row0 + r, k, D) / 4;
            rec_hi[off] = hi;
            rec_lo[off] = lo;
        }
    };
    constexpr size_t FE_REC = (size_t)4 * D * D, G_REC = (size_t)2 * D * D;
    // F = A - K (B A)   (or I - K B at t = 0 without a leading transition); stored transposed: ft[k][r] = F(r, k)
    if (pred) {
        bgemm<D, D, M>([&](int r, int k) { return X1[k * LD + r]; }, [&](int k, int j) { return w.BA[k * D + j]; },
                       [&](int r, int j, double v) { ft[j * D + r] = (float)(w.A[r * D + j] - v); });
    } else {
        bgemm<D, D, M>([&](int r, int k) { return X1[k * LD + r]; }, [&](int k, int j) { return w.B[k * D + j]; },
                       [&](int r, int j, double v) { ft[j * D + r] = (float)((r == j ? 1.0 : 0.0) - v); });
    }
    for (int idx = threadIdx.x; idx < M * D; idx += blockDim.x) {
        const int k = idx / D, r = idx % D;
        ft[(D + k) * D + r] = (float)X1[k * LD + r];
    }
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) w.sf[(size_t)t * D * D + i] = (float)Sf[i];
    __syncthreads();
    if (M == D && w.recFE) {
        float* fe = w.recFE + (size_t)t * FE_REC;
        emit_umma(fe, fe + 2 * D * D, ft, 0);                                   // F_t -> rows [0, D) of record t
        float* kr = w.recK + (size_t)t * G_REC;
        emit_umma(kr, kr + D * D, ft + D * D, 0);                               // K_t
        if (t == 0)                                                              // record 0 has no E_{-1}: zero rows [D, 2D)
            for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
                const uint32_t off = umma::elem_off(D + idx % D, idx / D, D) / 4;
                fe[off] = 0.f; fe[2 * D * D + off] = 0.f;
            }
    }
    // ---- evidence tables: the whitened innovation is  w_t = L^-1 (y_t - B A x_{t-1}) = [-(L^-1 B A) | L^-1] [x_{t-1} ; y_t]
    if (w.evT) {
        float* et = w.evT + (size_t)t * (D + M) * M;
        for (int idx = threadIdx.x; idx < M * D; idx += blockDim.x) {
            const int r = idx / D, k = idx % D;
            X0[r * LD + k] = pred ? w.BA[r * D + k] : w.B[r * D + k];
        }
        __syncthreads();
        btrsm_lower<M, D, LD>(X2, X0);
        for (int idx = threadIdx.x; idx < M * D; idx += blockDim.x) {
            const int k = idx / M, r = idx % M;
            et[k * M + r] = (float)(-X0[r * LD + k]);
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < M * M; idx += blockDim.x) X0[(idx / M) * LD + idx % M] = (idx / M == idx % M) ? 1.0 : 0.0;
        __syncthreads();
        btrsm_lower<M, M, LD>(X2, X0);
        for (int idx = threadIdx.x; idx < M * M; idx += blockDim.x) {
            const int k = idx / M, r = idx % M;
            et[(D + k) * M + r] = (float)X0[r * LD + k];
        }
        if (threadIdx.x == 0) {
            double sl = M * 0.91893853320467274178;   // M/2 log 2 pi
            for (int i = 0; i < M; ++i) sl += log(X2[i * LD + i]);
            w.evc[t] = sl;
        }
        __syncthreads();
    }
    // ---- backward gain
    float* bt = w.bwdT + (size_t)t * 2 * D * D;
    if (t == T - 1) {
        for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
            const int k = idx / D, r = idx % D;
            bt[k * D + r] = (k == r) ? 1.f : 0.f;
            bt[(D + k) * D + r] = 0.f;
            w.Gd[(size_t)t * D * D + idx] = 0.0;                 // suffix-scan element of the last step: (0, Sf)
            w.Cc[(size_t)t * D * D + idx] = Sf[idx];
        }
        return;                  // E_{T-1} = I, G_{T-1} = 0: the tensor-core sweep sets mu_s[T-1] = x_{T-1} directly
    }
    const double* Sp1 = w.Sp + (size_t)(t + 1) * D * D;
    double* As = X1;                       // K' (X1) is no longer needed: every reader finished before the barrier above
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
        As[(i / D) * LD + i % D] = w.A[i];
        X2[(i / D) * LD + i % D] = Sp1[i];
    }
    __syncthreads();
    // X0 = A Sf  (= (Sf A')')
    bgemm<D, D, D>([&](int i, int k) { return As[i * LD + k]; }, [&](int k, int j) { return Sf[k * D + j]; },
                   [&](int i, int j, double v) { X0[i * LD + j] = v; });
    bchol<D, LD>(X2, w.flag);
    btrsm_lower<D, D, LD>(X2, X0);                     // X0 = U' = Lp^-1 A Sf
    // C = Sf - U U' = Sf - X0' X0
    bgemm<D, D, D>([&](int i, int k) { return X0[k * LD + i]; }, [&](int k, int j) { return X0[k * LD + j]; },
                   [&](int i, int j, double v) { w.Cc[(size_t)t * D * D + i * D + j] = Sf[i * D + j] - v; });
    __syncthreads();
    btrsm_lower_t<D, D, LD>(X2, X0);                   // X0 = G' = Lp^-T U'   : G(r, k) = X0[k][r]
    for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
        const int k = idx / D, r = idx % D;
        const double g = X0[k * LD + r];
        bt[(D + k) * D + r] = (float)g;
        w.Gd[(size_t)t * D * D + r * D + k] = g;
    }
    // E = I - G A: E(r, j) = delta - sum_k G(r,k) A(k,j); stored transposed bt[j][r]
    bgemm<D, D, D>([&](int r, int k) { return X0[k * LD + r]; }, [&](int k, int j) { return As[k * LD + j]; },
                   [&](int r, int j, double v) { bt[j * D + r] = (float)((r == j ? 1.0 : 0.0) - v); });
    __syncthreads();
    if (M == D && w.recFE) {
        float* fe = w.recFE + (size_t)(t + 1) * FE_REC;                          // t + 1 <= T - 1 here
        emit_umma(fe, fe + 2 * D * D, bt, D);                                    // E_t -> rows [D, 2D) of record t + 1
        float* gr = w.recG + (size_t)t * G_REC;
        emit_umma(gr, gr + D * D, bt + D * D, 0);                                // G_t
    }
}

// Phase 3: smoothed covariances, sequential in t, one CTA:  Ss[t] = C[t] + G[t] Ss[t+1] G[t]'.
template <int D>
__global__ void __launch_bounds__(256) large_smooth_seq(LargeWs w, int T) {
    constexpr int LD = LD_<D>::v;
    extern __shared__ double sm[];
    double* S = sm;
    double* T1 = S + D * LD;
    double* Gs = T1 + D * LD;
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
        const double v = w.Sf[(size_t)(T - 1) * D * D + i];
        S[(i / D) * LD + i % D] = v;
        w.ss[(size_t)(T - 1) * D * D + i] = (float)v;
    }
    __syncthreads();
    for (int t = T - 2; t >= 0; --t) {
        const double* G = w.Gd + (size_t)t * D * D;
        const double* C = w.Cc + (size_t)t * D * D;
        for (int i = threadIdx.x; i < D * D; i += blockDim.x) Gs[(i / D) * LD + i % D] = G[i];
        __syncthreads();
        bgemm<D, D, D>([&](int i, int k) { return Gs[i * LD + k]; }, [&](int k, int j) { return S[k * LD + j]; },
                       [&](int i, int j, double v) { T1[i * LD + j] = v; });
        __syncthreads();
        bgemm<D, D, D>([&](int i, int k) { return T1[i * LD + k]; }, [&](int k, int j) { return Gs[j * LD + k]; },
                       [&](int i, int j, double v) { S[i * LD + j] = v + C[i * D + j]; });
        __syncthreads();
        for (int i = threadIdx.x; i < D * D; i += blockDim.x) w.ss[(size_t)t * D * D + i] = (float)S[(i / D) * LD + i % D];
    }
}

// ------------------------------------------------------------------------------------------------
// Time-parallel replacement of the two sequential phases (RXG_LARGE_SEQ=1 keeps the sequential ones).
//
// Forward, by DOUBLING: the model is time invariant, so the covariance parts (A, C, J) of the
// filtering scan element (Sarkka & Garcia-Fernandez 2021) are the same "gen" for every step >= 1.
// With G_r = gen (x) ... (x) gen (2^r factors) the filtered covariances satisfy
//     Sigma_f[k] = C( P[k - 2^r] (x) G_r ),   2^r <= k < 2^(r+1),      G_(r+1) = G_r (x) G_r,
// i.e. round r applies 2^r Riccati steps at once to 2^r already-known covariances, one CTA each:
// ceil(log2 T) launches instead of T dependent steps.  Prefixes have A = 0, J = 0, so only
//     C_new = A_G (I + C_i J_G)^-1 C_i A_G' + C_G
// is needed; with C_i = L L' and I + L' J_G L = R R' this is Z' Z + C_G, Z = R^-1 L' A_G'
// (two Cholesky factorisations, one triangular solve, four products; symmetric PSD by construction).
// ------------------------------------------------------------------------------------------------
struct ScanG { double *A, *C, *J; };

template <int D, int LD>
__device__ __forceinline__ void load_mat(double* dst, const double* src) {
    for (int i = threadIdx.x; i < D * D; i += blockDim.x) dst[(i / D) * LD + i % D] = src[i];
}

// first element (C_0 -> Sf[0]) and the generic element gen -> G0
template <int D, int M>
__global__ void __launch_bounds__(256) large_fwd_init(LargeWs w, ScanG g0, int transition_first) {
    constexpr int LD = LD_<D>::v;
    extern __shared__ double sm[];
    double* X0 = sm; double* X1 = X0 + D * LD; double* X2 = X1 + D * LD; double* X3 = X2 + D * LD;
    if (blockIdx.x == 0) {
        // S' = S0 (or A S0 A' + P); C_0 = S' - W' W, W = L^-1 B S', L L' = B S' B' + Q
        load_mat<D, LD>(X0, w.S0);
        __syncthreads();
        if (transition_first) {
            bgemm<D, D, D>([&](int i, int k) { return w.A[i * D + k]; }, [&](int k, int j) { return X0[k * LD + j]; },
                           [&](int i, int j, double v) { X1[i * LD + j] = v; });
            __syncthreads();
            bgemm<D, D, D>([&](int i, int k) { return X1[i * LD + k]; }, [&](int k, int j) { return w.A[j * D + k]; },
                           [&](int i, int j, double v) { X0[i * LD + j] = v + w.P[i * D + j]; });
            __syncthreads();
        }
        bgemm<M, D, D>([&](int i, int k) { return w.B[i * D + k]; }, [&](int k, int j) { return X0[k * LD + j]; },
                       [&](int i, int j, double v) { X1[i * LD + j] = v; });
        __syncthreads();
        bgemm<M, M, D>([&](int i, int k) { return X1[i * LD + k]; }, [&](int k, int j) { return w.B[j * D + k]; },
                       [&](int i, int j, double v) { X2[i * LD + j] = v + w.Q[i * M + j]; });
        bchol<M, LD>(X2, w.flag);
        btrsm_lower<M, D, LD>(X2, X1);
        bgemm<D, D, M>([&](int i, int k) { return X1[k * LD + i]; }, [&](int k, int j) { return X1[k * LD + j]; },
                       [&](int i, int j, double v) { w.Sf[i * D + j] = X0[i * LD + j] - v; });
    } else {
        // gen: L L' = B P B' + Q; W1 = L^-1 B P, W2 = L^-1 B, W3 = L^-1 B A
        //      A_gen = (I - W1' W2) A,  C_gen = P - W1' W1,  J_gen = W3' W3
        bgemm<M, D, D>([&](int i, int k) { return w.B[i * D + k]; }, [&](int k, int j) { return w.P[k * D + j]; },
                       [&](int i, int j, double v) { X0[i * LD + j] = v; });              // B P
        __syncthreads();
        bgemm<M, M, D>([&](int i, int k) { return X0[i * LD + k]; }, [&](int k, int j) { return w.B[j * D + k]; },
                       [&](int i, int j, double v) { X3[i * LD + j] = v + w.Q[i * M + j]; });
        for (int i = threadIdx.x; i < M * D; i += blockDim.x) {
            X1[(i / D) * LD + i % D] = w.B[i];
            X2[(i / D) * LD + i % D] = w.BA[i];
        }
        bchol<M, LD>(X3, w.flag);
        btrsm_lower<M, D, LD>(X3, X0);     // W1
        btrsm_lower<M, D, LD>(X3, X1);     // W2
        btrsm_lower<M, D, LD>(X3, X2);     // W3
        bgemm<D, D, M>([&](int i, int k) { return X0[k * LD + i]; }, [&](int k, int j) { return X0[k * LD + j]; },
                       [&](int i, int j, double v) { g0.C[i * D + j] = w.P[i * D + j] - v; });
        bgemm<D, D, M>([&](int i, int k) { return X2[k * LD + i]; }, [&](int k, int j) { return X2[k * LD + j]; },
                       [&](int i, int j, double v) { g0.J[i * D + j] = v; });
        // X3 <- I - W1' W2 (the Cholesky factor is no longer needed)
        __syncthreads();
        bgemm<D, D, M>([&](int i, int k) { return X0[k * LD + i]; }, [&](int k, int j) { return X1[k * LD + j]; },
                       [&](int i, int j, double v) { X3[i * LD + j] = (i == j ? 1.0 : 0.0) - v; });
        __syncthreads();
        bgemm<D, D, D>([&](int i, int k) { return X3[i * LD + k]; }, [&](int k, int j) { return w.A[k * D + j]; },
                       [&](int i, int j, double v) { g0.A[i * D + j] = v; });
    }
}

// shared core of a combine: given C_i (in X0) and J_j (staged in X2), leaves
//   X0 = L (lower Cholesky factor of C_i),  X1 = Y = R^-1 L'  with R R' = I + L' J_j L
template <int D, int LD>
__device__ __forceinline__ void combine_core(double* X0, double* X1, double* X2, int* flag) {
    bchol<D, LD>(X0, flag);
    auto Lf = [&](int i, int k) { return k <= i ? X0[i * LD + k] : 0.0; };
    bgemm<D, D, D>([&](int i, int k) { return X2[i * LD + k]; }, [&](int k, int j) { return Lf(k, j); },
                   [&](int i, int j, double v) { X1[i * LD + j] = v; });                 // J L
    __syncthreads();
    bgemm<D, D, D>([&](int i, int k) { return Lf(k, i); }, [&](int k, int j) { return X1[k * LD + j]; },
                   [&](int i, int j, double v) { X2[i * LD + j] = v + (i == j ? 1.0 : 0.0); });   // I + L' J L
    bchol<D, LD>(X2, flag);
    for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
        const int i = idx / D, j = idx % D;
        X1[i * LD + j] = Lf(j, i);                                                       // L'
    }
    __syncthreads();
    btrsm_lower<D, D, LD>(X2, X1);                                                       // Y = R^-1 L'
}

// round r: CTAs 0 .. n-1 advance prefixes by 2^r steps; the last CTA squares G
template <int D>
__global__ void __launch_bounds__(256) large_fwd_doubling(LargeWs w, ScanG gc, ScanG gn, int r, int T) {
    constexpr int LD = LD_<D>::v;
    extern __shared__ double sm[];
    double* X0 = sm; double* X1 = X0 + D * LD; double* X2 = X1 + D * LD; double* X3 = X2 + D * LD;
    const int step = 1 << r;
    const int n = min(step, T - step);           // prefixes produced this round: k = step .. step + n - 1
    if ((int)blockIdx.x < n) {
        const int k = step + blockIdx.x, i = k - step;
        load_mat<D, LD>(X0, w.Sf + (size_t)i * D * D);
        load_mat<D, LD>(X2, gc.J);
        load_mat<D, LD>(X3, gc.A);
        combine_core<D, LD>(X0, X1, X2, w.flag);
        // Z = Y A_G' ; Sf[k] = Z' Z + C_G
        bgemm<D, D, D>([&](int a, int kk) { return X1[a * LD + kk]; }, [&](int kk, int b) { return X3[b * LD + kk]; },
                       [&](int a, int b, double v) { X0[a * LD + b] = v; });
        __syncthreads();
        bgemm<D, D, D>([&](int a, int kk) { return X0[kk * LD + a]; }, [&](int kk, int b) { return X0[kk * LD + b]; },
                       [&](int a, int b, double v) { w.Sf[(size_t)k * D * D + a * D + b] = v + gc.C[a * D + b]; });
    } else {
        // G_next = G (x) G (full combine):  X2m = Y' Y = (I + C J)^-1 C;  X1m = A - X2m (J A);
        //   A_n = A X1m;  C_n = A X2m A' + C = Z' Z + C (Z = Y A');  J_n = sym(A' J X1m) + J
        double* X4 = X3 + D * LD; double* X5 = X4 + D * LD;
        load_mat<D, LD>(X0, gc.C);
        load_mat<D, LD>(X2, gc.J);
        load_mat<D, LD>(X3, gc.A);
        combine_core<D, LD>(X0, X1, X2, w.flag);                                          // X1 = Y
        bgemm<D, D, D>([&](int a, int kk) { return X1[kk * LD + a]; }, [&](int kk, int b) { return X1[kk * LD + b]; },
                       [&](int a, int b, double v) { X4[a * LD + b] = v; });              // X4 = X2m
        bgemm<D, D, D>([&](int a, int kk) { return gc.J[a * D + kk]; }, [&](int kk, int b) { return X3[kk * LD + b]; },
                       [&](int a, int b, double v) { X5[a * LD + b] = v; });              // X5 = J A
        __syncthreads();
        bgemm<D, D, D>([&](int a, int kk) { return X4[a * LD + kk]; }, [&](int kk, int b) { return X5[kk * LD + b]; },
                       [&](int a, int b, double v) { X0[a * LD + b] = X3[a * LD + b] - v; });   // X0 = X1m
        bgemm<D, D, D>([&](int a, int kk) { return X1[a * LD + kk]; }, [&](int kk, int b) { return X3[b * LD + kk]; },
                       [&](int a, int b, double v) { X2[a * LD + b] = v; });              // X2 = Z = Y A'
        __syncthreads();
        bgemm<D, D, D>([&](int a, int kk) { return X3[a * LD + kk]; }, [&](int kk, int b) { return X0[kk * LD + b]; },
                       [&](int a, int b, double v) { gn.A[a * D + b] = v; });
        bgemm<D, D, D>([&](int a, int kk) { return X2[kk * LD + a]; }, [&](int kk, int b) { return X2[kk * LD + b]; },
                       [&](int a, int b, double v) { gn.C[a * D + b] = v + gc.C[a * D + b]; });
        bgemm<D, D, D>([&](int a, int kk) { return gc.J[a * D + kk]; }, [&](int kk, int b) { return X0[kk * LD + b]; },
                       [&](int a, int b, double v) { X5[a * LD + b] = v; });              // X5 = J X1m
        __syncthreads();
        bgemm<D, D, D>([&](int a, int kk) { return X3[kk * LD + a]; }, [&](int kk, int b) { return X5[kk * LD + b]; },
                       [&](int a, int b, double v) { X4[a * LD + b] = v; });              // A' J X1m
        __syncthreads();
        for (int idx = threadIdx.x; idx < D * D; idx += blockDim.x) {
            const int a = idx / D, b = idx % D;
            gn.J[idx] = 0.5 * (X4[a * LD + b] + X4[b * LD + a]) + gc.J[idx];
        }
    }
}

// predicted covariances from the filtered ones (parallel over t): Sp[t] = A Sf[t-1] A' + P
template <int D>
__global__ void __launch_bounds__(256) large_predict(LargeWs w, int T, int transition_first) {
    constexpr int LD = LD_<D>::v;
    extern __shared__ double sm[];
    double* X0 = sm; double* X1 = X0 + D * LD;
    const int t = blockIdx.x;
    double* out = w.Sp + (size_t)t * D * D;
    if (t == 0 && !transition_first) {
        for (int i = threadIdx.x; i < D * D; i += blockDim.x) out[i] = w.S0[i];
        return;
    }
    load_mat<D, LD>(X0, t == 0 ? w.S0 : w.Sf + (size_t)(t - 1) * D * D);
    __syncthreads();
    bgemm<D, D, D>([&](int i, int k) { return w.A[i * D + k]; }, [&](int k, int j) { return X0[k * LD + j]; },
                   [&](int i, int j, double v) { X1[i * LD + j] = v; });
    __syncthreads();
    bgemm<D, D, D>([&](int i, int k) { return X1[i * LD + k]; }, [&](int k, int j) { return w.A[j * D + k]; },
                   [&](int i, int j, double v) { out[i * D + j] = v + w.P[i * D + j]; });
}

// backward Hillis-Steele round over the suffix elements (E, L): new[t] = old[t] (x) old[t + off]
template <int D>
__global__ void __launch_bounds__(256)
large_bwd_scan_round(const double* __restrict__ Es, const double* __restrict__ Ls, double* __restrict__ Ed,
                     double* __restrict__ Ld, float* __restrict__ ss_out, int off, int T) {
    constexpr int LD = LD_<D>::v;
    extern __shared__ double sm[];
    double* X0 = sm; double* X1 = X0 + D * LD; double* X2 = X1 + D * LD;
    const int t = blockIdx.x;
    const size_t o = (size_t)t * D * D;
    if (t + off >= T) {
        for (int i = threadIdx.x; i < D * D; i += blockDim.x) {
            const double l = Ls[o + i];
            Ed[o + i] = Es[o + i]; Ld[o + i] = l;
            if (ss_out) ss_out[o + i] = (float)l;
        }
        return;
    }
    const size_t o2 = (size_t)(t + off) * D * D;
    load_mat<D, LD>(X0, Es + o);
    load_mat<D, LD>(X1, Ls + o2);
    __syncthreads();
    bgemm<D, D, D>([&](int i, int k) { return X0[i * LD + k]; }, [&](int k, int j) { return X1[k * LD + j]; },
                   [&](int i, int j, double v) { X2[i * LD + j] = v; });                   // E_t L_late
    __syncthreads();
    bgemm<D, D, D>([&](int i, int k) { return X2[i * LD + k]; }, [&](int k, int j) { return X0[j * LD + k]; },
                   [&](int i, int j, double v) {
                       const double l = v + Ls[o + i * D + j];
                       Ld[o + i * D + j] = l;
                       if (ss_out) ss_out[o + i * D + j] = (float)l;
                   });
    bgemm<D, D, D>([&](int i, int k) { return X0[i * LD + k]; }, [&](int k, int j) { return Es[o2 + k * D + j]; },
                   [&](int i, int j, double v) { Ed[o + i * D + j] = v; });
}

// ------------------------------------------------------------------------------------------------
// mean sweep: a tile of NB chains per CTA, per-step GEMM  out[D x NB] = W_t'[(K2) x D]' * Z[(K2) x NB]
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cpa16(void* s, const void* g) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g));
}
__device__ __forceinline__ void cpa4(void* s, const void* g) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g));
}
__device__ __forceinline__ void cpa_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cpa_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// one step of the tile GEMM: thread (rg, cg) owns rows 4 rg .. 4 rg + 3 and columns 2 cg, 2 cg + 1
template <int D, int K2, int NB>
__device__ __forceinline__ void tile_step(const float* __restrict__ W, const float* __restrict__ Z, int rg, int cg,
                                          float (&acc)[4][2]) {
#pragma unroll
    for (int r = 0; r < 4; ++r) { acc[r][0] = 0.f; acc[r][1] = 0.f; }
#pragma unroll 8
    for (int k = 0; k < K2; ++k) {
        const float4 wv = *reinterpret_cast<const float4*>(W + k * D + 4 * rg);
        const float2 zv = *reinterpret_cast<const float2*>(Z + k * NB + 2 * cg);
        acc[0][0] = __fmaf_rn(wv.x, zv.x, acc[0][0]); acc[0][1] = __fmaf_rn(wv.x, zv.y, acc[0][1]);
        acc[1][0] = __fmaf_rn(wv.y, zv.x, acc[1][0]); acc[1][1] = __fmaf_rn(wv.y, zv.y, acc[1][1]);
        acc[2][0] = __fmaf_rn(wv.z, zv.x, acc[2][0]); acc[2][1] = __fmaf_rn(wv.z, zv.y, acc[2][1]);
        acc[3][0] = __fmaf_rn(wv.w, zv.x, acc[3][0]); acc[3][1] = __fmaf_rn(wv.w, zv.y, acc[3][1]);
    }
}

template <int D, int M, int NB, bool SMOOTH>
__global__ void __launch_bounds__((D / 4) * (NB / 2))
lgssm_block_sweep(const float* __restrict__ fwdT, const float* __restrict__ bwdT, const float* __restrict__ m0,
                  const float* __restrict__ m0c, const float* __restrict__ y, float* __restrict__ mean, int T,
                  int64_t batch) {
    constexpr int KF = D + M, KB = 2 * D, KMAX = KF > KB ? KF : KB;
    constexpr int NT = (D / 4) * (NB / 2);
    extern __shared__ __align__(16) float smf[];
    float* Wb[2] = {smf, smf + KMAX * D};
    float* Zb[2] = {smf + 2 * KMAX * D, smf + 2 * KMAX * D + KMAX * NB};
    const int tid = threadIdx.x;
    const int cg = tid % (NB / 2), rg = tid / (NB / 2);
    const int64_t b0 = (int64_t)blockIdx.x * NB;
    const int nb = (int)((batch - b0) < NB ? (batch - b0) : NB);

    auto load_W = [&](float* dst, const float* src, int K2) {
        for (int p = tid; p < K2 * D / 4; p += NT) cpa16(dst + 4 * p, src + 4 * p);
    };
    auto load_rows = [&](float* dst, const float* src_row0, int rows) {   // rows x NB from a [rows][batch] slab
        for (int p = tid; p < rows * NB; p += NT) {
            const int r = p / NB, c = p % NB;
            if (c < nb) cpa4(dst + r * NB + c, src_row0 + (size_t)r * batch + b0 + c);
        }
    };
    // zero both Z buffers once (inactive columns stay zero), then the initial state
    for (int p = tid; p < 2 * KMAX * NB; p += NT) Zb[0][p] = 0.f;
    __syncthreads();
    for (int p = tid; p < D * NB; p += NT)     // prior mean: shared, or per chain (streaming carry) for the active columns
        Zb[0][p] = m0c ? ((p % NB) < nb ? m0c[(size_t)(p / NB) * batch + b0 + (p % NB)] : 0.f) : m0[p / NB];
    load_W(Wb[0], fwdT, KF);
    load_rows(Zb[0] + D * NB, y, M);
    cpa_commit();

    float acc[4][2];
    // ---------------------------------------------------------------- forward
    for (int t = 0; t < T; ++t) {
        const int q = t & 1;
        if (t + 1 < T) {
            load_W(Wb[q ^ 1], fwdT + (size_t)(t + 1) * KF * D, KF);
            load_rows(Zb[q ^ 1] + D * NB, y + (size_t)(t + 1) * M * batch, M);
        }
        cpa_commit();
        cpa_wait<1>();
        __syncthreads();
        tile_step<D, KF, NB>(Wb[q], Zb[q], rg, cg, acc);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int row = 4 * rg + r;
            *reinterpret_cast<float2*>(Zb[q ^ 1] + row * NB + 2 * cg) = make_float2(acc[r][0], acc[r][1]);
            float* g = mean + ((size_t)t * D + row) * batch + b0 + 2 * cg;
            if (2 * cg < nb) g[0] = acc[r][0];          // scalar stores: the caller's mean need not be 8-byte aligned
            if (2 * cg + 1 < nb) g[1] = acc[r][1];
        }
        __syncthreads();
    }
    cpa_wait<0>();
    if (!SMOOTH) return;
    // ---------------------------------------------------------------- backward: Z = [mu_f[t] ; mu_s[t+1]]
    __syncthreads();
    for (int p = tid; p < D * NB; p += NT) { Zb[0][D * NB + p] = 0.f; }
    load_W(Wb[0], bwdT + (size_t)(T - 1) * KB * D, KB);
    load_rows(Zb[0], mean + (size_t)(T - 1) * D * batch, D);
    cpa_commit();
    for (int r = 0; r < T; ++r) {
        const int t = T - 1 - r, q = r & 1;
        if (t - 1 >= 0) {
            load_W(Wb[q ^ 1], bwdT + (size_t)(t - 1) * KB * D, KB);
            load_rows(Zb[q ^ 1], mean + (size_t)(t - 1) * D * batch, D);
        }
        cpa_commit();
        cpa_wait<1>();
        __syncthreads();
        tile_step<D, KB, NB>(Wb[q], Zb[q], rg, cg, acc);
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
            const int row = 4 * rg + rr;
            *reinterpret_cast<float2*>(Zb[q ^ 1] + (D + row) * NB + 2 * cg) = make_float2(acc[rr][0], acc[rr][1]);
            float* g = mean + ((size_t)t * D + row) * batch + b0 + 2 * cg;
            if (2 * cg < nb) g[0] = acc[rr][0];
            if (2 * cg + 1 < nb) g[1] = acc[rr][1];
        }
        __syncthreads();
    }
    cpa_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// neg_log_evidence of the large-state family: parallel over (chain tile, time slice).  Per step the tile GEMM
// w_t = [-(L^-1 B A) | L^-1] [mu_f[t-1] ; y_t] (the whitened innovation, tables from large_gain_tables) and
// q += |w_t|^2; partial[slice][chain] = sum over the slice, reduced deterministically by evidence_finish_kernel:
// nle = sum_t (M/2 log 2pi + log det L_t) + 1/2 sum_t |w_t|^2   (innovation form; = Bethe free energy on this tree,
// /root/reference/src/model/plugins/reactivemp_free_energy.jl:84-126).  mean[] must hold the FILTERED means.
template <int D, int M, int NB>
__global__ void __launch_bounds__((D / 4) * (NB / 2))
large_evidence_kernel(const float* __restrict__ evT, const float* __restrict__ m0, const float* __restrict__ m0c,
                      const float* __restrict__ y, const float* __restrict__ mean, double* __restrict__ partial, int T,
                      int64_t batch) {
    constexpr int K2 = D + M;
    constexpr int NT = (D / 4) * (NB / 2);
    extern __shared__ __align__(16) float smf[];
    float* Wb[2] = {smf, smf + K2 * M};
    float* Zb[2] = {smf + 2 * K2 * M, smf + 2 * K2 * M + K2 * NB};
    double* red = reinterpret_cast<double*>(smf + 2 * K2 * M + 2 * K2 * NB);     // [D/4][NB]
    const int tid = threadIdx.x;
    const int cg = tid % (NB / 2), rg = tid / (NB / 2);
    const int64_t b0 = (int64_t)blockIdx.x * NB;
    const int nb = (int)((batch - b0) < NB ? (batch - b0) : NB);
    const int t_lo = (int)(((int64_t)T * blockIdx.y) / gridDim.y), t_hi = (int)(((int64_t)T * (blockIdx.y + 1)) / gridDim.y);
    auto load_W = [&](float* dst, const float* src) {
        for (int p = tid; p < K2 * M / 4; p += NT) cpa16(dst + 4 * p, src + 4 * p);
    };
    auto load_rows = [&](float* dst, const float* src_row0, int rows) {
        for (int p = tid; p < rows * NB; p += NT) {
            const int r = p / NB, c = p % NB;
            if (c < nb) cpa4(dst + r * NB + c, src_row0 + (size_t)r * batch + b0 + c);
        }
    };
    auto load_Z = [&](float* dst, int t) {        // [mu_f[t-1] ; y_t]; the prior mean stands in for mu_f[-1]
        if (t > 0) load_rows(dst, mean + (size_t)(t - 1) * D * batch, D);
        else
            for (int p = tid; p < D * NB; p += NT)
                dst[p] = m0c ? ((p % NB) < nb ? m0c[(size_t)(p / NB) * batch + b0 + (p % NB)] : 0.f) : m0[p / NB];
        load_rows(dst + D * NB, y + (size_t)t * M * batch, M);
    };
    for (int p = tid; p < 2 * K2 * NB; p += NT) Zb[0][p] = 0.f;       // inactive columns stay zero
    __syncthreads();
    float q[2] = {0.f, 0.f};
    double qd[2] = {0.0, 0.0};
    if (t_lo < t_hi) {
        load_W(Wb[0], evT + (size_t)t_lo * K2 * M);
        load_Z(Zb[0], t_lo);
    }
    cpa_commit();
    float acc[4][2];
    for (int t = t_lo; t < t_hi; ++t) {
        const int qb = (t - t_lo) & 1;
        if (t + 1 < t_hi) {
            load_W(Wb[qb ^ 1], evT + (size_t)(t + 1) * K2 * M);
            load_Z(Zb[qb ^ 1], t + 1);
        }
        cpa_commit();
        cpa_wait<1>();
        __syncthreads();
        tile_step<M, K2, NB>(Wb[qb], Zb[qb], rg, cg, acc);
#pragma unroll
        for (int r = 0; r < 4; ++r) { q[0] = __fmaf_rn(acc[r][0], acc[r][0], q[0]); q[1] = __fmaf_rn(acc[r][1], acc[r][1], q[1]); }
        if (((t - t_lo) & 31) == 31) { qd[0] += (double)q[0]; qd[1] += (double)q[1]; q[0] = q[1] = 0.f; }
        __syncthreads();
    }
    cpa_wait<0>();
    red[rg * NB + 2 * cg] = qd[0] + (double)q[0];
    red[rg * NB + 2 * cg + 1] = qd[1] + (double)q[1];
    __syncthreads();
    if (tid < nb) {
        double s = 0.0;
        for (int r = 0; r < D / 4; ++r) s += red[r * NB + tid];
        partial[(size_t)blockIdx.y * batch + b0 + tid] = s;
    }
}
__global__ void evidence_finish_kernel(const double* __restrict__ partial, const double* __restrict__ evc, int nslices, int T,
                                       int64_t batch, float* __restrict__ nle) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= batch) return;
    double c = 0.0;
    for (int t = 0; t < T; ++t) c += evc[t];
    double s = 0.0;
    for (int i = 0; i < nslices; ++i) s += partial[(size_t)i * batch + b];
    nle[b] = (float)(c + 0.5 * s);
}

// cov[t][i][j][b] = tab[t][i*D + j] for every chain b (the contract's per-chain covariance output)
__global__ void broadcast_cov_kernel(const float* __restrict__ tab, float* __restrict__ cov, int64_t rows, int64_t batch) {
    const int64_t row = blockIdx.x;
    if (row >= rows) return;
    const float v = __ldg(tab + row);
    float* dst = cov + row * batch;
    for (int64_t b = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; b < batch; b += (int64_t)gridDim.y * blockDim.x) dst[b] = v;
}

__global__ void to_double_kernel(const float* __restrict__ src, double* __restrict__ dst, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = (double)src[i];
}
template <int D, int M>
__global__ void ba_kernel(const double* B, const double* A, double* BA) {
    for (int idx = threadIdx.x; idx < M * D; idx += blockDim.x) {
        const int i = idx / D, j = idx % D;
        double s = 0.0;
        for (int k = 0; k < D; ++k) s = fma(B[i * D + k], A[k * D + j], s);
        BA[idx] = s;
    }
}

template <int D, int M>
static int run_large(rxg_ctx* ctx, LgssmCall& c) {
    if ((c.flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN)) || c.ymask || c.u)
        return fail(ctx, RXG_ERR_UNSUPPORTED,
                    "lgssm (d=%d): the large-state family covers shared models without mask / offset", D);
    const size_t T = (size_t)c.T, DD = (size_t)D * D;
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
    const size_t o_model32 = carve((3 * DD + (size_t)M * D + (size_t)M * M + D) * 4);
    const size_t o_A = carve(DD * 8), o_B = carve((size_t)M * D * 8), o_P = carve(DD * 8), o_Q = carve((size_t)M * M * 8);
    const size_t o_S0 = carve(DD * 8), o_BA = carve((size_t)M * D * 8);
    const size_t o_Sp = carve(T * DD * 8), o_Sf = carve(T * DD * 8), o_Cc = carve(T * DD * 8), o_Gd = carve(T * DD * 8);
    const size_t o_fw = carve(T * (D + M) * D * 4), o_bw = carve(T * 2 * DD * 4), o_ss = carve(T * DD * 4), o_sf = carve(T * DD * 4);
    // d >= 16: the mean recursions run on the tensor cores (RXG_NO_UMMA=1: FP32-pipe block sweep, the cross-check)
    const bool use_umma = (D >= 16 && M == D) && (ctx->opt[RXG_OPT_NO_UMMA] == 0);
    const size_t o_fe = carve(use_umma ? T * 4 * DD * 4 : 0), o_gu = carve(use_umma ? T * 2 * DD * 4 : 0);
    const size_t o_ku = carve(use_umma ? T * 2 * DD * 4 : 0);
    constexpr int EV_NB = 32;
    const unsigned ev_tiles = (unsigned)((c.batch + EV_NB - 1) / EV_NB);
    int ev_slices = (int)((4 * (unsigned)ctx->sm_count + ev_tiles - 1) / ev_tiles);      // ~4 CTAs per SM in flight
    if (ev_slices < 1) ev_slices = 1;
    if (ev_slices > c.T) ev_slices = c.T;
    const size_t o_evT = carve(c.nle ? T * (D + M) * M * 4 : 0), o_evc = carve(c.nle ? T * 8 : 0);
    const size_t o_evp = carve(c.nle ? (size_t)ev_slices * c.batch * 8 : 0);
    const size_t o_scan = carve(6 * DD * 8);                                  // G_r ping-pong (A, C, J) x 2
    const size_t o_E2 = carve(T * DD * 8), o_L2 = carve(T * DD * 8);           // backward scan ping-pong
    const size_t o_flag = carve(4);
    char* base = (char*)workspace(ctx, off);
    if (!base) return RXG_ERR_CUDA;
    // model: host fp32 -> device fp32 -> device fp64
    float* m32 = (float*)(base + o_model32);
    float* dA = m32, *dB = dA + DD, *dP = dB + (size_t)M * D, *dQ = dP + DD, *dS0 = dQ + (size_t)M * M, *dm0 = dS0 + DD;
    RXG_CUDA(ctx, cudaMemcpyAsync(dA, c.A, DD * 4, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaMemcpyAsync(dB, c.B, (size_t)M * D * 4, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaMemcpyAsync(dP, c.P, DD * 4, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaMemcpyAsync(dQ, c.Q, (size_t)M * M * 4, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaMemcpyAsync(dS0, c.S0, DD * 4, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaMemcpyAsync(dm0, c.m0, (size_t)D * 4, cudaMemcpyHostToDevice, ctx->stream));
    LargeWs w;
    double *A64 = (double*)(base + o_A), *B64 = (double*)(base + o_B), *P64 = (double*)(base + o_P);
    double *Q64 = (double*)(base + o_Q), *S064 = (double*)(base + o_S0), *BA64 = (double*)(base + o_BA);
    auto cvt = [&](const float* s, double* d, int n) { to_double_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(s, d, n); };
    cvt(dA, A64, (int)DD); cvt(dB, B64, M * D); cvt(dP, P64, (int)DD); cvt(dQ, Q64, M * M); cvt(dS0, S064, (int)DD);
    ba_kernel<D, M><<<1, 256, 0, ctx->stream>>>(B64, A64, BA64);
    ctx->launches += 6;
    w.A = A64; w.B = B64; w.P = P64; w.Q = Q64; w.S0 = S064; w.BA = BA64;
    w.Sp = (double*)(base + o_Sp); w.Sf = (double*)(base + o_Sf); w.Cc = (double*)(base + o_Cc); w.Gd = (double*)(base + o_Gd);
    w.fwdT = (float*)(base + o_fw); w.bwdT = (float*)(base + o_bw); w.ss = (float*)(base + o_ss); w.sf = (float*)(base + o_sf);
    w.flag = bad_flag(ctx);      // shared with the status / return-code plumbing (rxg_api.cu)
    (void)o_flag;
    w.recFE = use_umma ? (float*)(base + o_fe) : nullptr;
    w.recG = use_umma ? (float*)(base + o_gu) : nullptr;
    w.recK = use_umma ? (float*)(base + o_ku) : nullptr;
    w.evT = c.nle ? (float*)(base + o_evT) : nullptr;
    w.evc = c.nle ? (double*)(base + o_evc) : nullptr;
    w.b_identity = (M == D) ? 1 : 0;
    for (int i = 0; i < M * D && w.b_identity; ++i) w.b_identity = (c.B[i] == ((i / D == i % D) ? 1.f : 0.f));
    const int tf = (c.flags & RXG_TRANSITION_FIRST) ? 1 : 0;
    constexpr int LD = LD_<D>::v;
    const size_t sm3 = (size_t)4 * D * LD * 8, sm2 = (size_t)3 * D * LD * 8;
    {   // per-DEVICE attributes: set on every call (a few microseconds), never cached per process
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_riccati_seq<D, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm3));
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_gain_tables<D, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_smooth_seq<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
    }
    const size_t sm4 = (size_t)4 * D * LD * 8, sm6 = (size_t)6 * D * LD * 8;
    {
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_fwd_init<D, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm4));
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_fwd_doubling<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm6));
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_predict<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_bwd_scan_round<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm2));
    }
    const bool seq = ctx->opt[RXG_OPT_LARGE_SEQ] != 0;
    if (ctx->profile) cudaEventRecord(ctx->ev[0], ctx->stream);
    if (seq) {
        large_riccati_seq<D, M><<<1, 256, sm3, ctx->stream>>>(w, c.T, tf);
        ctx->launches += 1;
    } else {
        // forward by doubling: ceil(log2 T) rounds, round r advances 2^r prefixes by 2^r steps
        double* gb = (double*)(base + o_scan);
        ScanG g[2] = {{gb, gb + DD, gb + 2 * DD}, {gb + 3 * DD, gb + 4 * DD, gb + 5 * DD}};
        large_fwd_init<D, M><<<2, 256, sm4, ctx->stream>>>(w, g[0], tf);
        ctx->launches += 1;
        int cur = 0;
        for (int r = 0; (1 << r) < c.T; ++r) {
            const int step = 1 << r;
            const int n = step < c.T - step ? step : c.T - step;
            large_fwd_doubling<D><<<n + 1, 256, sm6, ctx->stream>>>(w, g[cur], g[cur ^ 1], r, c.T);
            ctx->launches += 1;
            cur ^= 1;
        }
        large_predict<D><<<c.T, 256, sm2, ctx->stream>>>(w, c.T, tf);
        ctx->launches += 1;
    }
    large_gain_tables<D, M><<<c.T, 256, sm2, ctx->stream>>>(w, c.T, tf);
    ctx->launches += 1;
    if (c.smooth) {
        if (seq) {
            large_smooth_seq<D><<<1, 256, sm2, ctx->stream>>>(w, c.T);
            ctx->launches += 1;
        } else {
            // backward suffix scan over (E, L) = (G_t, C_t): ceil(log2 T) Hillis-Steele rounds, one CTA per step
            double* Eb[2] = {w.Gd, (double*)(base + o_E2)};
            double* Lb[2] = {w.Cc, (double*)(base + o_L2)};
            int cur = 0, nr = 0;
            for (int off = 1; off < c.T; off <<= 1) ++nr;
            if (nr == 0) {      // T == 1
                large_bwd_scan_round<D><<<c.T, 256, sm2, ctx->stream>>>(Eb[0], Lb[0], Eb[1], Lb[1], w.ss, c.T, c.T);
                ctx->launches += 1;
            }
            for (int off = 1, i = 0; off < c.T; off <<= 1, ++i) {
                large_bwd_scan_round<D><<<c.T, 256, sm2, ctx->stream>>>(Eb[cur], Lb[cur], Eb[cur ^ 1], Lb[cur ^ 1],
                                                                        (i == nr - 1) ? w.ss : nullptr, off, c.T);
                ctx->launches += 1;
                cur ^= 1;
            }
        }
    }
    int rc = check_cuda(ctx, cudaGetLastError(), "large gain kernels");
    if (rc != RXG_OK) return rc;
    if (c.tables_only) {
        if (c.cov && (c.flags & RXG_COV_SHARED_OUT))
            RXG_CUDA(ctx, cudaMemcpyAsync(c.cov, c.smooth ? w.ss : w.sf, T * DD * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        return RXG_OK;
    }

    constexpr int NB = 32;
    constexpr int KMAX = (D + M) > 2 * D ? (D + M) : 2 * D;
    const size_t smw = (size_t)(2 * KMAX * D + 2 * KMAX * NB) * 4;
    {
        RXG_CUDA(ctx, cudaFuncSetAttribute(lgssm_block_sweep<D, M, NB, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smw));
        RXG_CUDA(ctx, cudaFuncSetAttribute(lgssm_block_sweep<D, M, NB, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smw));
    }
    const unsigned blocks = (unsigned)((c.batch + NB - 1) / NB);
    auto sweep = [&](bool smooth) -> int {
        if (use_umma)   // tensor-pipe sweep (wgmma tf32, 3xTF32): 64 chains per CTA; u_t = K_t y_t pre-pass + recursion
            return launch_umma_sweep(ctx, D, smooth, w.recFE, w.recG, w.recK, dm0, c.mean0_chain, c.y, c.mean, c.T, c.batch);
        if (smooth) lgssm_block_sweep<D, M, NB, true><<<blocks, (D / 4) * (NB / 2), smw, ctx->stream>>>(w.fwdT, w.bwdT, dm0, c.mean0_chain, c.y, c.mean, c.T, c.batch);
        else        lgssm_block_sweep<D, M, NB, false><<<blocks, (D / 4) * (NB / 2), smw, ctx->stream>>>(w.fwdT, w.bwdT, dm0, c.mean0_chain, c.y, c.mean, c.T, c.batch);
        ctx->launches += 1;
        return check_cuda(ctx, cudaGetLastError(), "lgssm_block_sweep");
    };
    if (ctx->profile) cudaEventRecord(ctx->ev[1], ctx->stream);
    if (c.nle) {
        // the evidence is a function of the FILTERED means: filter-mode sweep, then the (time-parallel) evidence
        // kernels; a smoothing call re-runs the sweep in smoothing mode afterwards (the fused smoothing recursion
        // does not keep the filtered means)
        rc = sweep(false);
        if (rc != RXG_OK) return rc;
        const size_t sme = (size_t)(2 * (D + M) * M + 2 * (D + M) * EV_NB) * 4 + (size_t)(D / 4) * EV_NB * 8;
        RXG_CUDA(ctx, cudaFuncSetAttribute(large_evidence_kernel<D, M, EV_NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sme));
        large_evidence_kernel<D, M, EV_NB><<<dim3(ev_tiles, (unsigned)ev_slices), (D / 4) * (EV_NB / 2), sme, ctx->stream>>>(
            w.evT, dm0, c.mean0_chain, c.y, c.mean, (double*)(base + o_evp), c.T, c.batch);
        evidence_finish_kernel<<<(unsigned)((c.batch + 255) / 256), 256, 0, ctx->stream>>>(
            (const double*)(base + o_evp), w.evc, ev_slices, c.T, c.batch, c.nle);
        ctx->launches += 2;
        rc = check_cuda(ctx, cudaGetLastError(), "large_evidence_kernel");
        if (rc != RXG_OK) return rc;
    }
    if (c.smooth || !c.nle) {
        rc = sweep(c.smooth);
        if (rc != RXG_OK) return rc;
    }
    if (ctx->profile) cudaEventRecord(ctx->ev[2], ctx->stream);
    // Per-chain covariance output (the contract): T d^2 rows broadcast over the batch -- 67 GB at configs[2], pure HBM
    // writes.  It runs after the mean sweeps, not beside them: the broadcast streams through L2 and would evict the
    // per-step gain records that all chain tiles of the latency-bound tensor-core sweep share.
    if (c.cov) {
        const float* tab = c.smooth ? w.ss : w.sf;
        if (c.flags & RXG_COV_SHARED_OUT) {
            RXG_CUDA(ctx, cudaMemcpyAsync(c.cov, tab, T * DD * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        } else {
            const int64_t rows = (int64_t)(T * DD);
            dim3 grid((unsigned)rows, (unsigned)((c.batch + 4095) / 4096 > 16 ? 16 : (c.batch + 4095) / 4096));
            broadcast_cov_kernel<<<grid, 256, 0, ctx->stream>>>(tab, c.cov, rows, c.batch);
            ctx->launches += 1;
            rc = check_cuda(ctx, cudaGetLastError(), "broadcast_cov_kernel");
            if (rc != RXG_OK) return rc;
        }
    }
    if (c.status) return fill_status_from_flag(ctx, c.status, c.batch);
    return RXG_OK;
}

bool lgssm_large_supported(int d, int m) { return d == m && (d == 8 || d == 16 || d == 32 || d == 64); }

int lgssm_large_dispatch(rxg_ctx* ctx, LgssmCall& c) {
    switch (c.d) {
        case 8: return run_large<8, 8>(ctx, c);
        case 16: return run_large<16, 16>(ctx, c);
        case 32: return run_large<32, 32>(ctx, c);
        case 64: return run_large<64, 64>(ctx, c);
        default: return fail(ctx, RXG_ERR_UNSUPPORTED, "large-state family: d=%d unsupported", c.d);
    }
}

}  // namespace rxg
