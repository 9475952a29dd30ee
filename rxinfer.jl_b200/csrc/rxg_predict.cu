// Predictive distributions of the observations after a smoothing sweep (rxg_lgssm_smooth_predict_f32): the reference's
// message toward every y[t] and the forecasts of the next H observations [ref: result.predictions,
// src/inference/batch.jl:203-246; test/inference/prediction_tests.jl:193-420].
//
// The message toward y[t] is the cavity fwd_t x bwd_t (every message into x[t] except the one from y[t]) pushed through
// *(:out) with B and MvNormalMeanCovariance(:out) with Q.  With the smoothed posterior (mu_s, S_s) it has a closed form:
//     missing y[t]:   N(B mu_s, B S_s B' + Q)                        (the cavity is the posterior)
//     observed y[t]:  D_t = Q - B S_s B'  (SPD whenever the cavity is proper, also for m < d),
//                     N(y - Q D_t^-1 (y - B mu_s), Q D_t^-1 Q)
// and the forecasts step (x, S) <- (A x + u, A S A' + P) from (mu_s[T-1], S_s[T-1]).  D_t is a difference of nearly equal
// matrices when the observations dominate (Q << B S_prior B'): it is formed and factorised in fp64.
//
// The work is a post-pass on the smoother's final outputs, the same for every kernel family.  Two routes:
//   A  covariances chain independent (shared model, no per-chain mask, no RXG_PATH_PER_CHAIN):
//        k_predict_msg (one warp per step, fp64) turns the S_s table into per-step tables of the affine map
//            y_hat = F_t y + G_t mu,   F_t = I - K_t, G_t = K_t B, K_t = Q D_t^-1      (missing / forecast: F_t = 0, G_t = B)
//        and the prediction covariances; the means are then one streaming pass over (y, mu) -- register-resident for the
//        native small shapes (k_predict_mean_small, tables staged through shared memory), the per-slice left-GEMM of
//        rxg_rules_large.cu otherwise.  Per-chain covariance outputs are broadcast from the tables.
//   B  per-chain models / masks: k_predict_msg with one warp per (step, chain), matrices in shared memory (row stride + 1).
#include <math.h>

#include "rxg_internal.h"

namespace rxg {

namespace {

constexpr int PW_MAX_WARPS = 8;      // warps (= messages) per CTA of k_predict_msg
constexpr int PM_TC = 16;            // time steps per CTA of k_predict_mean_small
constexpr int FM_THREADS = 64;       // chains per CTA of k_forecast_mean

// per-warp shared-memory layout of k_predict_msg: fp64 work matrices first, fp32 operands after them
struct MsgLayout {
    int r1, dd, v;           // offsets in doubles: R1 = max(m x (d+1), m x (m+1)), Dd = m x (m+1), v = 2m
    int nd;                  // doubles in all
    int sg, bf, qf;          // offsets in floats (after the doubles): S_s d x (d+1), B m x (d+1), Q m x (m+1)
    int bytes;               // per warp, 16-byte multiple
};
__host__ __device__ inline MsgLayout msg_layout(int d, int m) {
    MsgLayout L;
    const int r1n = m * (d + 1) > m * (m + 1) ? m * (d + 1) : m * (m + 1);
    L.r1 = 0; L.dd = r1n; L.v = L.dd + m * (m + 1); L.nd = L.v + 2 * m;
    L.sg = 0; L.bf = d * (d + 1); L.qf = L.bf + m * (d + 1);
    const int nf = L.qf + m * (m + 1);
    L.bytes = (L.nd * 8 + nf * 4 + 15) / 16 * 16;
    return L;
}

struct MsgArgs {
    int d, m, T, H;
    int64_t batch;
    int per_chain;                       // 0: one item per step (route A tables), 1: one item per (step, chain)
    const float *B, *Q;                  // element e of chain b at [e * ms + b * mb]
    int64_t ms, mb;
    const float* sig;                    // S_s[t] of chain b: element e at sig[(t d^2 + e) * sig_s + b * sig_b]
    int64_t sig_s;
    const float* fsig;                   // forecast S_k (rows t >= T): element e at fsig[((t - T) d^2 + e) * fsig_s + b * sig_b]
    int64_t fsig_s, sig_b;
    const uint8_t* tmask;                // [T] or null
    const uint8_t* ymask;                // [T][batch] or null
    // route A
    float *F, *G, *C;                    // [T+H][m][m], [T+H][m][d], [T+H][m][m]
    int* bad;
    // route B
    const float *y, *mean, *fmean;       // [T][m][batch], [T][d][batch], [H][d][batch]
    float *pmean, *pcov;                 // [T+H][m][batch], [T+H][m][m][batch] or null
    int32_t* status;
};

__global__ void __launch_bounds__(32 * PW_MAX_WARPS) k_predict_msg(MsgArgs a) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int d = a.d, m = a.m, ldd = d + 1, ldm = m + 1;
    const MsgLayout L = msg_layout(d, m);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t nb = a.per_chain ? a.batch : 1;
    const int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (item >= (int64_t)(a.T + a.H) * nb) return;                    // whole warps only: no CTA-wide barrier below
    const int64_t b = item % nb;
    const int t = (int)(item / nb);
    unsigned char* base = smraw + (size_t)warp * L.bytes;
    double* R1 = reinterpret_cast<double*>(base) + L.r1;
    double* Dd = reinterpret_cast<double*>(base) + L.dd;
    double* v = reinterpret_cast<double*>(base) + L.v;
    float* fb = reinterpret_cast<float*>(base + (size_t)L.nd * 8);
    float *Sg = fb + L.sg, *Bf = fb + L.bf, *Qf = fb + L.qf;

    const bool fc = t >= a.T;
    const float* sp = fc ? a.fsig + (int64_t)(t - a.T) * d * d * a.fsig_s : a.sig + (int64_t)t * d * d * a.sig_s;
    const int64_t ss = fc ? a.fsig_s : a.sig_s, so = b * a.sig_b, mo = b * a.mb;
    for (int e = lane; e < d * d; e += 32) Sg[(e / d) * ldd + e % d] = __ldg(sp + (int64_t)e * ss + so);
    for (int e = lane; e < m * d; e += 32) Bf[(e / d) * ldd + e % d] = __ldg(a.B + (int64_t)e * a.ms + mo);
    for (int e = lane; e < m * m; e += 32) Qf[(e / m) * ldm + e % m] = __ldg(a.Q + (int64_t)e * a.ms + mo);
    __syncwarp();
    bool obs = !fc;
    if (obs && a.tmask) obs = a.tmask[t] != 0;
    if (obs && a.ymask) obs = a.ymask[(int64_t)t * a.batch + b] != 0;

    // W = B S_s (m x d) in R1, lane per column
    for (int j = lane; j < d; j += 32)
        for (int k = 0; k < m; ++k) {
            double s = 0.0;
            for (int i = 0; i < d; ++i) s = fma((double)Bf[k * ldd + i], (double)Sg[i * ldd + j], s);
            R1[k * ldd + j] = s;
        }
    __syncwarp();
    // B S_s B' (lower triangle, mirrored), then D = Q - B S_s B' (observed) or the prediction covariance B S_s B' + Q
    for (int l = lane; l < m; l += 32)
        for (int k = l; k < m; ++k) {
            double s = 0.0;
            for (int j = 0; j < d; ++j) s = fma(R1[k * ldd + j], (double)Bf[l * ldd + j], s);
            const double q = 0.5 * ((double)Qf[k * ldm + l] + (double)Qf[l * ldm + k]);
            Dd[k * ldm + l] = Dd[l * ldm + k] = obs ? q - s : q + s;
        }
    __syncwarp();

    bool bad = false;
    if (obs) {
        // Cholesky D = L L' (left-looking, lane per row), reciprocal pivots in v[0..m)
        const int r0 = lane, r1 = lane + 32;
        for (int j = 0; j < m; ++j) {
            double t0 = 0.0, t1 = 0.0;
            if (r0 < m && r0 >= j) {
                t0 = Dd[r0 * ldm + j];
                for (int c = 0; c < j; ++c) t0 = fma(-Dd[r0 * ldm + c], Dd[j * ldm + c], t0);
            }
            if (r1 < m && r1 >= j) {
                t1 = Dd[r1 * ldm + j];
                for (int c = 0; c < j; ++c) t1 = fma(-Dd[r1 * ldm + c], Dd[j * ldm + c], t1);
            }
            if ((j & 31) == lane) {
                double p = (j < 32) ? t0 : t1;
                if (!(p > 0.0)) { bad = true; p = 1e-30; }
                const double sq = sqrt(p);
                Dd[j * ldm + j] = sq;
                v[j] = 1.0 / sq;
            }
            __syncwarp();
            const double rj = v[j];
            if (r0 < m && r0 > j) Dd[r0 * ldm + j] = t0 * rj;
            if (r1 < m && r1 > j) Dd[r1 * ldm + j] = t1 * rj;
            __syncwarp();
        }
        // X = D^-1 Q (R1, row stride m + 1), lane per column: L z = Q[:, c], then L' x = z.  K = Q D^-1 = X'.
        for (int c = lane; c < m; c += 32) {
            for (int r = 0; r < m; ++r) {
                double s = (double)Qf[r * ldm + c];
                for (int p = 0; p < r; ++p) s = fma(-Dd[r * ldm + p], R1[p * ldm + c], s);
                R1[r * ldm + c] = s * v[r];
            }
            for (int r = m - 1; r >= 0; --r) {
                double s = R1[r * ldm + c];
                for (int p = r + 1; p < m; ++p) s = fma(-Dd[p * ldm + r], R1[p * ldm + c], s);
                R1[r * ldm + c] = s * v[r];
            }
        }
        __syncwarp();
        // prediction covariance Q D^-1 Q = Q X (lower triangle, mirrored) over the factor
        for (int l = lane; l < m; l += 32)
            for (int k = l; k < m; ++k) {
                double s = 0.0;
                for (int j = 0; j < m; ++j) s = fma((double)Qf[k * ldm + j], R1[j * ldm + l], s);
                Dd[k * ldm + l] = s;
            }
        __syncwarp();
        for (int l = lane; l < m; l += 32)
            for (int k = l + 1; k < m; ++k) Dd[l * ldm + k] = Dd[k * ldm + l];
        __syncwarp();
    }
    bad = __any_sync(0xffffffffu, bad);

    if (!a.per_chain) {
        // ---- route A: per-step tables
        const int64_t tt = t;
        for (int e = lane; e < m * m; e += 32) {
            const int k = e / m, l = e % m;
            a.F[tt * m * m + e] = obs ? (float)((k == l ? 1.0 : 0.0) - R1[l * ldm + k]) : 0.f;
            a.C[tt * m * m + e] = (float)Dd[k * ldm + l];
        }
        for (int e = lane; e < m * d; e += 32) {
            const int k = e / d, j = e % d;
            double s = 0.0;
            if (obs)
                for (int l = 0; l < m; ++l) s = fma(R1[l * ldm + k], (double)Bf[l * ldd + j], s);
            a.G[tt * m * d + e] = obs ? (float)s : Bf[k * ldd + j];
        }
        if (bad && lane == 0) atomicOr(a.bad, 1);
        return;
    }
    // ---- route B: this chain's mean and covariance.  mu (fp32) goes over the S_s copy, which is no longer read.
    const float* mu = fc ? a.fmean + (int64_t)(t - a.T) * d * a.batch : a.mean + (int64_t)t * d * a.batch;
    for (int i = lane; i < d; i += 32) Sg[i] = __ldg(mu + (int64_t)i * a.batch + b);
    __syncwarp();
    double* r = v + m;
    for (int k = lane; k < m; k += 32) {
        double s = 0.0;
        for (int j = 0; j < d; ++j) s = fma((double)Bf[k * ldd + j], (double)Sg[j], s);
        r[k] = obs ? (double)__ldg(a.y + ((int64_t)t * m + k) * a.batch + b) - s : s;        // innovation, or B mu
    }
    __syncwarp();
    for (int k = lane; k < m; k += 32) {
        double o = r[k];
        if (obs) {
            o = (double)__ldg(a.y + ((int64_t)t * m + k) * a.batch + b);
            for (int l = 0; l < m; ++l) o = fma(-R1[l * ldm + k], r[l], o);
        }
        a.pmean[((int64_t)t * m + k) * a.batch + b] = (float)o;
    }
    if (a.pcov)
        for (int e = lane; e < m * m; e += 32)
            a.pcov[((int64_t)t * m * m + e) * a.batch + b] = (float)Dd[(e / m) * ldm + e % m];
    if (bad && lane == 0 && a.status) atomicCAS(a.status + b, (int32_t)RXG_OK, (int32_t)RXG_ERR_NOT_SPD);
}

// Forecast covariance recursion S_k = A S_{k-1} A' + P from S_s[T-1], k = 1..H, fp64; one warp (= CTA) per chain
// (route A: one chain, the table).  out: element e of S_k at [((k-1) d^2 + e) * out_s + b * out_b].
__global__ void __launch_bounds__(32) k_forecast_cov(int d, int H, const float* __restrict__ A, const float* __restrict__ P,
                                                     int64_t ms, int64_t mb, const float* __restrict__ sig, int64_t sig_s,
                                                     int64_t sig_b, float* __restrict__ out, int64_t out_s, int64_t out_b) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int ld = d + 1, lane = threadIdx.x;
    const int64_t b = blockIdx.x;
    double* S = reinterpret_cast<double*>(smraw);
    double* W = S + d * ld;
    float* Af = reinterpret_cast<float*>(W + d * ld);
    float* Pf = Af + d * ld;
    for (int e = lane; e < d * d; e += 32) {
        const int i = e / d, j = e % d;
        S[i * ld + j] = (double)__ldg(sig + (int64_t)e * sig_s + b * sig_b);
        Af[i * ld + j] = __ldg(A + (int64_t)e * ms + b * mb);
        Pf[i * ld + j] = __ldg(P + (int64_t)e * ms + b * mb);
    }
    __syncwarp();
    for (int k = 0; k < H; ++k) {
        for (int j = lane; j < d; j += 32)                        // W = A S, lane per column
            for (int i = 0; i < d; ++i) {
                double s = 0.0;
                for (int p = 0; p < d; ++p) s = fma((double)Af[i * ld + p], S[p * ld + j], s);
                W[i * ld + j] = s;
            }
        __syncwarp();
        for (int j = lane; j < d; j += 32)                        // S = W A' + P, lower triangle, mirrored
            for (int i = j; i < d; ++i) {
                double s = 0.5 * ((double)Pf[i * ld + j] + (double)Pf[j * ld + i]);
                for (int p = 0; p < d; ++p) s = fma(W[i * ld + p], (double)Af[j * ld + p], s);
                S[i * ld + j] = S[j * ld + i] = s;
            }
        __syncwarp();
        for (int e = lane; e < d * d; e += 32)
            out[((int64_t)k * d * d + e) * out_s + b * out_b] = (float)S[(e / d) * ld + e % d];
        __syncwarp();
    }
}

// Forecast means x_k = A x_{k-1} + u from mu_s[T-1], one thread per chain; the state vectors live in shared memory
// ([d][FM_THREADS] per buffer: consecutive chains in consecutive banks).  With an input sequence (useq: row r at
// useq + r * d * ustride, + b if uchain) forecast k = 1..H adds row T + k - 1 instead of u.
__global__ void __launch_bounds__(FM_THREADS) k_forecast_mean(int d, int H, int64_t batch, const float* __restrict__ A,
                                                              const float* __restrict__ u, int64_t ms, int64_t mb,
                                                              const float* __restrict__ last_mean, float* __restrict__ out,
                                                              const float* __restrict__ useq, int64_t ustride, int uchain,
                                                              int T) {
    extern __shared__ float xs[];
    const int tid = threadIdx.x;
    const int64_t b = (int64_t)blockIdx.x * FM_THREADS + tid;
    if (b >= batch) return;
    float* x0 = xs;
    float* x1 = xs + d * FM_THREADS;
    for (int i = 0; i < d; ++i) x0[i * FM_THREADS + tid] = __ldg(last_mean + (int64_t)i * batch + b);
    for (int k = 0; k < H; ++k) {
        for (int i = 0; i < d; ++i) {
            float s = useq ? __ldg(useq + ((int64_t)(T + k) * d + i) * ustride + b * uchain)
                           : (u ? __ldg(u + (int64_t)i * ms + b * mb) : 0.f);
            for (int j = 0; j < d; ++j) s = __fmaf_rn(__ldg(A + (int64_t)(i * d + j) * ms + b * mb), x0[j * FM_THREADS + tid], s);
            x1[i * FM_THREADS + tid] = s;
            out[((int64_t)k * d + i) * batch + b] = s;
        }
        float* tmp = x0; x0 = x1; x1 = tmp;
    }
}

// Route A means at the native small shapes: y_hat = F_t y + G_t mu, one thread per chain, PM_TC steps per CTA with their
// tables staged in shared memory.  Rows t >= T are forecasts (mu from fmean, no y).
template <int D, int M>
__global__ void __launch_bounds__(256) k_predict_mean_small(int T, int TH, int64_t batch, const float* __restrict__ F,
                                                            const float* __restrict__ G, const uint8_t* __restrict__ tmask,
                                                            const float* __restrict__ y, const float* __restrict__ mean,
                                                            const float* __restrict__ fmean, float* __restrict__ pmean) {
    __shared__ float sF[PM_TC][M * M], sG[PM_TC][M * D];
    __shared__ int sObs[PM_TC];
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool on = b < batch;
    for (int t0 = blockIdx.y * PM_TC; t0 < TH; t0 += gridDim.y * PM_TC) {
        const int nt = TH - t0 < PM_TC ? TH - t0 : PM_TC;
        __syncthreads();                                              // the previous chunk's tables are no longer read
        for (int e = threadIdx.x; e < nt * M * M; e += blockDim.x) sF[e / (M * M)][e % (M * M)] = __ldg(F + (int64_t)t0 * M * M + e);
        for (int e = threadIdx.x; e < nt * M * D; e += blockDim.x) sG[e / (M * D)][e % (M * D)] = __ldg(G + (int64_t)t0 * M * D + e);
        for (int e = threadIdx.x; e < nt; e += blockDim.x) sObs[e] = (t0 + e < T) && (!tmask || tmask[t0 + e] != 0);
        __syncthreads();
        if (!on) continue;
        for (int q = 0; q < nt; ++q) {
            const int t = t0 + q;
            const float* mu = t < T ? mean + (int64_t)t * D * batch : fmean + (int64_t)(t - T) * D * batch;
            float x[D], o[M];
#pragma unroll
            for (int i = 0; i < D; ++i) x[i] = __ldg(mu + (int64_t)i * batch + b);
#pragma unroll
            for (int k = 0; k < M; ++k) {
                float s = 0.f;
#pragma unroll
                for (int j = 0; j < D; ++j) s = __fmaf_rn(sG[q][k * D + j], x[j], s);
                o[k] = s;
            }
            if (sObs[q]) {
                float yy[M];
#pragma unroll
                for (int l = 0; l < M; ++l) yy[l] = __ldg(y + ((int64_t)t * M + l) * batch + b);
#pragma unroll
                for (int k = 0; k < M; ++k)
#pragma unroll
                    for (int l = 0; l < M; ++l) o[k] = __fmaf_rn(sF[q][k * M + l], yy[l], o[k]);
            }
#pragma unroll
            for (int k = 0; k < M; ++k) pmean[((int64_t)t * M + k) * batch + b] = o[k];
        }
    }
}

template <int D, int M>
int launch_mean_small(rxg_ctx* ctx, int T, int TH, int64_t batch, const float* F, const float* G, const uint8_t* tmask,
                      const float* y, const float* mean, const float* fmean, float* pmean) {
    const int64_t gy = (TH + PM_TC - 1) / PM_TC;
    const dim3 grid((unsigned)((batch + 255) / 256), (unsigned)(gy < 65535 ? gy : 65535));
    k_predict_mean_small<D, M><<<grid, 256, 0, ctx->stream>>>(T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "k_predict_mean_small");
}

// native shapes with a register-resident mean kernel; returns RXG_ERR_UNSUPPORTED (without a message) for the others
int mean_small(rxg_ctx* ctx, int d, int m, int T, int TH, int64_t batch, const float* F, const float* G, const uint8_t* tmask,
               const float* y, const float* mean, const float* fmean, float* pmean) {
    switch (d * 16 + m) {
        case 1 * 16 + 1: return launch_mean_small<1, 1>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        case 2 * 16 + 1: return launch_mean_small<2, 1>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        case 2 * 16 + 2: return launch_mean_small<2, 2>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        case 3 * 16 + 3: return launch_mean_small<3, 3>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        case 4 * 16 + 1: return launch_mean_small<4, 1>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        case 4 * 16 + 2: return launch_mean_small<4, 2>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        case 4 * 16 + 4: return launch_mean_small<4, 4>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        case 6 * 16 + 6: return launch_mean_small<6, 6>(ctx, T, TH, batch, F, G, tmask, y, mean, fmean, pmean);
        default: return RXG_ERR_UNSUPPORTED;
    }
}

int set_smem(rxg_ctx* ctx, const void* fn, size_t smem, const char* what) {
    if (smem <= 48 * 1024) return RXG_OK;
    return check_cuda(ctx, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), what);
}

}  // namespace

int lgssm_predict_post(rxg_ctx* ctx, const LgssmCall& c, const PredictArgs& p) {
    const int d = c.d, m = c.m, T = c.T, H = p.H, TH = c.T + p.H;
    const int64_t batch = c.batch;
    const bool pc_model = (c.flags & RXG_MODEL_PER_CHAIN) != 0;
    const bool route_b = pc_model || (c.flags & RXG_PATH_PER_CHAIN) || c.ymask;
    const bool cov_shared = (c.flags & RXG_COV_SHARED_OUT) != 0;
    // source of S_s: the per-chain output (route B; chain 0 on route A), the [T][d][d] output, or the family's own table
    const float* sig = c.cov;
    int64_t sig_s = cov_shared ? 1 : batch;
    if (!route_b && !c.cov) {
        if (!c.cov_table)
            return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_smooth_predict (d=%d, m=%d): this kernel family keeps no covariance "
                                                  "table, pass post_cov", d, m);
        sig = c.cov_table; sig_s = 1;
    }
    // scratch: device copy of a shared model, route A tables, forecast buffers the caller did not ask for
    size_t off = 0;
    auto carve = [&](size_t nfloat) { size_t o = off; off += (nfloat * 4 + 255) / 256 * 256; return o; };
    const size_t nA = (size_t)d * d, nB = (size_t)m * d, nQ = (size_t)m * m;
    const size_t o_A = carve(pc_model ? 0 : nA), o_B = carve(pc_model ? 0 : nB), o_P = carve(pc_model ? 0 : nA);
    const size_t o_Q = carve(pc_model ? 0 : nQ), o_u = carve(pc_model || !c.u ? 0 : (size_t)d);
    const size_t o_F = carve(route_b ? 0 : (size_t)TH * nQ), o_G = carve(route_b ? 0 : (size_t)TH * nB);
    const bool own_C = !route_b && !(cov_shared && p.pred_cov);
    const size_t o_C = carve(own_C ? (size_t)TH * nQ : 0);
    const bool own_fs = H > 0 && !(p.fc_cov && (route_b || cov_shared));
    const size_t o_fs = carve(own_fs ? (size_t)H * nA * (route_b ? batch : 1) : 0);
    const bool own_fm = H > 0 && !p.fc_mean;
    const size_t o_fm = carve(own_fm ? (size_t)H * d * batch : 0);
    char* base = nullptr;          // nothing to carve (per-chain model, no owned forecast buffers): no scratch at all
    if (off > 0 && !(base = (char*)predict_scratch(ctx, off))) return RXG_ERR_CUDA;
    auto at = [&](size_t o) { return (float*)(base + o); };

    const float *A = c.A, *B = c.B, *P = c.P, *Q = c.Q, *u = c.u;
    const int64_t ms = pc_model ? batch : 1, mb = pc_model ? 1 : 0;
    if (!pc_model) {     // shared model: host arrays, staged (pageable sources are copied before the call returns)
        RXG_CUDA(ctx, cudaMemcpyAsync(at(o_A), c.A, nA * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(at(o_B), c.B, nB * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(at(o_P), c.P, nA * 4, cudaMemcpyHostToDevice, ctx->stream));
        RXG_CUDA(ctx, cudaMemcpyAsync(at(o_Q), c.Q, nQ * 4, cudaMemcpyHostToDevice, ctx->stream));
        if (c.u) RXG_CUDA(ctx, cudaMemcpyAsync(at(o_u), c.u, (size_t)d * 4, cudaMemcpyHostToDevice, ctx->stream));
        A = at(o_A); B = at(o_B); P = at(o_P); Q = at(o_Q); u = c.u ? at(o_u) : nullptr;
    }
    float* fsig = own_fs ? at(o_fs) : p.fc_cov;
    float* fmean = own_fm ? at(o_fm) : p.fc_mean;
    const int64_t nch = route_b ? batch : 1, sig_b = route_b ? 1 : 0;

    // ---- forecasts: covariance recursion (one warp per chain / the table) and means (one thread per chain)
    if (H > 0) {
        const size_t smem = (size_t)d * (d + 1) * (2 * 8 + 2 * 4);
        int rc = set_smem(ctx, (const void*)k_forecast_cov, smem, "cudaFuncSetAttribute(k_forecast_cov)");
        if (rc != RXG_OK) return rc;
        k_forecast_cov<<<(unsigned)nch, 32, smem, ctx->stream>>>(d, H, A, P, ms, mb, sig + (int64_t)(T - 1) * d * d * sig_s, sig_s,
                                                                 sig_b, fsig, route_b ? batch : 1, sig_b);
        k_forecast_mean<<<(unsigned)((batch + FM_THREADS - 1) / FM_THREADS), FM_THREADS, (size_t)2 * d * FM_THREADS * 4,
                          ctx->stream>>>(d, H, batch, A, u, ms, mb, c.mean + (int64_t)(T - 1) * d * batch, fmean,
                                         c.useq, c.useq_chain ? batch : 1, c.useq_chain ? 1 : 0, T);
        ctx->launches += 2;
        RXG_CUDA(ctx, cudaGetLastError());
    }

    // ---- the messages toward y: route A tables (one warp per step) or route B outputs (one warp per step and chain)
    MsgArgs a = {};
    a.d = d; a.m = m; a.T = T; a.H = H; a.batch = batch; a.per_chain = route_b ? 1 : 0;
    a.B = B; a.Q = Q; a.ms = ms; a.mb = mb;
    a.sig = sig; a.sig_s = sig_s; a.fsig = fsig; a.fsig_s = route_b ? batch : 1; a.sig_b = sig_b;
    a.tmask = c.tmask; a.ymask = c.ymask;
    float* Ctab = own_C ? at(o_C) : p.pred_cov;
    if (!route_b) { a.F = at(o_F); a.G = at(o_G); a.C = Ctab; a.bad = bad_flag(ctx); if (!a.bad) return RXG_ERR_CUDA; }
    a.y = c.y; a.mean = c.mean; a.fmean = fmean; a.pmean = p.pred_mean; a.pcov = p.pred_cov; a.status = c.status;
    {
        const MsgLayout L = msg_layout(d, m);
        int nw = (48 * 1024) / L.bytes;
        if (nw < 1) nw = 1;
        if (nw > PW_MAX_WARPS) nw = PW_MAX_WARPS;
        const size_t smem = (size_t)nw * L.bytes;
        int rc = set_smem(ctx, (const void*)k_predict_msg, smem, "cudaFuncSetAttribute(k_predict_msg)");
        if (rc != RXG_OK) return rc;
        const int64_t items = (int64_t)TH * nch;
        k_predict_msg<<<(unsigned)((items + nw - 1) / nw), 32 * nw, smem, ctx->stream>>>(a);
        ctx->launches += 1;
        RXG_CUDA(ctx, cudaGetLastError());
    }
    if (route_b) return RXG_OK;

    // ---- route A means: y_hat = F_t y + G_t mu
    int rc = mean_small(ctx, d, m, T, TH, batch, a.F, a.G, c.tmask, c.y, c.mean, fmean, p.pred_mean);
    if (rc == RXG_ERR_UNSUPPORTED) {
        // [m x d] . [d x batch] and [m x m] . [m x batch] per step: the left-GEMM with one matrix per slice
        rc = left_gemm_per_slice(ctx, m, d, batch, a.G, c.mean, p.pred_mean, T, (int64_t)d * batch, (int64_t)m * batch, 0);
        if (rc == RXG_OK)
            rc = left_gemm_per_slice(ctx, m, m, batch, a.F, c.y, p.pred_mean, T, (int64_t)m * batch, (int64_t)m * batch, 1);
        if (rc == RXG_OK && H > 0)
            rc = left_gemm_per_slice(ctx, m, d, batch, a.G + (size_t)T * nB, fmean, p.pred_mean + (int64_t)T * m * batch, H,
                                     (int64_t)d * batch, (int64_t)m * batch, 0);
    }
    if (rc != RXG_OK) return rc;
    // ---- per-chain covariance outputs: broadcast of the chain-independent tables
    if (p.pred_cov && !cov_shared) {
        rc = launch_replicate_cov(ctx, ctx->stream, Ctab, 1, p.pred_cov, (int64_t)TH * m * m, batch, 1, -1);
        if (rc != RXG_OK) return rc;
    }
    if (H > 0 && p.fc_cov && !cov_shared) {
        rc = launch_replicate_cov(ctx, ctx->stream, fsig, 1, p.fc_cov, (int64_t)H * d * d, batch, 1, -1);
        if (rc != RXG_OK) return rc;
    }
    if (c.status) return fill_status_from_flag(ctx, c.status, batch);
    return RXG_OK;
}

}  // namespace rxg
