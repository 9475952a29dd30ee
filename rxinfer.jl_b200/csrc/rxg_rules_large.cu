// Per-rule kernels for the Gaussian family at state sizes without a register-resident instantiation (d = 7, 9 ... 64;
// BASELINE configs[2] is d = 64: mu 64 floats, Sigma 4096 floats per message -- SURVEY.md 8a).  Same entry points, same
// structure-of-arrays layout ([row][col][n], message index innermost) as csrc/rxg_rules.cu; three building blocks:
//   * k_ew            element-wise rules (MvNormalMeanCovariance(:out / :mu), +(:out / :in), prod in (xi, W)): one flat pass,
//                     every access a full 128-byte line -- HBM bound like their small-d twins;
//   * k_left_gemm     Y[M][N] = op(A)[M x K] X[K][N] with a SHARED PointMass matrix A and a huge N: the layout makes both
//                     halves of `A S A'` (and of `A'W A`) plain left-multiplications -- S[r][c][n] is the row-major matrix
//                     [d] x [d n], and for a fixed first index the slab [c][n] is a [d] x [n] matrix.  One thread = one
//                     column, A' staged in shared memory and read as float4 (4 FMAs per LDS), up to 64 accumulators in
//                     registers.  CUDA cores: 2 M K flops per K + M floats of traffic = 16 flop/B at d = 64, i.e. FP32-issue
//                     bound (a tensor-core version of this product is what DESIGN.md section 7 lists next);
//   * k_cholinv_warp  FastCholesky.cholinv twin (every `mean_cov` / `weightedmean_precision` / *(:in) / marginal of the
//                     reference): one warp = one message, the matrix in shared memory (row stride d + 1: conflict-free for
//                     lane-per-row and lane-per-column access), left-looking Cholesky with lane-per-row, L^-1 by forward
//                     substitution with lane-per-column (stored transposed in the upper triangle), W = L^-T L^-1 written
//                     over the lower triangle; 8 messages per CTA so that global loads / stores are 32-byte sectors.
// [ref: rule bodies upstream ReactiveMP rules/multiplication, rules/mv_normal_mean_covariance, rules/addition; bound at
//  /root/reference/src/model/plugins/reactivemp_inference.jl:509-540; marginal fold :365-455]
#include "rxg_internal.h"

namespace rxg {

constexpr int RL_MSGS = 8;          // messages (= warps) per CTA of k_cholinv_warp (6 at d > 58, see cholinv_warp)

// o[r][i] = (a ? a[r][i] : 0) + sb * (b ? (b_bcast ? b[r] : b[r][i]) : 0)
__global__ void __launch_bounds__(256)
k_ew(int64_t rows, int64_t n, const float* __restrict__ a, const float* __restrict__ b, int b_bcast, float sb,
     float* __restrict__ o) {
    const int64_t total = rows * n;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        float v = a ? __ldg(a + idx) : 0.f;
        if (b) v = __fmaf_rn(sb, b_bcast ? __ldg(b + idx / n) : __ldg(b + idx), v);
        o[idx] = v;
    }
}

// Y = op(A) X per batch slice (blockIdx.y): op(A) is M x K; transA = 0: A stored M x K row-major; 1: A stored K x M row-major.
// MODE 0: one matrix for every slice; MODE 1: every slice its own matrix (A + slice * a_slice); MODE 2: as 1, and the
// product is added to Y.  A template parameter, so that the MODE 0 instantiations of the rule kernels keep their registers.
// A is staged per CTA (coalesced global reads; shared-memory row stride MMAX + 4 keeps the float4 reads aligned and the
// transposing stores at 4-way instead of 32-way bank conflicts).  One thread = LG_NC columns (j, j + 128): every float4 of A'
// read from shared memory feeds 4 * LG_NC FMAs -- with one column per thread the broadcast LDS.128 stream (16 per row at
// M = 64, one shared-memory pipe for the four schedulers) costs as many cycles as the 64 FMAs it feeds.
constexpr int LG_NC = 2;
template <int MMAX, int MODE>
__global__ void __launch_bounds__(128)
k_left_gemm(int M, int K, int64_t N, const float* __restrict__ A, int transA, const float* __restrict__ X,
            float* __restrict__ Y, int64_t x_slice, int64_t y_slice, int64_t a_slice) {
    extern __shared__ __align__(16) float At[];                      // [K][LDA]: At[k][m] = op(A)(m, k), zero padded
    if (MODE > 0) A += (int64_t)blockIdx.y * a_slice;
    constexpr int LDA = MMAX + 4;
    for (int idx = threadIdx.x; idx < K * LDA; idx += blockDim.x) At[idx] = 0.f;
    __syncthreads();
    for (int idx = threadIdx.x; idx < M * K; idx += blockDim.x) {
        const int m = transA ? idx % M : idx / K, k = transA ? idx / M : idx % K;      // idx walks A as it lies in memory
        At[k * LDA + m] = __ldg(A + idx);
    }
    __syncthreads();
    X += (int64_t)blockIdx.y * x_slice;
    Y += (int64_t)blockIdx.y * y_slice;
    int64_t j[LG_NC];
    bool on[LG_NC];
#pragma unroll
    for (int c = 0; c < LG_NC; ++c) {
        j[c] = ((int64_t)blockIdx.x * LG_NC + c) * blockDim.x + threadIdx.x;
        on[c] = j[c] < N;
        if (!on[c]) j[c] = N - 1;                                     // clamp: loads stay in bounds, the store is skipped
    }
    float acc[LG_NC][MMAX];
#pragma unroll
    for (int c = 0; c < LG_NC; ++c)
#pragma unroll
        for (int m = 0; m < MMAX; ++m) acc[c][m] = 0.f;
    float xn[LG_NC];
#pragma unroll
    for (int c = 0; c < LG_NC; ++c) xn[c] = __ldg(X + j[c]);
    for (int k = 0; k < K; ++k) {
        float x[LG_NC];
#pragma unroll
        for (int c = 0; c < LG_NC; ++c) {
            x[c] = xn[c];
            if (k + 1 < K) xn[c] = __ldg(X + (int64_t)(k + 1) * N + j[c]);   // next row in flight under this row's FMAs
        }
        const float4* a4 = reinterpret_cast<const float4*>(At + k * LDA);
#pragma unroll
        for (int q = 0; q < MMAX / 4; ++q) {
            const float4 a = a4[q];
#pragma unroll
            for (int c = 0; c < LG_NC; ++c) {
                acc[c][4 * q + 0] = __fmaf_rn(a.x, x[c], acc[c][4 * q + 0]);
                acc[c][4 * q + 1] = __fmaf_rn(a.y, x[c], acc[c][4 * q + 1]);
                acc[c][4 * q + 2] = __fmaf_rn(a.z, x[c], acc[c][4 * q + 2]);
                acc[c][4 * q + 3] = __fmaf_rn(a.w, x[c], acc[c][4 * q + 3]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < LG_NC; ++c)
        if (on[c]) {
#pragma unroll
            for (int m = 0; m < MMAX; ++m)
                if (m < M) Y[(int64_t)m * N + j[c]] = MODE == 2 ? acc[c][m] + Y[(int64_t)m * N + j[c]] : acc[c][m];
        }
}

struct RuleList { const float* v[8]; const float* M[8]; };

// (vo, Mo) = (Minv vsum, Minv),  Minv = cholinv(sum_q M_q),  vsum = sum_q v_q     (k = 1: mean_cov / weightedmean_precision;
// k > 1: marginal = product of k (xi, W) messages, then mean_cov).  vo / Mo may be null (only the other one is wanted).
__global__ void __launch_bounds__(32 * RL_MSGS)
k_cholinv_warp(int64_t n, int d, int k, RuleList in, float* __restrict__ vo, float* __restrict__ Mo,
               int32_t* __restrict__ status) {
    extern __shared__ float sm[];
    const int ld = d + 1;
    const int per = d * ld + 3 * d;                                   // matrix, reciprocal diagonal, v, result
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nm = blockDim.x >> 5;                                   // messages (= warps) of this CTA: 8, or 6 when 8 would not leave room for two CTAs per SM
    const int64_t i0 = (int64_t)blockIdx.x * nm;
    // ---- cooperative load (+ sum over the k inputs): 8 consecutive messages per (row, col) = one 32-byte sector
    for (int e = threadIdx.x; e < d * d * nm; e += blockDim.x) {
        const int msg = e % nm, el = e / nm;
        const int64_t i = i0 + msg;
        if (i < n) {
            float s = 0.f;
            for (int q = 0; q < k; ++q) s += __ldg(in.M[q] + (int64_t)el * n + i);
            sm[msg * per + (el / d) * ld + (el % d)] = s;
        }
    }
    for (int e = threadIdx.x; e < d * nm; e += blockDim.x) {
        const int msg = e % nm, el = e / nm;
        const int64_t i = i0 + msg;
        if (i < n) {
            float s = 0.f;
            for (int q = 0; q < k; ++q) s += __ldg(in.v[q] + (int64_t)el * n + i);
            sm[msg * per + d * ld + d + el] = s;
        }
    }
    __syncthreads();
    const int64_t i = i0 + warp;
    float* L = sm + warp * per;
    float* rd = L + d * ld;
    float* v = rd + d;
    float* res = v + d;
    bool bad = false;
    if (i < n) {
        // ---- left-looking Cholesky, lane per row: column j of L from columns 0 .. j-1
        const int r0 = lane, r1 = lane + 32;                              // the (at most) two rows of this lane
        for (int j = 0; j < d; ++j) {
            float t0 = 0.f, t1 = 0.f;
            if (r0 < d && r0 >= j) {
                t0 = L[r0 * ld + j];
                for (int c = 0; c < j; ++c) t0 = __fmaf_rn(-L[r0 * ld + c], L[j * ld + c], t0);
            }
            if (r1 < d && r1 >= j) {
                t1 = L[r1 * ld + j];
                for (int c = 0; c < j; ++c) t1 = __fmaf_rn(-L[r1 * ld + c], L[j * ld + c], t1);
            }
            if ((j & 31) == lane) {
                float p = (j < 32) ? t0 : t1;
                if (!(p > 0.f)) { bad = true; p = 1e-30f; }
                const float sq = sqrtf(p);
                L[j * ld + j] = sq;
                rd[j] = 1.f / sq;
            }
            __syncwarp();
            const float rj = rd[j];
            if (r0 < d && r0 > j) L[r0 * ld + j] = t0 * rj;
            if (r1 < d && r1 > j) L[r1 * ld + j] = t1 * rj;
            __syncwarp();
        }
        bad = __any_sync(0xffffffffu, bad);
        // ---- X = L^-1, lane per column c; X[r][c] (r > c) is kept at U[c][r] (upper triangle), X[c][c] = rd[c].
        //      (Lane-private loop bounds: measured faster than warp-uniform loops with predicates, 3.9 vs 5.7 ms for
        //      16 384 messages at d = 64 -- the uniform version does twice the iterations.)
        for (int c = lane; c < d; c += 32) {
            const float xc = rd[c];
            for (int r = c + 1; r < d; ++r) {
                float s = L[r * ld + c] * xc;
                for (int q = c + 1; q < r; ++q) s = __fmaf_rn(L[r * ld + q], L[c * ld + q], s);      // L[r][q] X[q][c]
                L[c * ld + r] = -s * rd[r];
            }
        }
        __syncwarp();
        // ---- W = X'X, lane per column b, lower triangle a >= b:  W[a][b] = sum_{r >= a} X[r][a] X[r][b]
        //      (reads the upper triangle + rd, writes the lower triangle: no overlap)
        for (int b = lane; b < d; b += 32) {
            for (int a = b; a < d; ++a) {
                const float xaa = rd[a];
                float s = xaa * ((a == b) ? xaa : L[b * ld + a]);                                       // r = a
                for (int r = a + 1; r < d; ++r) s = __fmaf_rn(L[a * ld + r], L[b * ld + r], s);
                L[a * ld + b] = s;
            }
        }
        __syncwarp();
        // the upper triangle still holds X: mirror W over it so that the store loop reads a full matrix
        for (int b = lane; b < d; b += 32)
            for (int a = b + 1; a < d; ++a) L[b * ld + a] = L[a * ld + b];
        __syncwarp();
        // ---- res = W v, lane per row
        for (int r = lane; r < d; r += 32) {
            float s = 0.f;
            for (int c = 0; c < d; ++c) s = __fmaf_rn(L[r * ld + c], v[c], s);
            res[r] = s;
        }
        if (status && lane == 0) status[i] = bad ? RXG_ERR_NOT_SPD : RXG_OK;
    }
    __syncthreads();
    if (Mo)
        for (int e = threadIdx.x; e < d * d * nm; e += blockDim.x) {
            const int msg = e % nm, el = e / nm;
            const int64_t ii = i0 + msg;
            if (ii < n) Mo[(int64_t)el * n + ii] = sm[msg * per + (el / d) * ld + (el % d)];
        }
    if (vo)
        for (int e = threadIdx.x; e < d * nm; e += blockDim.x) {
            const int msg = e % nm, el = e / nm;
            const int64_t ii = i0 + msg;
            if (ii < n) vo[(int64_t)el * n + ii] = sm[msg * per + d * ld + 2 * d + el];
        }
}

// ------------------------------------------------------------------------------------------------ host side
bool rules_small(int d) { return (d >= 1 && d <= 6) || d == 8; }
bool rules_small2(int dout, int din) {
    switch (dout * 16 + din) {
        case 1 * 16 + 1: case 1 * 16 + 2: case 2 * 16 + 2: case 3 * 16 + 3: case 1 * 16 + 4: case 2 * 16 + 4: case 4 * 16 + 4:
        case 6 * 16 + 6: case 8 * 16 + 8: return dout <= 8 && din <= 8;
        default: return false;
    }
}

static int ew(rxg_ctx* ctx, int64_t rows, int64_t n, const float* a, const float* b, int bcast, float sb, float* o) {
    const int64_t total = rows * n;
    if (total == 0) return RXG_OK;
    const int64_t want = (total + 255) / 256, cap = (int64_t)ctx->sm_count * 16;
    const unsigned grid = (unsigned)(want < cap ? want : cap);
    k_ew<<<grid, 256, 0, ctx->stream>>>(rows, n, a, b, bcast, sb, o);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "k_ew");
}
static int left_gemm(rxg_ctx* ctx, int M, int K, int64_t N, const float* A, int transA, const float* X, float* Y, int slices,
                     int64_t x_slice, int64_t y_slice, int64_t a_slice = 0, int accumulate = 0) {
    const dim3 grid((unsigned)((N + 128 * LG_NC - 1) / (128 * LG_NC)), (unsigned)slices);
    const int mmax = M <= 16 ? 16 : (M <= 32 ? 32 : 64);
    const size_t smem = (size_t)K * (mmax + 4) * sizeof(float);
    const int mode = a_slice == 0 ? 0 : (accumulate ? 2 : 1);
#define RXG_LG(MM, MO) k_left_gemm<MM, MO><<<grid, 128, smem, ctx->stream>>>(M, K, N, A, transA, X, Y, x_slice, y_slice, a_slice)
#define RXG_LG_MODES(MM) do { if (mode == 0) RXG_LG(MM, 0); else if (mode == 1) RXG_LG(MM, 1); else RXG_LG(MM, 2); } while (0)
    if (mmax == 16) RXG_LG_MODES(16);
    else if (mmax == 32) RXG_LG_MODES(32);
    else RXG_LG_MODES(64);
#undef RXG_LG_MODES
#undef RXG_LG
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "k_left_gemm");
}
// Y[s] (+)= A[s] X[s] for `slices` slices with one row-major M x K matrix per slice (a_slice = M K); the grid's y dimension
// caps one launch at 65 535 slices
int left_gemm_per_slice(rxg_ctx* ctx, int M, int K, int64_t N, const float* A, const float* X, float* Y, int64_t slices,
                        int64_t x_slice, int64_t y_slice, int accumulate) {
    for (int64_t s0 = 0; s0 < slices; s0 += 65535) {
        const int64_t ns = slices - s0 < 65535 ? slices - s0 : 65535;
        int rc = left_gemm(ctx, M, K, N, A + s0 * M * K, 0, X + s0 * x_slice, Y + s0 * y_slice, (int)ns, x_slice, y_slice,
                           (int64_t)M * K, accumulate);
        if (rc != RXG_OK) return rc;
    }
    return RXG_OK;
}
static int cholinv_warp(rxg_ctx* ctx, int64_t n, int d, int k, const RuleList& in, float* vo, float* Mo, int32_t* status) {
    // 8 messages per CTA (one 32-byte sector per element) unless that leaves room for only one CTA per SM (d > 58): then 6,
    // so that two CTAs = 12 warps share an SM -- the kernel is latency bound
    const size_t per_msg = ((size_t)d * (d + 1) + 3 * d) * sizeof(float);
    const int nm = (RL_MSGS * per_msg > 113 * 1024) ? 6 : RL_MSGS;
    const size_t smem = nm * per_msg;
    if (smem > 48 * 1024) {   // per-device function attribute: set on every call (microseconds), no per-process "done" flag
        int rc = check_cuda(ctx, cudaFuncSetAttribute(k_cholinv_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                            "cudaFuncSetAttribute(k_cholinv_warp)");
        if (rc != RXG_OK) return rc;
    }
    k_cholinv_warp<<<(unsigned)((n + nm - 1) / nm), 32 * nm, smem, ctx->stream>>>(n, d, k, in, vo, Mo, status);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "k_cholinv_warp");
}

#define RXG_TRY(x) do { int _rc = (x); if (_rc != RXG_OK) return _rc; } while (0)

// (mu, S + Sigma)   /   from data: (y, Sigma)
int rules_large_add_cov(rxg_ctx* ctx, int64_t n, int d, const float* mu_in, const float* S_in, const float* Sigma, int shared,
                        float* mu_out, float* S_out) {
    RXG_TRY(ew(ctx, d, n, mu_in, nullptr, 0, 0.f, mu_out));
    return ew(ctx, (int64_t)d * d, n, S_in, Sigma, shared, 1.f, S_out);
}
// (v1 + sv v2, M1 + M2)
int rules_large_pair_axpy(rxg_ctx* ctx, int64_t n, int d, const float* v1, const float* M1, const float* v2, const float* M2,
                          float sv, float* vo, float* Mo) {
    RXG_TRY(ew(ctx, d, n, v1, v2, 0, sv, vo));
    return ew(ctx, (int64_t)d * d, n, M1, M2, 0, 1.f, Mo);
}
// (A mu, A S A'), A shared
int rules_large_mul_out(rxg_ctx* ctx, int64_t n, int dout, int din, const float* A, const float* mu_in, const float* S_in,
                        float* mu_out, float* S_out) {
    float* T = (float*)workspace(ctx, (size_t)dout * din * n * sizeof(float));
    if (!T) return RXG_ERR_CUDA;
    RXG_TRY(left_gemm(ctx, dout, din, n, A, 0, mu_in, mu_out, 1, 0, 0));
    RXG_TRY(left_gemm(ctx, dout, din, (int64_t)din * n, A, 0, S_in, T, 1, 0, 0));                 // T[o][c][i] = sum_r A[o][r] S[r][c][i]
    return left_gemm(ctx, dout, din, n, A, 0, T, S_out, dout, (int64_t)din * n, (int64_t)dout * n); // Z[o][p][i] = sum_c A[p][c] T[o][c][i]
}
// (A' W mu, A' W A), W = cholinv(S_out), A shared (dout x din)
int rules_large_mul_in(rxg_ctx* ctx, int64_t n, int dout, int din, const float* A, const float* mu_out, const float* S_out,
                       float* xi_in, float* W_in, int32_t* status) {
    const size_t nW = (size_t)dout * dout * n, nx = (size_t)dout * n, nT = (size_t)dout * din * n;
    float* ws = (float*)workspace(ctx, (nW + nx + nT) * sizeof(float));
    if (!ws) return RXG_ERR_CUDA;
    float *W = ws, *xo = ws + nW, *T = xo + nx;
    RuleList in = {};
    in.v[0] = mu_out; in.M[0] = S_out;
    RXG_TRY(cholinv_warp(ctx, n, dout, 1, in, xo, W, status));
    RXG_TRY(left_gemm(ctx, din, dout, n, A, 1, xo, xi_in, 1, 0, 0));                               // A' (W mu)
    RXG_TRY(left_gemm(ctx, din, dout, n, A, 1, W, T, dout, (int64_t)dout * n, (int64_t)din * n));  // T[r][c][i] = sum_k A[k][c] W[r][k][i]
    return left_gemm(ctx, din, dout, (int64_t)din * n, A, 1, T, W_in, 1, 0, 0);                    // Win[a][c][i] = sum_r A[r][a] T[r][c][i]
}
// k = 1: conversions between (mu, S) and (xi, W); k > 1: marginal of k (xi, W) messages
int rules_large_convert(rxg_ctx* ctx, int64_t n, int d, int k, const float* const* v_list, const float* const* M_list,
                        float* vo, float* Mo, int32_t* status) {
    RuleList in = {};
    for (int q = 0; q < k; ++q) { in.v[q] = v_list[q]; in.M[q] = M_list[q]; }
    return cholinv_warp(ctx, n, d, k, in, vo, Mo, status);
}

}  // namespace rxg
