// General-shape front end of the fused LGSSM sweeps: routes ANY (d, m) in 1..64 to a kernel family.
//
//   native shapes (register kernels d <= 6, large-state family d = m in {8,16,32,64})  -> as before
//   per-chain models / missing data / forced per-chain path at other shapes            -> lgssm_generic_chain (one CTA per chain)
//   shared model at any other (d, m)                                                   -> EMBEDDED in the next native shape
//   transition offset u on the large-state family                                      -> removed by linearity
//
// Embedding: the model is padded to (D', M') >= (d, m) with decoupled dummy coordinates,
//     A' = [A 0; 0 0]   P' = [P 0; 0 I]   S0' = [S0 0; 0 I]   m0' = [m0; 0]   u' = [u; 0]
//     B' = [B 0; 0 0]   Q' = [Q 0; 0 I]   y'  = [y; 0]
// Block-diagonal structure is preserved exactly by every message of the schedule (zeros stay zeros in floating
// point), so the posteriors of the real coordinates are those of the original model; each dummy observation adds
// exactly 1/2 log 2 pi per step to the evidence (innovation 0, innovation variance 1), which is subtracted.
// Offset by linearity: x_t = z_t + xi_t with the deterministic trajectory z_t = A z_{t-1} + u_t (z = 0 at the prior;
// u_t = u for a constant offset, row t of the input sequence with RXG_U_SEQ_*); xi follows the offset-free model
// observed through y_t - B z_t, covariances and evidence are unchanged (the shift has a Jacobian of 1), and
// E[x_t | y] = z_t + E[xi_t | y].  A shared offset / sequence gives one host trajectory (fp64); a per-chain sequence
// gives one trajectory per chain (input_traj_kernel).
// [ref: the reference handles any d, m and the `+` node generically: test/models/statespace/mlgssm_test.jl:8-17,
//  ulgssm_tests.jl:7-16.]
#include <math.h>

#include <vector>

#include "rxg_internal.h"

namespace rxg {

namespace {

__global__ void pad_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int T, int r, int R, int64_t batch) {
    // dst[t][k][b] = k < r ? src[t][k][b] : 0
    const int64_t n = (int64_t)T * R * batch;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i % batch, tk = i / batch;
        const int k = (int)(tk % R);
        const int64_t t = tk / R;
        dst[i] = k < r ? __ldg(src + (t * r + k) * batch + b) : 0.f;
    }
}
__global__ void unpad_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int T, int r, int R, int64_t batch) {
    // dst[t][k][b] = src[t][k][b], k < r  (src has R rows per step)
    const int64_t n = (int64_t)T * r * batch;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i % batch, tk = i / batch;
        const int k = (int)(tk % r);
        const int64_t t = tk / r;
        dst[i] = __ldg(src + (t * R + k) * batch + b);
    }
}
// cov[t][i][j][b] = tab[t][i][j] (sub-block of a [T][R][R] table), or the [T][r][r] table itself when batch == 0
__global__ void subblock_cov_kernel(const float* __restrict__ tab, float* __restrict__ cov, int T, int r, int R, int64_t batch) {
    const int64_t row = blockIdx.x;                      // (t, i, j)
    const int j = (int)(row % r), i = (int)((row / r) % r);
    const int64_t t = row / ((int64_t)r * r);
    const float v = __ldg(tab + (t * R + i) * R + j);
    if (batch == 0) { if (threadIdx.x == 0 && blockIdx.y == 0) cov[row] = v; return; }
    float* out = cov + row * batch;
    for (int64_t b = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; b < batch; b += (int64_t)gridDim.y * blockDim.x) out[b] = v;
}
// mask[t][b] = tmask[t]: a shared pattern expanded for the kernel families that only know per-chain masks
__global__ void expand_mask_kernel(const uint8_t* __restrict__ tmask, uint8_t* __restrict__ mask, int T, int64_t batch) {
    const int64_t n = (int64_t)T * batch;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) mask[i] = tmask[i / batch];
}
__global__ void add_const_kernel(float* __restrict__ v, int64_t n, float c) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] += c;
}
// dst[t][k][b] = src[t][k][b] + sign * traj[t][k]
__global__ void shift_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, const float* __restrict__ traj,
                                  int64_t rows, int64_t batch, float sign) {
    const int64_t n = rows * batch;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = src[i] + sign * __ldg(traj + i / batch);
}

unsigned grid_for(rxg_ctx* ctx, int64_t n) {
    int64_t g = (n + 255) / 256;
    const int64_t cap = (int64_t)ctx->sm_count * 16;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

void* aux(rxg_ctx* ctx, int slot, size_t bytes) {
    if (ctx->aux_bytes[slot] >= bytes && ctx->aux_buf[slot]) return ctx->aux_buf[slot];
    if (ctx->aux_buf[slot]) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->aux_buf[slot]); ctx->aux_buf[slot] = nullptr; ctx->aux_bytes[slot] = 0; }
    const size_t sz = (bytes + ((size_t)1 << 20) - 1) >> 20 << 20;
    if (cudaMalloc(&ctx->aux_buf[slot], sz) != cudaSuccess) { check_cuda(ctx, cudaGetLastError(), "cudaMalloc(aux)"); ctx->aux_buf[slot] = nullptr; return nullptr; }
    ctx->aux_bytes[slot] = sz;
    return ctx->aux_buf[slot];
}

bool small_native(int d, int m) {
    switch (d * 16 + m) {
        case 1 * 16 + 1: case 2 * 16 + 1: case 2 * 16 + 2: case 3 * 16 + 3:
        case 4 * 16 + 1: case 4 * 16 + 2: case 4 * 16 + 4: case 6 * 16 + 6: return true;
        default: return false;
    }
}
// smallest native shape that contains (d, m)
bool embedding_shape(int d, int m, int* D, int* M) {
    static const int cand[][2] = {{1, 1}, {2, 1}, {2, 2}, {3, 3}, {4, 1}, {4, 2}, {4, 4}, {6, 6}, {8, 8}, {16, 16}, {32, 32}, {64, 64}};
    for (const auto& c : cand)
        if (c[0] >= d && c[1] >= m) { *D = c[0]; *M = c[1]; return true; }
    return false;
}

// z_t = A z_{t-1} + u_t per chain (u[T][d][batch]; z = 0 at the prior and at t = 0 without a transition), written to
// z[T][d][batch], and ys = y - B z_t.  Block = 32 chains x NY row threads; A and B in shared memory (broadcast reads),
// z_{t-1} / z_t of the 32 chains double buffered in shared memory: one barrier per step.
__global__ void __launch_bounds__(1024) input_traj_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                          const float* __restrict__ u, const float* __restrict__ y,
                                                          float* __restrict__ ys, float* __restrict__ z, int d, int m, int T,
                                                          int64_t batch, int tf) {
    extern __shared__ float sh[];
    float* sA = sh;                    // d x d
    float* sB = sA + d * d;            // m x d
    float* sz = sB + m * d;            // [2][d][32]
    const int lane = threadIdx.x, ny = blockDim.y;
    const int tid = threadIdx.y * 32 + lane, nt = 32 * ny;
    for (int e = tid; e < d * d; e += nt) sA[e] = A[e];
    for (int e = tid; e < m * d; e += nt) sB[e] = B[e];
    const int64_t b = (int64_t)blockIdx.x * 32 + lane;
    const bool on = b < batch;
    __syncthreads();
    for (int t = 0; t < T; ++t) {
        const float* zp = sz + ((t + 1) & 1) * d * 32;
        float* zc = sz + (t & 1) * d * 32;
        const bool pred = t > 0 || tf;
        for (int i = threadIdx.y; i < d; i += ny) {
            float s = 0.f;
            if (pred && on) {
                s = __ldg(u + ((int64_t)t * d + i) * batch + b);
                if (t > 0)
                    for (int j = 0; j < d; ++j) s = __fmaf_rn(sA[i * d + j], zp[j * 32 + lane], s);
            }
            zc[i * 32 + lane] = s;
            if (on) z[((int64_t)t * d + i) * batch + b] = s;
        }
        __syncthreads();
        if (on)
            for (int k = threadIdx.y; k < m; k += ny) {
                float s = __ldg(y + ((int64_t)t * m + k) * batch + b);
                for (int j = 0; j < d; ++j) s = __fmaf_rn(-sB[k * d + j], zc[j * 32 + lane], s);
                ys[((int64_t)t * m + k) * batch + b] = s;
            }
    }
}
__global__ void add_kernel(float* __restrict__ v, const float* __restrict__ w, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) v[i] += __ldg(w + i);
}

// offset / input sequence on the large-state family, removed by linearity (shared model)
int large_with_offset(rxg_ctx* ctx, LgssmCall& c) {
    if (c.useq_chain) {
        const int d = c.d, m = c.m, T = c.T;
        const int64_t batch = c.batch;
        const size_t nz = (size_t)T * d * batch, ny = (size_t)T * m * batch;
        size_t off = 0;
        auto carve = [&](size_t n) { size_t o = off; off += (n * 4 + 255) / 256 * 256; return o; };
        const size_t o_AB = carve((size_t)d * d + (size_t)m * d), o_ys = carve(c.tables_only ? 0 : ny);
        char* base = (char*)aux(ctx, 3, off);
        float* zb = (float*)aux(ctx, 2, nz * 4);
        if (!base || !zb) return RXG_ERR_CUDA;
        float *dAB = (float*)(base + o_AB), *ys = (float*)(base + o_ys);
        LgssmCall c2 = c;
        c2.useq = nullptr; c2.useq_chain = false;
        if (!c.tables_only) {
            RXG_CUDA(ctx, cudaMemcpyAsync(dAB, c.A, (size_t)d * d * 4, cudaMemcpyHostToDevice, ctx->stream));
            RXG_CUDA(ctx, cudaMemcpyAsync(dAB + (size_t)d * d, c.B, (size_t)m * d * 4, cudaMemcpyHostToDevice, ctx->stream));
            const int rows = d > m ? d : m, nyt = rows < 32 ? rows : 32;
            const size_t smem = ((size_t)d * d + (size_t)m * d + 2 * (size_t)d * 32) * 4;
            RXG_CUDA(ctx, cudaFuncSetAttribute(input_traj_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            input_traj_kernel<<<(unsigned)((batch + 31) / 32), dim3(32, nyt), smem, ctx->stream>>>(
                dAB, dAB + (size_t)d * d, c.useq, c.y, ys, zb, d, m, T, batch, (c.flags & RXG_TRANSITION_FIRST) ? 1 : 0);
            ctx->launches += 1;
            RXG_CUDA(ctx, cudaGetLastError());
            c2.y = ys;
        }
        int rc = lgssm_large_dispatch(ctx, c2);
        if (rc != RXG_OK) return rc;
        if (!c.tables_only && c.mean) {
            add_kernel<<<grid_for(ctx, (int64_t)nz), 256, 0, ctx->stream>>>(c.mean, zb, (int64_t)nz);
            ctx->launches += 1;
        }
        c.fused_peer_stores = false;
        return check_cuda(ctx, cudaGetLastError(), "input trajectory kernels");
    }
    const int d = c.d, m = c.m, T = c.T;
    std::vector<double> z((size_t)d, 0.0), zn((size_t)d);
    std::vector<float> traj((size_t)T * d), btraj((size_t)T * m);
    const bool tf = (c.flags & RXG_TRANSITION_FIRST) != 0;
    for (int t = 0; t < T; ++t) {
        if (t > 0 || tf) {
            const float* ut = c.useq_host ? c.useq_host + (size_t)t * d : c.u;
            for (int i = 0; i < d; ++i) {
                double s = (double)ut[i];
                for (int j = 0; j < d; ++j) s += (double)c.A[i * d + j] * z[j];
                zn[i] = s;
            }
            z = zn;
        }
        for (int i = 0; i < d; ++i) traj[(size_t)t * d + i] = (float)z[i];
        for (int k = 0; k < m; ++k) {
            double s = 0.0;
            for (int j = 0; j < d; ++j) s += (double)c.B[k * d + j] * z[j];
            btraj[(size_t)t * m + k] = (float)s;
        }
    }
    const size_t ny = (size_t)T * m * c.batch;
    float* tr = (float*)aux(ctx, 2, ((size_t)T * (d + m)) * 4);
    float* ys = (float*)aux(ctx, 3, ny * 4);
    if (!tr || !ys) return RXG_ERR_CUDA;
    float* btr = tr + (size_t)T * d;
    // pageable host source: the copy is staged by the runtime before the call returns
    RXG_CUDA(ctx, cudaMemcpyAsync(tr, traj.data(), traj.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaMemcpyAsync(btr, btraj.data(), btraj.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    LgssmCall c2 = c;
    c2.u = nullptr; c2.useq = nullptr; c2.useq_host = nullptr;
    if (!c.tables_only) {
        shift_rows_kernel<<<grid_for(ctx, (int64_t)ny), 256, 0, ctx->stream>>>(c.y, ys, btr, (int64_t)T * m, c.batch, -1.f);
        c2.y = ys;
    }
    int rc = lgssm_large_dispatch(ctx, c2);
    if (rc != RXG_OK) return rc;
    if (!c.tables_only && c.mean) {
        const int64_t nm = (int64_t)T * d * c.batch;
        shift_rows_kernel<<<grid_for(ctx, nm), 256, 0, ctx->stream>>>(c.mean, c.mean, tr, (int64_t)T * d, c.batch, +1.f);
    }
    ctx->launches += 2;
    c.fused_peer_stores = false;
    return check_cuda(ctx, cudaGetLastError(), "offset shift kernels");
}

int embedded(rxg_ctx* ctx, LgssmCall& c, int D, int M) {
    const int d = c.d, m = c.m, T = c.T;
    const int64_t batch = c.batch;
    std::vector<float> A((size_t)D * D, 0.f), B((size_t)M * D, 0.f), P((size_t)D * D, 0.f), Q((size_t)M * M, 0.f),
        S0((size_t)D * D, 0.f), m0((size_t)D, 0.f), u((size_t)D, 0.f);
    for (int i = 0; i < d; ++i) {
        for (int j = 0; j < d; ++j) { A[i * D + j] = c.A[i * d + j]; P[i * D + j] = c.P[i * d + j]; S0[i * D + j] = c.S0[i * d + j]; }
        m0[i] = c.m0[i];
        if (c.u) u[i] = c.u[i];
    }
    for (int i = d; i < D; ++i) { P[i * D + i] = 1.f; S0[i * D + i] = 1.f; }
    for (int k = 0; k < m; ++k) {
        for (int j = 0; j < d; ++j) B[k * D + j] = c.B[k * d + j];
        for (int l = 0; l < m; ++l) Q[k * M + l] = c.Q[k * m + l];
    }
    for (int k = m; k < M; ++k) Q[k * M + k] = 1.f;
    const bool want_cov = c.cov != nullptr;
    const bool cov_shared = (c.flags & RXG_COV_SHARED_OUT) != 0;
    const size_t n_y = (size_t)T * M * batch, n_mean = (size_t)T * D * batch, n_tab = (size_t)T * D * D, n_m0 = (size_t)D * batch;
    size_t off = 0;
    auto carve = [&](size_t n) { size_t o = off; off += (n * 4 + 255) / 256 * 256; return o; };
    const size_t o_y = carve(c.tables_only ? 0 : n_y), o_mean = carve(c.tables_only ? 0 : n_mean);
    const size_t o_tab = carve(want_cov ? n_tab : 0), o_m0 = carve(c.mean0_chain ? n_m0 : 0);
    const size_t o_u = carve(c.useq ? (size_t)T * D * (c.useq_chain ? batch : 1) : 0);
    std::vector<float> useq_pad(c.useq_host ? (size_t)T * D : 0, 0.f);     // shared input sequence, padded on the host
    for (size_t t = 0; c.useq_host && t < (size_t)T; ++t)
        for (int i = 0; i < d; ++i) useq_pad[t * D + i] = c.useq_host[t * d + i];
    char* base = (char*)aux(ctx, 0, off);
    if (!base) return RXG_ERR_CUDA;
    float *yp = (float*)(base + o_y), *meanp = (float*)(base + o_mean), *tab = (float*)(base + o_tab), *m0p = (float*)(base + o_m0);
    LgssmCall c2 = c;
    c2.d = D; c2.m = M;
    c2.A = A.data(); c2.B = B.data(); c2.P = P.data(); c2.Q = Q.data(); c2.m0 = m0.data(); c2.S0 = S0.data();
    c2.u = c.u ? u.data() : nullptr;
    if (c.useq) {
        float* up = (float*)(base + o_u);
        if (c.useq_chain) {
            pad_rows_kernel<<<grid_for(ctx, (int64_t)T * D * batch), 256, 0, ctx->stream>>>(c.useq, up, T, d, D, batch);
            ctx->launches += 1;
        } else {
            // pageable host source: the runtime has read it before the call returns
            RXG_CUDA(ctx, cudaMemcpyAsync(up, useq_pad.data(), useq_pad.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
            c2.useq_host = useq_pad.data();
        }
        c2.useq = up;
    }
    c2.po = PeerOut{};                       // the embedded sweep writes padded rows: no in-kernel peer stores
    c2.want_cov_table = false; c2.cov_table = nullptr; c2.ev_tables = nullptr;
    if (!c.tables_only) {
        pad_rows_kernel<<<grid_for(ctx, (int64_t)n_y), 256, 0, ctx->stream>>>(c.y, yp, T, m, M, batch);
        c2.y = yp; c2.mean = meanp;
        ctx->launches += 1;
    }
    if (c.mean0_chain) {
        pad_rows_kernel<<<grid_for(ctx, (int64_t)n_m0), 256, 0, ctx->stream>>>(c.mean0_chain, m0p, 1, d, D, batch);
        c2.mean0_chain = m0p;
        ctx->launches += 1;
    }
    c2.cov = want_cov ? tab : nullptr;
    c2.flags = c.flags | (want_cov ? (unsigned)RXG_COV_SHARED_OUT : 0u);
    int rc = lgssm_dispatch(ctx, c2);
    if (rc != RXG_OK) return rc;
    if (!c.tables_only) {
        unpad_rows_kernel<<<grid_for(ctx, (int64_t)T * d * batch), 256, 0, ctx->stream>>>(meanp, c.mean, T, d, D, batch);
        ctx->launches += 1;
    }
    if (want_cov) {
        const int64_t rows = (int64_t)T * d * d;
        if (cov_shared) subblock_cov_kernel<<<dim3((unsigned)rows, 1), 32, 0, ctx->stream>>>(tab, c.cov, T, d, D, 0);
        else {
            const unsigned gy = (unsigned)((batch + 4095) / 4096 > 16 ? 16 : (batch + 4095) / 4096);
            subblock_cov_kernel<<<dim3((unsigned)rows, gy), 256, 0, ctx->stream>>>(tab, c.cov, T, d, D, batch);
        }
        ctx->launches += 1;
    }
    if (c.nle && !c.tables_only && M > m) {
        // each dummy observation contributes exactly 1/2 log 2 pi per step
        const int nobs = c.n_observed >= 0 ? c.n_observed : T;        // dummy observations exist only at observed steps
        add_const_kernel<<<(unsigned)((batch + 255) / 256), 256, 0, ctx->stream>>>(c.nle, batch,
                                                                                   (float)(-(double)(M - m) * nobs * 0.91893853320467274178));
        ctx->launches += 1;
    }
    c.fused_peer_stores = false;
    return check_cuda(ctx, cudaGetLastError(), "embedding kernels");
}

}  // namespace

int lgssm_generic_chain(rxg_ctx* ctx, const LgssmCall& c);   // rxg_lgssm_generic.cu

bool lgssm_supported(int d, int m) { return d >= 1 && m >= 1 && d <= 64 && m <= 64; }
bool lgssm_native_small(int d, int m) { return small_native(d, m); }

int lgssm_dispatch(rxg_ctx* ctx, LgssmCall& c) {
    if (!lgssm_supported(c.d, c.m))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm: d and m must be in 1..64 (got d=%d, m=%d)", c.d, c.m);
    if (small_native(c.d, c.m)) return lgssm_dispatch_native(ctx, c);
    int De = 0, Me = 0;
    const bool emb_small = embedding_shape(c.d, c.m, &De, &Me) && small_native(De, Me);
    if (c.tmask && !emb_small) {
        // the large-state gain kernels have no missing-data variant: expand the shared pattern and take the generic kernel
        if (!c.cov || (c.flags & RXG_COV_SHARED_OUT))
            return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm (d=%d): a shared mask on the large-state family needs the per-chain covariance output", c.d);
        uint8_t* mk = (uint8_t*)aux(ctx, 1, (size_t)c.T * c.batch);
        if (!mk) return RXG_ERR_CUDA;
        expand_mask_kernel<<<grid_for(ctx, (int64_t)c.T * c.batch), 256, 0, ctx->stream>>>(c.tmask, mk, c.T, c.batch);
        ctx->launches += 1;
        LgssmCall c2 = c;
        c2.tmask = nullptr; c2.ymask = mk;
        c.fused_peer_stores = false;
        return lgssm_generic_chain(ctx, c2);
    }
    const bool per_chain = (c.flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN)) != 0 || c.ymask != nullptr;
    if (per_chain) {
        if (c.tables_only) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: tables-only call on the per-chain path");
        c.fused_peer_stores = false;
        return lgssm_generic_chain(ctx, c);
    }
    if (lgssm_large_supported(c.d, c.m)) {
        if (c.useq) return large_with_offset(ctx, c);
        if (c.u) {
            bool nz = false;
            for (int i = 0; i < c.d; ++i) nz |= (c.u[i] != 0.f);
            if (nz) return large_with_offset(ctx, c);
            LgssmCall c2 = c;
            c2.u = nullptr;
            int rc = lgssm_large_dispatch(ctx, c2);
            c.fused_peer_stores = c2.fused_peer_stores;
            return rc;
        }
        return lgssm_large_dispatch(ctx, c);
    }
    int D = 0, M = 0;
    if (!embedding_shape(c.d, c.m, &D, &M))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm: no kernel family contains (d=%d, m=%d)", c.d, c.m);
    return embedded(ctx, c, D, M);
}

}  // namespace rxg
