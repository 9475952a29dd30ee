// Peer-mapped all-gather of posterior marginals over NVLink / NVSwitch -- no NCCL on the data path.
//
// north_star: "the batch dimension shards across the GPUs of one node with one all-gather of posterior marginals at
// the end".  A separate collective after the sweep costs (G-1)/G of the gathered bytes over NVLink AFTER the
// compute has finished.  Here every rank
// maps its peers' gathered buffers (CUDA IPC, NVLink P2P) and
//   * the fused smoothing sweep stores each smoothed mean (and, for the literal full gather, each covariance)
//     straight into all G gathered buffers while the backward recursion is still running (st.global on peer
//     addresses from lgssm_shared_kernel: the transfer overlaps the sweep step by step, there is no second pass
//     over the posteriors and no collective launch at all);
//   * with RXG_COV_REPLICATE (shared model => the covariances are chain independent, SURVEY.md appendix A.1)
//     the covariance slabs of the other ranks are broadcast-filled LOCALLY from the [T][d][d] table by
//     replicate_cov_kernel on a side stream that starts as soon as the gain tables exist, i.e. concurrently with
//     the sweep and its NVLink stores;
//   * kernel families without fused stores (per-chain path, d >= 8, HGF ...) push their finished slab with
//     peer_push_kernel (one read of the local slab, G-1 remote writes);
//   * a device-side barrier (one flag per rank in every rank's buffer, st.release.sys / ld.acquire.sys) closes
//     the call: when it completes on rank g, every rank's stores into g's gathered buffers have been performed.
// [ref: the reference has no distributed path; SURVEY.md section 8(e) defines partitioning and the collective.]
#include <stdio.h>

#include "rxg_internal.h"

using namespace rxg;

namespace rxg {

struct PeerFlags { int* f[RXG_MAX_PEERS]; };

// signal epoch to every rank, then wait until every rank has signalled it to us.  One CTA, one thread per rank.
__global__ void peer_barrier_kernel(PeerFlags pf, int n, int rank, int epoch, int* __restrict__ err) {
    const int g = threadIdx.x;
    if (g >= n) return;
    __threadfence_system();                       // everything this rank's earlier kernels wrote is visible first
    int* remote = pf.f[g] + rank;
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(remote), "r"(epoch) : "memory");
    const int* mine = pf.f[rank] + g;
    const long long t0 = clock64();
    for (;;) {
        int v;
        asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
        if (v - epoch >= 0) break;
        if (clock64() - t0 > 20000000000LL) { atomicOr(err, 2); break; }     // ~10 s: a peer never arrived
        __nanosleep(200);
    }
}

struct PushDst { float* p[RXG_MAX_PEERS]; int n; };

// dst[g][i] = src[i] for every peer g: one coalesced read of the local slab, n remote (NVLink) writes
__global__ void __launch_bounds__(256) peer_push_kernel(const float4* __restrict__ src, PushDst d, int64_t n4,
                                                         const float* __restrict__ src_tail, int64_t n_tail_off, int n_tail) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 v = __ldg(src + i);
        for (int g = 0; g < d.n; ++g) reinterpret_cast<float4*>(d.p[g])[i] = v;
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < n_tail) {
        const float v = src_tail[threadIdx.x];
        for (int g = 0; g < d.n; ++g) d.p[g][n_tail_off + threadIdx.x] = v;
    }
}

// unaligned slabs (odd element counts): same copy, one float per thread
__global__ void __launch_bounds__(256) peer_push_scalar_kernel(const float* __restrict__ src, PushDst d, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = __ldg(src + i);
        for (int g = 0; g < d.n; ++g) d.p[g][i] = v;
    }
}

// Replicates the chain-independent covariances of a shared model into the rank-major gathered layout
// [G][rows][b] without moving them over NVLink: every rank holds the same rows = T*d*d values (the
// gain tables depend on the model only), so the gather of 4 d^2 of the 4 (d + d^2) bytes per
// (chain, step) degenerates into a broadcast fill at HBM write speed.  src_stride = b (value taken
// from the first chain of the local slab) or 1 ([T][d][d] table); slab `skip` is left alone (-1: none).
__global__ void __launch_bounds__(256) replicate_cov_kernel(const float* __restrict__ src, int64_t src_stride,
                                                            float* __restrict__ dst, int64_t rows, int64_t b, int G, int skip) {
    const int64_t row = blockIdx.x;
    const float v = __ldg(src + row * src_stride);
    for (int g = blockIdx.y; g < G; g += gridDim.y) {
        if (g == skip) continue;
        float* out = dst + ((int64_t)g * rows + row) * b;
        const int64_t head = (4 - ((reinterpret_cast<uintptr_t>(out) >> 2) & 3)) & 3;   // floats to 16-byte alignment
        const int64_t h = head < b ? head : b;
        if (threadIdx.x < h) out[threadIdx.x] = v;
        const int64_t n4 = (b - h) / 4;
        float4* o4 = reinterpret_cast<float4*>(out + h);
        const float4 v4 = make_float4(v, v, v, v);
        for (int64_t i = threadIdx.x; i < n4; i += blockDim.x) __stcs(o4 + i, v4);     // streaming: never re-read here
        const int64_t tail = h + 4 * n4;
        if (tail + threadIdx.x < b) out[tail + threadIdx.x] = v;
    }
}

int launch_replicate_cov(rxg_ctx* ctx, cudaStream_t st, const float* src, int64_t src_stride, float* dst, int64_t rows,
                         int64_t b, int G, int skip) {
    const int gy = G < 8 ? G : 8;
    replicate_cov_kernel<<<dim3((unsigned)rows, (unsigned)gy), 256, 0, st>>>(src, src_stride, dst, rows, b, G, skip);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "replicate_cov_kernel");
}

int ensure_aux_stream(rxg_ctx* ctx) {
    if (ctx->s_aux) return RXG_OK;
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);       // lo = numerically greatest = lowest priority
    RXG_CUDA(ctx, cudaStreamCreateWithPriority(&ctx->s_aux, cudaStreamNonBlocking, lo));
    RXG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_aux[0], cudaEventDisableTiming));
    RXG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_aux[1], cudaEventDisableTiming));
    return RXG_OK;
}

static int peer_push(rxg_ctx* ctx, const float* local, float* const* dst, int ndst, int64_t n) {
    if (ndst == 0 || n == 0) return RXG_OK;
    PushDst d = {};
    d.n = ndst;
    bool al = (reinterpret_cast<uintptr_t>(local) & 15) == 0;
    for (int g = 0; g < ndst; ++g) { d.p[g] = dst[g]; al = al && (reinterpret_cast<uintptr_t>(dst[g]) & 15) == 0; }
    const int64_t cap0 = (int64_t)ctx->sm_count * 8;
    if (!al) {
        int64_t blocks = (n + 255) / 256;
        if (blocks > cap0) blocks = cap0;
        peer_push_scalar_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(local, d, n);
        ctx->launches += 1;
        return check_cuda(ctx, cudaGetLastError(), "peer_push_scalar_kernel");
    }
    const int64_t n4 = n / 4;
    const int nt = (int)(n - 4 * n4);
    int64_t blocks = (n4 + 255) / 256;
    const int64_t cap = (int64_t)ctx->sm_count * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    peer_push_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>((const float4*)local, d, n4, local + 4 * n4, 4 * n4, nt);
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "peer_push_kernel");
}

static int peer_barrier(rxg_ctx* ctx) {
    if (ctx->peer_n <= 1) return RXG_OK;
    PeerFlags pf = {};
    for (int g = 0; g < ctx->peer_n; ++g) pf.f[g] = ctx->peer_flags[g];
    ctx->peer_epoch += 1;
    peer_barrier_kernel<<<1, 32, 0, ctx->stream>>>(pf, ctx->peer_n, ctx->peer_rank, (int)ctx->peer_epoch, bad_flag(ctx));
    ctx->launches += 1;
    return check_cuda(ctx, cudaGetLastError(), "peer_barrier_kernel");
}

}  // namespace rxg

extern "C" {

int rxg_device_alloc(rxg_ctx* ctx, size_t bytes, void** dev_ptr) {
    if (!ctx || !dev_ptr || bytes == 0) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    *dev_ptr = nullptr;
    RXG_CUDA(ctx, cudaMalloc(dev_ptr, bytes));
    return RXG_OK;
}
int rxg_device_free(rxg_ctx* ctx, void* dev_ptr) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    RXG_CUDA(ctx, cudaFree(dev_ptr));
    return RXG_OK;
}
int rxg_device_memset(rxg_ctx* ctx, void* dev_ptr, int value, size_t bytes) {
    if (!ctx || !dev_ptr) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    RXG_CUDA(ctx, cudaMemsetAsync(dev_ptr, value, bytes, ctx->stream));
    RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

int rxg_memcpy_h2d(rxg_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes) {
    if (!ctx || (bytes && (!dst_dev || !src_host))) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    RXG_CUDA(ctx, cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}
int rxg_memcpy_d2h(rxg_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes) {
    if (!ctx || (bytes && (!dst_host || !src_dev))) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    RXG_CUDA(ctx, cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

int rxg_peer_export(rxg_ctx* ctx, const void* dev_ptr, void* handle64) {
    if (!ctx || !dev_ptr || !handle64) return RXG_ERR_BAD_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    RXG_CUDA(ctx, cudaIpcGetMemHandle(&h, const_cast<void*>(dev_ptr)));
    memcpy(handle64, &h, 64);
    return RXG_OK;
}
int rxg_peer_open(rxg_ctx* ctx, const void* handle64, void** dev_ptr) {
    if (!ctx || !dev_ptr || !handle64) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    *dev_ptr = nullptr;
    RXG_CUDA(ctx, cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return RXG_OK;
}
int rxg_peer_close(rxg_ctx* ctx, void* dev_ptr) {
    if (!ctx || !dev_ptr) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    RXG_CUDA(ctx, cudaIpcCloseMemHandle(dev_ptr));
    return RXG_OK;
}

int rxg_peer_group(rxg_ctx* ctx, int nranks, int rank, void* const* flag_ptrs) {
    if (!ctx || nranks < 1 || nranks > RXG_MAX_PEERS || rank < 0 || rank >= nranks || (nranks > 1 && !flag_ptrs))
        return ctx ? fail(ctx, RXG_ERR_BAD_ARG, "peer_group: 1 <= nranks <= %d, 0 <= rank < nranks", RXG_MAX_PEERS) : RXG_ERR_BAD_ARG;
    if (nranks > 1) {      // everything the gather calls need later is created now (no allocation inside a gather)
        RXG_CUDA(ctx, cudaSetDevice(ctx->device));
        int rc0 = ensure_aux_stream(ctx);
        if (rc0 != RXG_OK) return rc0;
        if (!bad_flag(ctx)) return RXG_ERR_CUDA;
        // CUDA loads a kernel's module at its FIRST launch (lazy loading), which may wait for running kernels; a rank
        // whose peer is already spinning in the barrier must not hit that inside a gather: load the gather kernels now
        cudaFuncAttributes fa;
        RXG_CUDA(ctx, cudaFuncGetAttributes(&fa, peer_barrier_kernel));
        RXG_CUDA(ctx, cudaFuncGetAttributes(&fa, peer_push_kernel));
        RXG_CUDA(ctx, cudaFuncGetAttributes(&fa, peer_push_scalar_kernel));
        RXG_CUDA(ctx, cudaFuncGetAttributes(&fa, replicate_cov_kernel));
    }
    ctx->peer_n = nranks;
    ctx->peer_rank = rank;
    ctx->peer_epoch = 0;
    for (int g = 0; g < RXG_MAX_PEERS; ++g) ctx->peer_flags[g] = (g < nranks && flag_ptrs) ? (int*)flag_ptrs[g] : nullptr;
    for (int g = 0; g < nranks && nranks > 1; ++g)
        if (!ctx->peer_flags[g]) return fail(ctx, RXG_ERR_BAD_ARG, "peer_group: null flag buffer for rank %d", g);
    return RXG_OK;
}

int rxg_peer_barrier(rxg_ctx* ctx, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (ctx->peer_n < 1) return fail(ctx, RXG_ERR_BAD_ARG, "peer_barrier: rxg_peer_group has not been called");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    int rc = begin_bad_flag(ctx);
    if (rc == RXG_OK) rc = peer_barrier(ctx);
    if (rc != RXG_OK) return rc;
    return end_bad_flag(ctx, !(flags & RXG_ASYNC));
}

int rxg_peer_allgather_f32(rxg_ctx* ctx, int64_t n_local, const float* local, float* const* gathered, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return fail(ctx, RXG_ERR_UNSUPPORTED, "peer_allgather takes device pointers");
    if (ctx->peer_n < 1) return fail(ctx, RXG_ERR_BAD_ARG, "peer_allgather: rxg_peer_group has not been called");
    if (n_local < 1 || !gathered) return fail(ctx, RXG_ERR_BAD_ARG, "peer_allgather: bad argument");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const int G = ctx->peer_n, r = ctx->peer_rank;
    for (int g = 0; g < G; ++g)
        if (!gathered[g]) return fail(ctx, RXG_ERR_BAD_ARG, "peer_allgather: null gathered buffer for rank %d", g);
    float* own = gathered[r] + (int64_t)r * n_local;
    int rc = begin_bad_flag(ctx);
    if (rc != RXG_OK) return rc;
    // one kernel stores the local array into slab r of EVERY buffer, the own one included when `local` lives elsewhere
    // (no cudaMemcpy: a device-to-device copy issued by the host may serialise with a peer's spinning barrier kernel
    // when several ranks share one process)
    const float* src = local ? local : own;
    float* dst[RXG_MAX_PEERS];
    int nd = 0;
    for (int g = 0; g < G; ++g)
        if (g != r || src != own) dst[nd++] = gathered[g] + (int64_t)r * n_local;
    rc = peer_push(ctx, src, dst, nd, n_local);
    if (rc == RXG_OK) rc = peer_barrier(ctx);
    if (rc != RXG_OK) return rc;
    return end_bad_flag(ctx, !(flags & RXG_ASYNC));
}

int rxg_lgssm_smooth_gather_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch_local, const float* A, const float* B,
                                const float* P, const float* Q, const float* m0, const float* S0, const float* u,
                                const float* y, const uint8_t* ymask, float* const* gathered_mean,
                                float* const* gathered_cov, float* neg_log_evidence, int32_t* status, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (flags & (RXG_U_SEQ_SHARED | RXG_U_SEQ_CHAIN))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_smooth_gather: per-step input sequences (RXG_U_SEQ_*) are not supported here");
    if (!(flags & RXG_PTR_DEVICE)) return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_smooth_gather takes device pointers");
    if (ctx->peer_n < 1) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: rxg_peer_group has not been called");
    if (d < 1 || m < 1 || T < 1 || batch_local < 1) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: d, m, T, batch must be >= 1");
    if (!A || !B || !P || !Q || !m0 || !S0 || !y || !gathered_mean) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: null pointer argument");
    if (flags & RXG_COV_SHARED_OUT) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: the gathered covariances are per chain");
    if (!lgssm_supported(d, m)) return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_smooth_gather: (d=%d, m=%d) unsupported", d, m);
    const int G = ctx->peer_n, r = ctx->peer_rank;
    const bool shared_mask = (flags & RXG_MASK_SHARED) && ymask;
    const bool per_chain = (flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN)) != 0 || (ymask != nullptr && !shared_mask);
    if (shared_mask && (flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN)))
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: RXG_MASK_SHARED belongs to the shared-model gain-table path");
    const bool replicate = gathered_cov && (flags & RXG_COV_REPLICATE);
    if (replicate && per_chain)
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: RXG_COV_REPLICATE needs chain-independent covariances (shared model, no mask)");
    if (!gathered_mean[r] || (gathered_cov && !gathered_cov[r])) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: null own buffer");
    for (int g = 0; g < G; ++g)
        if (!gathered_mean[g] || (gathered_cov && !replicate && !gathered_cov[g]))
            return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: null gathered buffer for rank %d", g);
    if (per_chain && !gathered_cov) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_gather: the per-chain path needs the covariance buffers (stash)");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    const int64_t slab_m = (int64_t)T * d * batch_local, slab_c = slab_m * d;

    LgssmCall c;
    c.d = d; c.m = m; c.T = T; c.batch = batch_local;
    c.A = A; c.B = B; c.P = P; c.Q = Q; c.m0 = m0; c.S0 = S0; c.u = u;
    c.y = y; c.ymask = shared_mask ? nullptr : ymask; c.nle = neg_log_evidence; c.status = status;
    if (shared_mask) {
        int rcm = stage_shared_mask(ctx, T, ymask, c);
        if (rcm != RXG_OK) return rcm;
    }
    c.mean = gathered_mean[r] + r * slab_m;
    c.cov = gathered_cov ? gathered_cov[r] + r * slab_c : nullptr;
    c.flags = flags & ~(unsigned)(RXG_COV_REPLICATE | RXG_ASYNC | RXG_MASK_SHARED);
    c.smooth = true;
    float* pm[RXG_MAX_PEERS - 1];
    float* pc[RXG_MAX_PEERS - 1];
    int np = 0;
    for (int g = 0; g < G; ++g)
        if (g != r) {
            pm[np] = gathered_mean[g] + r * slab_m;
            pc[np] = (gathered_cov && !replicate) ? gathered_cov[g] + r * slab_c : nullptr;
            ++np;
        }
    // Fused in-kernel peer stores (default) or push-after-sweep (RXG_OPT_GATHER_MODE = 2, kept for comparison).
    const long long gmode = ctx->opt[RXG_OPT_GATHER_MODE];
    const bool fuse = gmode != 2;
    if (fuse) {
        for (int k = 0; k < np; ++k) { c.po.mean[k] = pm[k]; c.po.cov[k] = pc[k]; }
        c.po.n_mean = np;
        c.po.n_cov = (gathered_cov && !replicate) ? np : 0;
    }
    if (replicate && G > 1) {
        // the kernel family leaves the chain-independent covariance table in its workspace (no allocation here: a
        // device allocation may synchronise with a peer's spinning barrier when several ranks share one process)
        c.want_cov_table = true;
        c.ev_tables = ctx->ev_aux[0];
    }
    int rc = begin_bad_flag(ctx);
    if (rc == RXG_OK) rc = lgssm_dispatch(ctx, c);
    if (rc != RXG_OK) return rc;
    if (G > 1) {
        if (replicate) {
            // local broadcast fill of the other ranks' covariance slabs on the low-priority side stream
            const int64_t rows = (int64_t)T * d * d;
            if (c.cov_table) {      // the table exists as soon as the gain kernels are done (ev_tables): overlaps the whole sweep
                RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->s_aux, ctx->ev_aux[0], 0));
                rc = launch_replicate_cov(ctx, ctx->s_aux, c.cov_table, 1, gathered_cov[r], rows, batch_local, G, r);
            } else {                        // other kernel families: replicate from the finished local slab
                RXG_CUDA(ctx, cudaEventRecord(ctx->ev_aux[0], ctx->stream));
                RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->s_aux, ctx->ev_aux[0], 0));
                rc = launch_replicate_cov(ctx, ctx->s_aux, c.cov, batch_local, gathered_cov[r], rows, batch_local, G, r);
            }
            if (rc != RXG_OK) return rc;
            RXG_CUDA(ctx, cudaEventRecord(ctx->ev_aux[1], ctx->s_aux));
        }
        if (!c.fused_peer_stores) {         // this kernel family has no in-kernel peer stores: push the finished slabs
            rc = peer_push(ctx, c.mean, pm, np, slab_m);
            if (rc == RXG_OK && gathered_cov && !replicate) rc = peer_push(ctx, c.cov, pc, np, slab_c);
            if (rc != RXG_OK) return rc;
        }
        if (replicate) RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_aux[1], 0));
        rc = peer_barrier(ctx);
        if (rc != RXG_OK) return rc;
    }
    return end_bad_flag(ctx, !(flags & RXG_ASYNC));
}

}  // extern "C"
