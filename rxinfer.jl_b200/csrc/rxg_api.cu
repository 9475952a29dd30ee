// C ABI of librxgauss: context, error handling, workspace, the whole-chain LGSSM entry points
// (device- and host-pointer variants) and the NCCL all-gather of posterior marginals.
// See include/rxgauss.h for the contract and the reference interfaces each entry replaces.
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <immintrin.h>
#include <sched.h>

#include <map>
#include <mutex>
#include <thread>
#include <vector>

#include "rxg_internal.h"

namespace rxg {

int fail(rxg_ctx* ctx, int code, const char* fmt, ...) {
    if (ctx) {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof(buf), fmt, ap);
        va_end(ap);
        ctx->err = buf;
    }
    return code;
}

int check_cuda(rxg_ctx* ctx, cudaError_t e, const char* what) {
    if (e == cudaSuccess) return RXG_OK;
    return fail(ctx, RXG_ERR_CUDA, "CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
}

static void* grow(rxg_ctx* ctx, void** buf, size_t* have, size_t want) {
    if (*have >= want && *buf) return *buf;
    if (*buf) {
        // the stream may still be using the old buffer
        cudaStreamSynchronize(ctx->stream);
        cudaFree(*buf);
        *buf = nullptr;
        *have = 0;
    }
    size_t sz = (want + ((size_t)1 << 20) - 1) >> 20 << 20;
    cudaError_t e = cudaMalloc(buf, sz);
    if (e != cudaSuccess) {
        check_cuda(ctx, e, "cudaMalloc(workspace)");
        *buf = nullptr;
        return nullptr;
    }
    *have = sz;
    return *buf;
}
int* bad_flag(rxg_ctx* ctx) {
    if (!ctx->d_bad) {
        if (cudaMalloc(&ctx->d_bad, 4) != cudaSuccess || cudaMallocHost(&ctx->h_bad, 4) != cudaSuccess) {
            check_cuda(ctx, cudaGetLastError(), "bad_flag alloc");
            return nullptr;
        }
        *ctx->h_bad = 0;
        cudaMemset(ctx->d_bad, 0, 4);
    }
    return ctx->d_bad;
}
// a kernel, not cudaMemsetAsync: a host-issued device memset can serialise behind another stream's RUNNING kernel (the
// spinning barrier of a peer rank that lives in the same process), a kernel launch on this stream cannot
__global__ void clear_flag_kernel(int* f) { *f = 0; }
int begin_bad_flag(rxg_ctx* ctx) {
    if (!bad_flag(ctx)) return RXG_ERR_CUDA;
    clear_flag_kernel<<<1, 1, 0, ctx->stream>>>(ctx->d_bad);
    return check_cuda(ctx, cudaGetLastError(), "bad flag reset");
}
static int examine_bad_flag(rxg_ctx* ctx) {      // the stream has been synchronised
    if (!ctx->bad_pending) return RXG_OK;
    ctx->bad_pending = false;
    if (*ctx->h_bad & 2)
        return fail(ctx, RXG_ERR_NCCL, "peer barrier timed out: a rank of the peer group never reached the gather");
    if (*ctx->h_bad != 0)
        return fail(ctx, RXG_ERR_NOT_SPD, "a Cholesky pivot of the model's covariance recursion was not positive "
                                          "(A, B, P, Q, S0 do not define SPD predicted / innovation covariances)");
    return RXG_OK;
}
int end_bad_flag(rxg_ctx* ctx, bool sync_now) {
    if (!ctx->d_bad) return RXG_OK;
    int rc = check_cuda(ctx, cudaMemcpyAsync(ctx->h_bad, ctx->d_bad, 4, cudaMemcpyDeviceToHost, ctx->stream), "bad flag read-back");
    if (rc != RXG_OK) return rc;
    ctx->bad_pending = true;
    if (!sync_now) return RXG_OK;
    rc = check_cuda(ctx, cudaStreamSynchronize(ctx->stream), "cudaStreamSynchronize");
    if (rc != RXG_OK) return rc;
    return examine_bad_flag(ctx);
}
// one missing-data pattern for the whole batch (RXG_MASK_SHARED): a host array [T], staged like the model
int stage_shared_mask(rxg_ctx* ctx, int T, const uint8_t* host_mask, LgssmCall& c) {
    if (ctx->tmask_bytes < (size_t)T) {
        if (ctx->d_tmask) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->d_tmask); ctx->d_tmask = nullptr; ctx->tmask_bytes = 0; }
        RXG_CUDA(ctx, cudaMalloc(&ctx->d_tmask, ((size_t)T + 255) / 256 * 256));
        ctx->tmask_bytes = ((size_t)T + 255) / 256 * 256;
    }
    RXG_CUDA(ctx, cudaMemcpyAsync(ctx->d_tmask, host_mask, (size_t)T, cudaMemcpyHostToDevice, ctx->stream));
    int nobs = 0;
    for (int t = 0; t < T; ++t) nobs += host_mask[t] != 0;
    c.tmask = (const uint8_t*)ctx->d_tmask;
    c.n_observed = nobs;
    return RXG_OK;
}
int stage_inputs(rxg_ctx* ctx, unsigned flags, const float* u, int rows, int d, LgssmCall& c) {
    const unsigned f = flags & (RXG_U_SEQ_SHARED | RXG_U_SEQ_CHAIN);
    c.u = u; c.useq = nullptr; c.useq_host = nullptr; c.useq_chain = false;
    if (!f) return RXG_OK;
    if (f == (RXG_U_SEQ_SHARED | RXG_U_SEQ_CHAIN))
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: RXG_U_SEQ_SHARED and RXG_U_SEQ_CHAIN are exclusive");
    if (!u) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: an RXG_U_SEQ_* flag needs the input sequence u");
    c.u = nullptr;
    if (f == RXG_U_SEQ_CHAIN) {
        if (!(flags & RXG_PTR_DEVICE))
            return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm: a per-chain input sequence (RXG_U_SEQ_CHAIN) takes device pointers");
        c.useq = u; c.useq_chain = true;
        return RXG_OK;
    }
    const size_t bytes = (size_t)rows * d * 4;
    if (!grow(ctx, &ctx->d_useq, &ctx->useq_bytes, bytes)) return RXG_ERR_CUDA;
    // pageable host source: the runtime has read it before the call returns
    RXG_CUDA(ctx, cudaMemcpyAsync(ctx->d_useq, u, bytes, cudaMemcpyHostToDevice, ctx->stream));
    c.useq = (const float*)ctx->d_useq; c.useq_host = u;
    return RXG_OK;
}
void* workspace(rxg_ctx* ctx, size_t bytes) { return grow(ctx, &ctx->ws, &ctx->ws_bytes, bytes); }
void* staging(rxg_ctx* ctx, size_t bytes) { return grow(ctx, &ctx->stage, &ctx->stage_bytes, bytes); }
void* predict_scratch(rxg_ctx* ctx, size_t bytes) { return grow(ctx, &ctx->pred_buf, &ctx->pred_bytes, bytes); }

}  // namespace rxg

using namespace rxg;

static std::mutex g_host_mu;
static std::map<void*, size_t> g_host_mapped;      // interleaved allocations: base -> length

static int numa_node_count() {
    int n = 0;
    for (; n < 64; ++n) {
        char path[96];
        snprintf(path, sizeof(path), "/sys/devices/system/node/node%d", n);
        if (access(path, F_OK) != 0) break;
    }
    return n;
}


extern "C" {

int rxg_version(void) { return RXG_VERSION; }

int rxg_create(rxg_ctx** out, int device, unsigned flags) {
    if (!out) return RXG_ERR_BAD_ARG;
    if (flags != 0) return RXG_ERR_BAD_ARG;      // no creation flags are defined (reserved)
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) return RXG_ERR_NO_DEVICE;   // no CPU fallback, by design
    if (device < 0 || device >= n) return RXG_ERR_BAD_ARG;
    if (cudaSetDevice(device) != cudaSuccess) return RXG_ERR_CUDA;
    rxg_ctx* ctx = new rxg_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete ctx;
        return RXG_ERR_CUDA;
    }
    ctx->own_stream = true;
    // options: defaults, then the RXG_* environment variables (read here and nowhere else)
    ctx->opt[RXG_OPT_HOST_BCAST_MIN_MB] = 64;
    static const struct { int id; const char* env; } kEnv[] = {
        {RXG_OPT_GAIN_SEQ, "RXG_GAIN_SEQ"}, {RXG_OPT_LARGE_SEQ, "RXG_LARGE_SEQ"}, {RXG_OPT_NO_UMMA, "RXG_NO_UMMA"},
        {RXG_OPT_SWEEP_VARIANT, "RXG_SWEEP_VARIANT"}, {RXG_OPT_FORCE_CPT, "RXG_FORCE_CPT"},
        {RXG_OPT_HOST_THREADS, "RXG_HOST_THREADS"}, {RXG_OPT_HOST_COV_D2H, "RXG_HOST_COV_D2H"},
        {RXG_OPT_HOST_BCAST_MIN_MB, "RXG_HOST_BCAST_MIN_MB"}, {RXG_OPT_HOST_SLICES, "RXG_HOST_SLICES"},
        {RXG_OPT_GATHER_MODE, "RXG_GATHER_MODE"}, {RXG_OPT_POLYA_PATH, "RXG_POLYA_PATH"}};
    for (const auto& e : kEnv)
        if (const char* v = getenv(e.env)) ctx->opt[e.id] = atoll(v);
    *out = ctx;
    return RXG_OK;
}

int rxg_set_option(rxg_ctx* ctx, int option, long long value) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (option < 0 || option >= RXG_OPT_COUNT_) return fail(ctx, RXG_ERR_BAD_ARG, "rxg_set_option: unknown option %d", option);
    ctx->opt[option] = value;
    return RXG_OK;
}
int rxg_get_option(const rxg_ctx* ctx, int option, long long* value) {
    if (!ctx || !value || option < 0 || option >= RXG_OPT_COUNT_) return RXG_ERR_BAD_ARG;
    *value = ctx->opt[option];
    return RXG_OK;
}

int rxg_comm_destroy_internal(rxg_ctx* ctx);

int rxg_destroy(rxg_ctx* ctx) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    rxg_comm_destroy_internal(ctx);
    if (ctx->ws) cudaFree(ctx->ws);
    if (ctx->stage) cudaFree(ctx->stage);
    if (ctx->d_bad) cudaFree(ctx->d_bad);
    for (int i = 0; i < 4; ++i) if (ctx->aux_buf[i]) cudaFree(ctx->aux_buf[i]);
    if (ctx->d_tmask) cudaFree(ctx->d_tmask);
    if (ctx->d_useq) cudaFree(ctx->d_useq);
    if (ctx->pred_buf) cudaFree(ctx->pred_buf);
    if (ctx->h_bad) cudaFreeHost(ctx->h_bad);
    for (int i = 0; i < 4; ++i) if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
    if (ctx->s_in) {
        cudaStreamSynchronize(ctx->s_in); cudaStreamSynchronize(ctx->s_out);
        cudaStreamDestroy(ctx->s_in); cudaStreamDestroy(ctx->s_out);
        for (int q = 0; q < 2; ++q) { cudaEventDestroy(ctx->ev_in[q]); cudaEventDestroy(ctx->ev_comp[q]); cudaEventDestroy(ctx->ev_out[q]); }
        cudaEventDestroy(ctx->ev_start);
    }
    if (ctx->h_tab) cudaFreeHost(ctx->h_tab);
    if (ctx->ev_tab) cudaEventDestroy(ctx->ev_tab);
    if (ctx->s_aux) {
        cudaStreamSynchronize(ctx->s_aux);
        cudaStreamDestroy(ctx->s_aux);
        cudaEventDestroy(ctx->ev_aux[0]); cudaEventDestroy(ctx->ev_aux[1]);
    }
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return RXG_OK;
}

const char* rxg_last_error(const rxg_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int rxg_set_stream(rxg_ctx* ctx, void* cuda_stream) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (ctx->own_stream && ctx->stream) {
        cudaStreamSynchronize(ctx->stream);
        cudaStreamDestroy(ctx->stream);
    }
    ctx->stream = (cudaStream_t)cuda_stream;
    ctx->own_stream = false;
    return RXG_OK;
}

int rxg_sync(rxg_ctx* ctx) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return examine_bad_flag(ctx);      // a deferred (RXG_ASYNC) call may have flagged a non-SPD model
}

// Pinned host memory.  On a multi-socket host the pages are INTERLEAVED over the NUMA nodes (mmap + mbind +
// cudaHostRegister): a host-pointer call writes 4 (d + d^2) bytes per (chain, step) into the caller's output, and one
// socket's DRAM write bandwidth (~170 GB/s measured on the 2 x 8562Y+ box) is then the end-to-end limit; interleaving
// lets the host-side covariance broadcast and the PCIe DMA use the memory controllers of every socket.
int rxg_host_alloc(void** out, size_t bytes) {
    if (!out || bytes == 0) return RXG_ERR_BAD_ARG;
    *out = nullptr;
    const int nodes = numa_node_count();
    const char* off = getenv("RXG_HOST_NO_INTERLEAVE");
    if (nodes > 1 && bytes >= ((size_t)64 << 20) && !(off && atoi(off) != 0)) {
        const size_t len = (bytes + 4095) / 4096 * 4096;
        void* p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (p != MAP_FAILED) {
            unsigned long mask = (nodes >= 64) ? ~0UL : ((1UL << nodes) - 1);
            const long rc = syscall(SYS_mbind, p, len, 3 /* MPOL_INTERLEAVE */, &mask, (unsigned long)(nodes + 1), 0U);
            if (rc == 0 && cudaHostRegister(p, len, cudaHostRegisterDefault) == cudaSuccess) {
                std::lock_guard<std::mutex> lk(g_host_mu);
                g_host_mapped[p] = len;
                *out = p;
                return RXG_OK;
            }
            cudaGetLastError();
            munmap(p, len);
        }
    }
    return cudaMallocHost(out, bytes) == cudaSuccess ? RXG_OK : RXG_ERR_CUDA;
}
int rxg_host_free(void* p) {
    if (!p) return RXG_OK;
    size_t len = 0;
    {
        std::lock_guard<std::mutex> lk(g_host_mu);
        auto it = g_host_mapped.find(p);
        if (it != g_host_mapped.end()) { len = it->second; g_host_mapped.erase(it); }
    }
    if (len) {
        cudaHostUnregister(p);
        munmap(p, len);
        return RXG_OK;
    }
    return cudaFreeHost(p) == cudaSuccess ? RXG_OK : RXG_ERR_CUDA;
}

int rxg_supports(int d, int m) { return lgssm_supported(d, m) ? 1 : 0; }

long long rxg_launch_count(const rxg_ctx* ctx) { return ctx ? ctx->launches : -1; }

int rxg_set_profiling(rxg_ctx* ctx, int enabled) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (enabled && !ctx->ev[0]) {
        RXG_CUDA(ctx, cudaSetDevice(ctx->device));
        for (int i = 0; i < 4; ++i) RXG_CUDA(ctx, cudaEventCreate(&ctx->ev[i]));
    }
    ctx->profile = enabled != 0;
    return RXG_OK;
}
int rxg_profile_last_ms(rxg_ctx* ctx, float* main_kernel_ms, float* gain_kernels_ms) {
    if (!ctx || !ctx->ev[0]) return RXG_ERR_BAD_ARG;
    RXG_CUDA(ctx, cudaEventSynchronize(ctx->ev[2]));
    if (main_kernel_ms) RXG_CUDA(ctx, cudaEventElapsedTime(main_kernel_ms, ctx->ev[1], ctx->ev[2]));
    if (gain_kernels_ms) RXG_CUDA(ctx, cudaEventElapsedTime(gain_kernels_ms, ctx->ev[0], ctx->ev[1]));
    return RXG_OK;
}

// ------------------------------------------------------------------------------------------------
// whole-chain LGSSM sweeps
// ------------------------------------------------------------------------------------------------
// Host threads this process may use for the covariance broadcast of host-pointer calls:
// min(affinity, cgroup CPU quota) shared between the ranks of a local job (LOCAL_WORLD_SIZE, read once).
static int host_fill_threads() {
    static const int cached = [] {
    long n = 0;
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof(set), &set) == 0) n = CPU_COUNT(&set);
    if (n < 1) n = (long)std::thread::hardware_concurrency();
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[64]; long per = 0;
        if (fscanf(f, "%63s %ld", q, &per) == 2 && strcmp(q, "max") != 0 && per > 0) {
            const long lim = atol(q) / per;
            if (lim >= 1 && lim < n) n = lim;
        }
        fclose(f);
    }
    if (const char* e = getenv("LOCAL_WORLD_SIZE")) { const int w = atoi(e); if (w > 1) n /= w; }
    if (n > 64) n = 64;        // beyond this the memory controllers, not the cores, are the limit
    return (int)(n < 1 ? 1 : n);
    }();
    return cached;
}
extern "C" int rxg_host_fill_threads(void) { return host_fill_threads(); }

static int lgssm_entry(rxg_ctx* ctx, bool smooth, int d, int m, int T, int64_t batch, const float* A,
                       const float* B, const float* P, const float* Q, const float* m0, const float* S0,
                       const float* u, const float* y, const uint8_t* ymask, float* mean, float* cov, float* nle,
                       int32_t* status, unsigned flags, const PredictArgs* pred = nullptr) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (d < 1 || m < 1 || T < 1 || batch < 1) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: d, m, T, batch must be >= 1");
    if (!A || !B || !P || !Q || !m0 || !S0 || !y || !mean) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: null pointer argument");
    if (!cov && smooth && (flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN)))
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: post_cov is required on the per-chain path (it is the stash)");
    if (!lgssm_supported(d, m))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm: d and m must be in 1..64 (got d=%d, m=%d)", d, m);
    const bool per_chain_model = (flags & RXG_MODEL_PER_CHAIN) != 0;
    // a shared missing-data pattern (RXG_MASK_SHARED) keeps the covariances chain independent: only a per-chain mask
    // rules the de-duplicated output out
    const bool per_chain_mask = ymask && !(flags & RXG_MASK_SHARED);
    if ((flags & RXG_COV_SHARED_OUT) && (per_chain_model || (flags & RXG_PATH_PER_CHAIN) || per_chain_mask))
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: RXG_COV_SHARED_OUT needs the shared-model gain-table path");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));

    LgssmCall c;
    c.d = d; c.m = m; c.T = T; c.batch = batch;
    c.A = A; c.B = B; c.P = P; c.Q = Q; c.m0 = m0; c.S0 = S0; c.u = u;
    c.flags = flags; c.smooth = smooth;
    {
        const int rci = stage_inputs(ctx, flags, u, T + (pred ? pred->H : 0), d, c);
        if (rci != RXG_OK) return rci;
    }
    if ((flags & RXG_MASK_SHARED) && ymask) {
        if (per_chain_model || (flags & RXG_PATH_PER_CHAIN))
            return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: RXG_MASK_SHARED belongs to the shared-model gain-table path");
        int rcm = stage_shared_mask(ctx, T, ymask, c);
        if (rcm != RXG_OK) return rcm;
        ymask = nullptr;
    }

    if (flags & RXG_PTR_DEVICE) {
        if (!cov && (ymask || per_chain_model || (flags & RXG_PATH_PER_CHAIN)))
            return fail(ctx, RXG_ERR_BAD_ARG, "lgssm: cov output required on the per-chain path");
        c.y = y; c.ymask = ymask; c.mean = mean; c.cov = cov; c.nle = nle; c.status = status;
        // predictions without a covariance output: the family's own [T][d][d] table (where it keeps one) feeds the post-pass
        if (pred && !cov) c.want_cov_table = true;
        int rc = begin_bad_flag(ctx);
        if (rc == RXG_OK) rc = lgssm_dispatch(ctx, c);
        if (rc == RXG_OK && pred) rc = lgssm_predict_post(ctx, c, *pred);
        if (rc != RXG_OK) return rc;
        return end_bad_flag(ctx, !(flags & RXG_ASYNC));
    }

    // ---- host-pointer call: stage through device memory.  The batch is cut into slices that are
    // pipelined over three streams (H2D of slice s+1 | sweep of slice s | D2H of slice s-1): PCIe is
    // full duplex, so the 4(m)-byte/step upload hides behind the 4(d + d^2)-byte/step download.
    // Batch is the innermost axis, so a slice is a pitched 2-D region of every host array.
    if (per_chain_model)
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm: per-chain model arrays must be device pointers");
    // Shared model, per-chain covariances requested into a HOST buffer: they do not depend on the chain, so the device
    // produces the [T][d][d] table once, that table crosses PCIe (T d^2 floats), and the per-chain copies are
    // materialised by host threads while the means are still in flight -- same bytes in the caller's buffer, 4 d^2 of
    // the 4 (d + d^2) bytes per (chain, step) less PCIe traffic.  RXG_HOST_COV_D2H=1 forces the full device->host copy;
    // with fewer than 6 host threads per rank the PCIe copy wins and is kept.
    bool host_bcast = cov && !(flags & RXG_COV_SHARED_OUT) && !ymask && !(flags & RXG_PATH_PER_CHAIN);
    if (ctx->opt[RXG_OPT_HOST_COV_D2H] != 0) host_bcast = false;
    const size_t bcast_min_mb = (size_t)ctx->opt[RXG_OPT_HOST_BCAST_MIN_MB];   // below this the hand-off is not worth it
    if ((size_t)T * d * d * (size_t)batch * 4 < (bcast_min_mb << 20)) host_bcast = false;
    const int fill_threads = !host_bcast ? 0 : (ctx->opt[RXG_OPT_HOST_THREADS] > 0 ? (int)ctx->opt[RXG_OPT_HOST_THREADS] : host_fill_threads());
    if (fill_threads < 4) host_bcast = false;
    if (host_bcast) c.flags |= RXG_COV_SHARED_OUT;
    const bool cov_shared = (c.flags & RXG_COV_SHARED_OUT) != 0;
    const bool need_cov_dev = cov || ymask || (flags & RXG_PATH_PER_CHAIN);
    int ns = 1;
    if (batch >= 16384) ns = (int)((batch + 8191) / 8192);
    if (ns > 64) ns = 64;
    if (ctx->opt[RXG_OPT_HOST_SLICES] >= 1) ns = (int)ctx->opt[RXG_OPT_HOST_SLICES];
    const int64_t bs = ((batch + ns - 1) / ns + 3) / 4 * 4;          // slice width, multiple of 4 chains
    ns = (int)((batch + bs - 1) / bs);
    const int nbuf = ns > 1 ? 2 : 1;
    const size_t n_y = (size_t)T * m * bs, n_mean = (size_t)T * d * bs;
    const size_t n_cov = need_cov_dev ? (cov_shared ? (size_t)T * d * d : (size_t)T * d * d * bs) : 0;
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
    size_t o_y[2], o_mean[2], o_cov[2], o_mask[2], o_nle[2], o_st[2];
    for (int q = 0; q < nbuf; ++q) {
        o_y[q] = carve(n_y * 4); o_mean[q] = carve(n_mean * 4); o_cov[q] = carve(n_cov * 4);
        o_mask[q] = carve(ymask ? (size_t)T * bs : 0);
        o_nle[q] = carve(nle ? (size_t)bs * 4 : 0); o_st[q] = carve(status ? (size_t)bs * 4 : 0);
    }
    char* base = (char*)staging(ctx, off);
    if (!base) return RXG_ERR_CUDA;
    if (ns > 1 && !ctx->s_in) {
        RXG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking));
        RXG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking));
        for (int q = 0; q < 2; ++q) {
            RXG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_in[q], cudaEventDisableTiming));
            RXG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_comp[q], cudaEventDisableTiming));
            RXG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_out[q], cudaEventDisableTiming));
        }
        RXG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_start, cudaEventDisableTiming));
    }
    {
        int rcb = begin_bad_flag(ctx);
        if (rcb != RXG_OK) return rcb;
    }
    cudaStream_t s_in = ns > 1 ? ctx->s_in : ctx->stream, s_out = ns > 1 ? ctx->s_out : ctx->stream;
    if (ns > 1) {   // the side streams start after whatever the caller queued on the ctx stream
        RXG_CUDA(ctx, cudaEventRecord(ctx->ev_start, ctx->stream));
        RXG_CUDA(ctx, cudaStreamWaitEvent(s_in, ctx->ev_start, 0));
        RXG_CUDA(ctx, cudaStreamWaitEvent(s_out, ctx->ev_start, 0));
    }
    if (host_bcast) {
        // The covariance table depends on the model only: compute it (gain tables, no sweep) and fetch it BEFORE the first
        // observation slice is uploaded, so that the host-side broadcast can start right away.
        if (ctx->h_tab_bytes < (size_t)T * d * d * 4) {
            if (ctx->h_tab) cudaFreeHost(ctx->h_tab);
            ctx->h_tab = nullptr; ctx->h_tab_bytes = 0;
            RXG_CUDA(ctx, cudaMallocHost(&ctx->h_tab, (size_t)T * d * d * 4));
            ctx->h_tab_bytes = (size_t)T * d * d * 4;
        }
        if (!ctx->ev_tab) RXG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->ev_tab, cudaEventDisableTiming));
        LgssmCall c0 = c;
        c0.batch = bs; c0.tables_only = true;
        c0.y = nullptr; c0.mean = nullptr; c0.nle = nullptr; c0.status = nullptr; c0.ymask = nullptr;
        c0.cov = (float*)(base + o_cov[0]);
        int rc0 = lgssm_dispatch(ctx, c0);
        if (rc0 != RXG_OK) return rc0;
        RXG_CUDA(ctx, cudaMemcpyAsync(ctx->h_tab, c0.cov, (size_t)T * d * d * 4, cudaMemcpyDeviceToHost, ctx->stream));
        RXG_CUDA(ctx, cudaEventRecord(ctx->ev_tab, ctx->stream));
    }
    const size_t hp = (size_t)batch * 4;       // host pitch of every fp32 array (bytes)
    for (int sidx = 0; sidx < ns; ++sidx) {
        const int q = sidx & (nbuf - 1);
        const int64_t b0 = (int64_t)sidx * bs;
        const int64_t nb = (b0 + bs <= batch) ? bs : (batch - b0);
        const size_t dp = (size_t)nb * 4;      // device pitch = slice width
        float* d_y = (float*)(base + o_y[q]);
        c.batch = nb;
        c.y = d_y;
        c.mean = (float*)(base + o_mean[q]);
        c.cov = n_cov ? (float*)(base + o_cov[q]) : nullptr;
        c.ymask = ymask ? (const uint8_t*)(base + o_mask[q]) : nullptr;
        c.nle = nle ? (float*)(base + o_nle[q]) : nullptr;
        c.status = status ? (int32_t*)(base + o_st[q]) : nullptr;
        // H2D (buffer q was last read by the sweep of slice sidx-2)
        if (ns > 1 && sidx >= 2) RXG_CUDA(ctx, cudaStreamWaitEvent(s_in, ctx->ev_comp[q], 0));
        RXG_CUDA(ctx, cudaMemcpy2DAsync(d_y, dp, y + b0, hp, dp, (size_t)T * m, cudaMemcpyHostToDevice, s_in));
        if (ymask)
            RXG_CUDA(ctx, cudaMemcpy2DAsync((void*)c.ymask, (size_t)nb, ymask + b0, (size_t)batch, (size_t)nb, (size_t)T,
                                            cudaMemcpyHostToDevice, s_in));
        if (ns > 1) {
            RXG_CUDA(ctx, cudaEventRecord(ctx->ev_in[q], s_in));
            RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_in[q], 0));
            if (sidx >= 2) RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_out[q], 0));   // outputs of sidx-2 drained
        }
        int rc = lgssm_dispatch(ctx, c);
        if (rc != RXG_OK) return rc;
        if (ns > 1) {
            RXG_CUDA(ctx, cudaEventRecord(ctx->ev_comp[q], ctx->stream));
            RXG_CUDA(ctx, cudaStreamWaitEvent(s_out, ctx->ev_comp[q], 0));
        }
        // D2H
        RXG_CUDA(ctx, cudaMemcpy2DAsync(mean + b0, hp, c.mean, dp, dp, (size_t)T * d, cudaMemcpyDeviceToHost, s_out));
        if (cov) {
            if (host_bcast) {
                // nothing to copy per slice: the table was fetched before the first slice, the host threads fill `cov`
            } else if (cov_shared)
                RXG_CUDA(ctx, cudaMemcpyAsync(cov, c.cov, (size_t)T * d * d * 4, cudaMemcpyDeviceToHost, s_out));
            else
                RXG_CUDA(ctx, cudaMemcpy2DAsync(cov + b0, hp, c.cov, dp, dp, (size_t)T * d * d, cudaMemcpyDeviceToHost, s_out));
        }
        if (nle) RXG_CUDA(ctx, cudaMemcpyAsync(nle + b0, c.nle, (size_t)nb * 4, cudaMemcpyDeviceToHost, s_out));
        if (status) RXG_CUDA(ctx, cudaMemcpyAsync(status + b0, c.status, (size_t)nb * 4, cudaMemcpyDeviceToHost, s_out));
        if (ns > 1) RXG_CUDA(ctx, cudaEventRecord(ctx->ev_out[q], s_out));
    }
    if (ns > 1)      // completion of the call == completion of the ctx stream
        for (int q = 0; q < nbuf; ++q) RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_out[q], 0));
    if (host_bcast) {
        // everything above is enqueued; broadcast the covariances on the host while the slices stream through the GPU
        RXG_CUDA(ctx, cudaEventSynchronize(ctx->ev_tab));
        host_broadcast_cov(cov, (const float*)ctx->h_tab, (int64_t)T * d * d, batch, fill_threads);
    }
    return end_bad_flag(ctx, !(flags & RXG_ASYNC));
}

int rxg_lgssm_smooth_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch, const float* A, const float* B,
                         const float* P, const float* Q, const float* m0, const float* S0, const float* u,
                         const float* y, const uint8_t* ymask, float* post_mean, float* post_cov,
                         float* neg_log_evidence, int32_t* status, unsigned flags) {
    return lgssm_entry(ctx, true, d, m, T, batch, A, B, P, Q, m0, S0, u, y, ymask, post_mean, post_cov,
                       neg_log_evidence, status, flags);
}

int rxg_lgssm_filter_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch, const float* A, const float* B,
                         const float* P, const float* Q, const float* m0, const float* S0, const float* u,
                         const float* y, const uint8_t* ymask, float* filt_mean, float* filt_cov,
                         float* neg_log_evidence, int32_t* status, unsigned flags) {
    return lgssm_entry(ctx, false, d, m, T, batch, A, B, P, Q, m0, S0, u, y, ymask, filt_mean, filt_cov,
                       neg_log_evidence, status, flags);
}

// The smoothing sweep, unchanged (same dispatch, same outputs), followed by the prediction post-pass of rxg_predict.cu.
int rxg_lgssm_smooth_predict_f32(rxg_ctx* ctx, int d, int m, int T, int H, int64_t batch, const float* A, const float* B,
                                 const float* P, const float* Q, const float* m0, const float* S0, const float* u,
                                 const float* y, const uint8_t* ymask, float* post_mean, float* post_cov,
                                 float* neg_log_evidence, float* pred_mean, float* pred_cov, float* fc_mean, float* fc_cov,
                                 int32_t* status, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_smooth_predict takes device pointers (set RXG_PTR_DEVICE)");
    if (H < 0) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_predict: the horizon H must be >= 0 (got %d)", H);
    if (!pred_mean) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_smooth_predict: pred_mean is required");
    // without post_cov the chain-independent route reads the family's own covariance table, which only the register-resident
    // families keep: refuse the other shapes before anything runs
    const bool per_chain_route = (flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN)) || (ymask && !(flags & RXG_MASK_SHARED));
    if (!post_cov && !per_chain_route && !lgssm_native_small(d, m))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_smooth_predict (d=%d, m=%d): this shape keeps no covariance table of its "
                                              "own, pass post_cov", d, m);
    const PredictArgs pa = {H, pred_mean, pred_cov, fc_mean, fc_cov};
    return lgssm_entry(ctx, true, d, m, T, batch, A, B, P, Q, m0, S0, u, y, ymask, post_mean, post_cov,
                       neg_log_evidence, status, flags, &pa);
}

// Streaming engine, one time-chunk.  The reference's streaming executor re-triggers a one-step graph per
// datum and carries q(x_t) into the next step's prior through @autoupdates; here a chunk of Tc data is
// one fused filtering sweep, and the carry is explicit: per-chain means (device) + the chain-independent
// covariance (host, d x d) in, the same pair for the last step of the chunk out.
int rxg_lgssm_filter_chunk_f32(rxg_ctx* ctx, int d, int m, int T, int64_t batch, const float* A, const float* B,
                               const float* P, const float* Q, const float* u, const float* prev_mean,
                               float* carry_cov, const float* y, float* filt_mean, float* filt_cov,
                               float* neg_log_evidence, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_filter_chunk takes device pointers");
    if (flags & (RXG_MODEL_PER_CHAIN | RXG_PATH_PER_CHAIN))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_filter_chunk: shared-model gain-table path only");
    if (d < 1 || m < 1 || T < 1 || batch < 1) return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_filter_chunk: d, m, T, batch must be >= 1");
    if (!A || !B || !P || !Q || !prev_mean || !carry_cov || !y || !filt_mean || !filt_cov)
        return fail(ctx, RXG_ERR_BAD_ARG, "lgssm_filter_chunk: null pointer argument");
    if (!lgssm_supported(d, m))
        return fail(ctx, RXG_ERR_UNSUPPORTED, "lgssm_filter_chunk: (d=%d, m=%d) is outside the compiled kernel families", d, m);
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::vector<float> zero((size_t)d, 0.f);
    int rc0 = RXG_OK;
    LgssmCall c;
    c.d = d; c.m = m; c.T = T; c.batch = batch;
    c.A = A; c.B = B; c.P = P; c.Q = Q; c.m0 = zero.data(); c.S0 = carry_cov;
    rc0 = stage_inputs(ctx, flags, u, T, d, c);
    if (rc0 != RXG_OK) return rc0;
    c.mean0_chain = prev_mean;
    c.y = y; c.ymask = nullptr; c.mean = filt_mean; c.cov = filt_cov; c.nle = neg_log_evidence; c.status = nullptr;
    c.flags = (flags | RXG_TRANSITION_FIRST) & ~(unsigned)RXG_ASYNC;
    c.smooth = false;
    int rc = begin_bad_flag(ctx);
    if (rc == RXG_OK) rc = lgssm_dispatch(ctx, c);
    if (rc != RXG_OK) return rc;
    // carry out: the filtered covariance of the last step (chain independent)
    const size_t dd = (size_t)d * d;
    if (flags & RXG_COV_SHARED_OUT)
        RXG_CUDA(ctx, cudaMemcpyAsync(carry_cov, filt_cov + (size_t)(T - 1) * dd, dd * 4, cudaMemcpyDeviceToHost, ctx->stream));
    else
        RXG_CUDA(ctx, cudaMemcpy2DAsync(carry_cov, 4, filt_cov + (size_t)(T - 1) * dd * batch, (size_t)batch * 4, 4, dd,
                                        cudaMemcpyDeviceToHost, ctx->stream));
    return end_bad_flag(ctx, true);      // carry_cov is a host output: always synchronous
}

// ------------------------------------------------------------------------------------------------
// NCCL (resolved at run time so that the library loads on hosts without NCCL)
// ------------------------------------------------------------------------------------------------
typedef struct { char internal[128]; } nccl_uid_t;
typedef int (*fn_get_uid)(nccl_uid_t*);
typedef int (*fn_comm_init)(void**, int, nccl_uid_t, int);
typedef int (*fn_comm_destroy)(void*);
typedef int (*fn_allgather)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef const char* (*fn_errstr)(int);
typedef int (*fn_group)(void);

static void* g_nccl = nullptr;
static fn_get_uid p_get_uid;
static fn_comm_init p_comm_init;
static fn_comm_destroy p_comm_destroy;
static fn_allgather p_allgather;
static fn_errstr p_errstr;
static fn_group p_group_start, p_group_end;

static int nccl_load(rxg_ctx* ctx) {
    if (g_nccl) return RXG_OK;
    const char* names[] = {"libnccl.so.2", "libnccl.so", nullptr};
    for (int i = 0; names[i] && !g_nccl; ++i) g_nccl = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
    if (!g_nccl) return fail(ctx, RXG_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
    p_get_uid = (fn_get_uid)dlsym(g_nccl, "ncclGetUniqueId");
    p_comm_init = (fn_comm_init)dlsym(g_nccl, "ncclCommInitRank");
    p_comm_destroy = (fn_comm_destroy)dlsym(g_nccl, "ncclCommDestroy");
    p_allgather = (fn_allgather)dlsym(g_nccl, "ncclAllGather");
    p_errstr = (fn_errstr)dlsym(g_nccl, "ncclGetErrorString");
    p_group_start = (fn_group)dlsym(g_nccl, "ncclGroupStart");
    p_group_end = (fn_group)dlsym(g_nccl, "ncclGroupEnd");
    if (!p_get_uid || !p_comm_init || !p_comm_destroy || !p_allgather || !p_group_start || !p_group_end) {
        g_nccl = nullptr;
        return fail(ctx, RXG_ERR_NCCL, "libnccl is missing required symbols");
    }
    return RXG_OK;
}

int rxg_comm_unique_id(void* id128) {
    if (!id128) return RXG_ERR_BAD_ARG;
    int rc = nccl_load(nullptr);
    if (rc != RXG_OK) return rc;
    nccl_uid_t uid;
    if (p_get_uid(&uid) != 0) return RXG_ERR_NCCL;
    memcpy(id128, &uid, sizeof(uid));
    return RXG_OK;
}

int rxg_comm_init(rxg_ctx* ctx, int nranks, int rank, const void* id128) {
    if (!ctx || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return RXG_ERR_BAD_ARG;
    int rc = nccl_load(ctx);
    if (rc != RXG_OK) return rc;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    nccl_uid_t uid;
    memcpy(&uid, id128, sizeof(uid));
    int r = p_comm_init(&ctx->comm, nranks, uid, rank);
    if (r != 0) return fail(ctx, RXG_ERR_NCCL, "ncclCommInitRank failed: %s", p_errstr ? p_errstr(r) : "?");
    ctx->nranks = nranks;
    ctx->rank = rank;
    return RXG_OK;
}

int rxg_comm_destroy_internal(rxg_ctx* ctx) {
    if (ctx->comm && p_comm_destroy) p_comm_destroy(ctx->comm);
    ctx->comm = nullptr;
    return RXG_OK;
}

}  // extern "C"

// Diagnostic: a pure streaming kernel with a chosen read : write mix (nr input rows summed, the sum stored into nw
// output rows), float4 per thread, grid-stride over a persistent grid.  It has no dependent chain and no tables, i.e. it
// shows what HBM delivers for the sweep's traffic mix (29 % reads / 71 % writes ~ nr = 2, nw = 5).
__global__ void __launch_bounds__(256) stream_mix_kernel(const float4* __restrict__ src, float4* __restrict__ dst, int64_t n4,
                                                         int nr, int nw) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r = 0; r < nr; ++r) { const float4 v = __ldg(src + (int64_t)r * n4 + i); a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
        for (int w = 0; w < nw; ++w) dst[(int64_t)w * n4 + i] = a;
    }
}

extern "C" {

int rxg_selftest_stream_f32(rxg_ctx* ctx, int64_t n, int n_read, int n_write, const float* src, float* dst, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE) || (!src && n_read > 0) || (!dst && n_write > 0) || n < 4 || (n & 3) || n_read < 0 || n_write < 0)
        return fail(ctx, RXG_ERR_BAD_ARG, "selftest_stream: device pointers, n a positive multiple of 4");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    stream_mix_kernel<<<ctx->sm_count * 16, 256, 0, ctx->stream>>>((const float4*)src, (float4*)dst, n / 4, n_read, n_write);
    ctx->launches += 1;
    RXG_CUDA(ctx, cudaGetLastError());
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

int rxg_allgather_posteriors(rxg_ctx* ctx, int d, int T, int64_t batch_local, const float* post_mean,
                             const float* post_cov, float* gathered_mean, float* gathered_cov, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!(flags & RXG_PTR_DEVICE)) return fail(ctx, RXG_ERR_UNSUPPORTED, "allgather takes device pointers");
    if (!ctx->comm) return fail(ctx, RXG_ERR_NCCL, "allgather: rxg_comm_init has not been called");
    if (d < 1 || T < 1 || batch_local < 1 || !post_mean || !gathered_mean || (post_cov && !gathered_cov))
        return fail(ctx, RXG_ERR_BAD_ARG, "allgather: bad argument");
    const size_t n_mean = (size_t)T * d * batch_local, n_cov = n_mean * d;
    const int nccl_float = 7;
    const bool replicate = post_cov && (flags & RXG_COV_REPLICATE);
    if ((flags & RXG_COV_SHARED_OUT) && post_cov && !replicate)
        return fail(ctx, RXG_ERR_BAD_ARG, "allgather: a [T][d][d] covariance table can only be replicated (RXG_COV_REPLICATE)");
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (replicate) {
        // local broadcast fill on a side stream, concurrent with the NVLink gather of the means
        int rca = ensure_aux_stream(ctx);
        if (rca != RXG_OK) return rca;
        RXG_CUDA(ctx, cudaEventRecord(ctx->ev_aux[0], ctx->stream));
        RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->s_aux, ctx->ev_aux[0], 0));
        rca = launch_replicate_cov(ctx, ctx->s_aux, post_cov, (flags & RXG_COV_SHARED_OUT) ? 1 : batch_local, gathered_cov,
                                   (int64_t)T * d * d, batch_local, ctx->nranks, -1);
        if (rca != RXG_OK) return rca;
        RXG_CUDA(ctx, cudaEventRecord(ctx->ev_aux[1], ctx->s_aux));
    }
    int r = p_group_start();
    if (r == 0) r = p_allgather(post_mean, gathered_mean, n_mean, nccl_float, ctx->comm, ctx->stream);
    if (r == 0 && post_cov && !replicate) r = p_allgather(post_cov, gathered_cov, n_cov, nccl_float, ctx->comm, ctx->stream);
    int r2 = p_group_end();
    if (r == 0) r = r2;
    if (replicate) RXG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_aux[1], 0));
    if (r != 0) return fail(ctx, RXG_ERR_NCCL, "ncclAllGather failed: %s", p_errstr ? p_errstr(r) : "?");
    ctx->launches += (post_cov && !replicate) ? 2 : 1;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

}  // extern "C"
