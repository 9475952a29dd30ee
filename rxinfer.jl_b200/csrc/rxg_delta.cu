// Delta node entries (include/rxgauss.h, "Delta node"): user CUDA functions compiled at run time with NVRTC against
// the embedded rxg_delta.cuh, one module per (source, names, d, m, method, unscented parameters), cached per context.
//
// NVRTC is resolved with dlopen on first use, as NCCL is (rxg_api.cu): linking it statically would add about 120 MB
// to the library, and a dynamic link would tie the library to whichever copy the build found.  The module is loaded
// with the runtime's library API (cudaLibraryLoadData), so the library still links no libcuda.
#include "rxg_internal.h"

#include <ctype.h>
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "rxg_delta.cuh"      // compiled here for the layout of rxgd::Params (and to catch header errors at build time)

extern const char rxg_delta_header_src[];     // rxg_delta.cuh, embedded by build.py
typedef rxgd::Params rxgd_params_t;

struct rxg_delta_model {
    cudaLibrary_t lib = nullptr;
    cudaKernel_t k_smooth = nullptr, k_filter = nullptr;
    int d = 0, m = 0, method = 0;
    bool has_g = false;
};

namespace {

// ------------------------------------------------------------------ NVRTC (the few entry points used, by dlsym)
typedef struct _nvrtcProgram* nvrtcProgram;
typedef int (*fn_create)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*);
typedef int (*fn_compile)(nvrtcProgram, int, const char* const*);
typedef int (*fn_size)(nvrtcProgram, size_t*);
typedef int (*fn_get)(nvrtcProgram, char*);
typedef int (*fn_destroy)(nvrtcProgram*);

struct Nvrtc {
    void* dl = nullptr;
    fn_create create = nullptr;
    fn_compile compile = nullptr;
    fn_size cubin_size = nullptr, log_size = nullptr;
    fn_get cubin = nullptr, log = nullptr;
    fn_destroy destroy = nullptr;
};

std::mutex g_mu;            // guards g_nvrtc, g_ctx
Nvrtc g_nvrtc;

struct CtxState {
    std::string nvrtc_path;       // RXG_NVRTC at rxg_create, or empty (the soname); used only if this ctx loads NVRTC
    std::map<std::string, std::unique_ptr<rxg_delta_model>> cache;
    long long compiles = 0;
};
std::map<const rxg_ctx*, CtxState> g_ctx;

// loads NVRTC once per process: the first call's path wins and later paths (another context's RXG_NVRTC) are ignored;
// false with the reason in `err`
bool nvrtc_load(const std::string& path, std::string& err) {
    if (g_nvrtc.dl) return true;
    const char* name = path.empty() ? "libnvrtc.so.12" : path.c_str();
    void* dl = dlopen(name, RTLD_NOW | RTLD_LOCAL);
    if (!dl) {
        const char* e = dlerror();
        err = std::string("cannot load NVRTC (") + name + "): " + (e ? e : "unknown error") +
              "; install the CUDA 12 runtime compiler or point RXG_NVRTC at libnvrtc.so.12";
        return false;
    }
    Nvrtc n;
    n.dl = dl;
    n.create = (fn_create)dlsym(dl, "nvrtcCreateProgram");
    n.compile = (fn_compile)dlsym(dl, "nvrtcCompileProgram");
    n.cubin_size = (fn_size)dlsym(dl, "nvrtcGetCUBINSize");
    n.cubin = (fn_get)dlsym(dl, "nvrtcGetCUBIN");
    n.log_size = (fn_size)dlsym(dl, "nvrtcGetProgramLogSize");
    n.log = (fn_get)dlsym(dl, "nvrtcGetProgramLog");
    n.destroy = (fn_destroy)dlsym(dl, "nvrtcDestroyProgram");
    if (!n.create || !n.compile || !n.cubin_size || !n.cubin || !n.log_size || !n.log || !n.destroy) {
        dlclose(dl);
        err = std::string(name) + " lacks the NVRTC entry points this library uses";
        return false;
    }
    g_nvrtc = n;
    return true;
}

struct Spec {
    std::string source, f, g;
    int d, m, method;
    double ut[3];
};

int check_spec(const char* source, const char* f_name, const char* g_name, int d, int m, int method, const double* ut,
               Spec& s, std::string& err) {
    if (!source || !f_name || !*f_name) { err = "delta: source and f_name are required"; return RXG_ERR_BAD_ARG; }
    if (d < 1 || d > 8 || m < 1 || m > 8) { err = "delta: d and m must be in 1..8"; return RXG_ERR_BAD_ARG; }
    if (method != RXG_DELTA_LINEARIZATION && method != RXG_DELTA_UNSCENTED) {
        err = "delta: method must be RXG_DELTA_LINEARIZATION or RXG_DELTA_UNSCENTED";
        return RXG_ERR_BAD_ARG;
    }
    s.source = source; s.f = f_name; s.g = g_name ? g_name : "";
    s.d = d; s.m = m; s.method = method;
    // the unscented parameters only shape the Unscented module; ReactiveMP's Unscented() defaults otherwise
    s.ut[0] = 1e-3; s.ut[1] = 2.0; s.ut[2] = 0.0;
    if (ut && method == RXG_DELTA_UNSCENTED) { s.ut[0] = ut[0]; s.ut[1] = ut[1]; s.ut[2] = ut[2]; }
    if (method == RXG_DELTA_UNSCENTED && !(s.ut[0] > 0.0 && s.ut[0] * s.ut[0] * (d + s.ut[2]) > 0.0)) {
        err = "delta: the unscented parameters need alpha > 0 and d + kappa > 0";
        return RXG_ERR_BAD_ARG;
    }
    for (const std::string& n : {s.f, s.g})
        for (char c : n)
            if (!(isalnum((unsigned char)c) || c == '_' || c == ':')) {
                err = "delta: function names must be C++ identifiers";
                return RXG_ERR_BAD_ARG;
            }
    return RXG_OK;
}

std::string key_of(const Spec& s) {
    char buf[160];
    snprintf(buf, sizeof(buf), "|%d|%d|%d|%.17g|%.17g|%.17g|", s.d, s.m, s.method, s.ut[0], s.ut[1], s.ut[2]);
    return s.f + "|" + s.g + buf + s.source;
}

// the embedded header, the user's source and the instantiation tail: what NVRTC compiles
std::string program_text(const Spec& s) {
    char cfg[512];
    snprintf(cfg, sizeof(cfg),
             "struct RxgDeltaConfig {\n"
             "    enum { D = %d, M = %d, METHOD = %d, HAS_G = %d };\n"
             "    static constexpr double ALPHA = %.17g, BETA = %.17g, KAPPA = %.17g;\n",
             s.d, s.m, s.method, s.g.empty() ? 0 : 1, s.ut[0], s.ut[1], s.ut[2]);
    std::string t = std::string(rxg_delta_header_src) + "\n#line 1 \"user_source\"\n" + s.source +
                    "\n#line 1 \"rxg_delta_tail\"\n" + cfg;
    t += "    struct F { template <class S> __device__ static void eval(const S* x, S* z) { " + s.f + "<S>(x, z); } };\n";
    if (s.g.empty())
        t += "    struct G { template <class S> __device__ static void eval(const S*, S*) {} };\n";
    else
        t += "    struct G { template <class S> __device__ static void eval(const S* x, S* y) { " + s.g + "<S>(x, y); } };\n";
    t += "};\n"
         "extern \"C\" __global__ void __launch_bounds__(128) rxg_delta_smooth(rxgd::Params p, int T, long long batch,\n"
         "        const float* y, const unsigned char* ymask, float* post_mean, float* post_cov, float* filt_mean,\n"
         "        float* filt_cov, int* status) {\n"
         "    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;\n"
         "    if (b < batch) rxgd::smooth_chain<RxgDeltaConfig>(p, T, batch, b, y, ymask, post_mean, post_cov, filt_mean,\n"
         "                                                     filt_cov, status);\n"
         "}\n"
         "extern \"C\" __global__ void __launch_bounds__(128) rxg_delta_filter(rxgd::Params p, int T, long long batch,\n"
         "        const float* y, const unsigned char* ymask, float* carry_mean, float* carry_cov, float* carry_tau,\n"
         "        int iters, float* filt_mean, float* filt_cov, float* filt_tau, int* status) {\n"
         "    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;\n"
         "    if (b < batch) rxgd::filter_chain<RxgDeltaConfig>(p, T, batch, b, y, ymask, carry_mean, carry_cov, carry_tau,\n"
         "                                                     iters, filt_mean, filt_cov, filt_tau, status);\n"
         "}\n";
    return t;
}

void copy_log(const std::string& log, char* buf, size_t cap) {
    if (!buf || cap == 0) return;
    const size_t n = log.size() < cap - 1 ? log.size() : cap - 1;
    memcpy(buf, log.data(), n);
    buf[n] = 0;
}

// NVRTC compile for sm_90a: RXG_OK with the CUBIN, RXG_ERR_BAD_ARG with the compiler log, RXG_ERR_UNSUPPORTED without
// NVRTC.  Called with g_mu held.
int compile(const Spec& s, const std::string& nvrtc_path, std::vector<char>& cubin, std::string& log) {
    if (!nvrtc_load(nvrtc_path, log)) return RXG_ERR_UNSUPPORTED;
    const std::string text = program_text(s);
    nvrtcProgram prog = nullptr;
    if (g_nvrtc.create(&prog, text.c_str(), "rxg_delta.cu", 0, nullptr, nullptr) != 0) {
        log = "delta: nvrtcCreateProgram failed";
        return RXG_ERR_UNSUPPORTED;
    }
    const char* opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "--ptxas-options=-v"};
    const int rc = g_nvrtc.compile(prog, 3, opts);
    size_t n = 0;
    g_nvrtc.log_size(prog, &n);
    log.assign(n, '\0');
    if (n) g_nvrtc.log(prog, &log[0]);
    while (!log.empty() && log.back() == '\0') log.pop_back();
    if (rc == 0) {
        g_nvrtc.cubin_size(prog, &n);
        cubin.resize(n);
        g_nvrtc.cubin(prog, cubin.data());
    }
    g_nvrtc.destroy(&prog);
    return rc == 0 ? RXG_OK : RXG_ERR_BAD_ARG;
}

// the model constants every chain shares, packed into the kernels' by-value parameter block
void pack(rxgd_params_t& p, const rxg_delta_model* mo, const float* m0, const float* S0, const float* P, const float* B,
          const float* Q) {
    const int d = mo->d, m = mo->m;
    memset(&p, 0, sizeof(p));
    if (m0) memcpy(p.m0, m0, sizeof(float) * d);
    if (S0) memcpy(p.S0, S0, sizeof(float) * d * d);
    if (P) memcpy(p.P, P, sizeof(float) * d * d);
    if (B) memcpy(p.B, B, sizeof(float) * m * d);
    if (Q) memcpy(p.Q, Q, sizeof(float) * m * m);
}

bool host_spd(const float* a, int n) {
    double inv[64], ld;
    return rxg::host_spd_inv(a, n, inv, &ld);
}

int launch(rxg_ctx* ctx, cudaKernel_t k, int64_t batch, void** args, unsigned flags) {
    const unsigned threads = 128;
    const dim3 grid((unsigned)((batch + threads - 1) / threads));
    RXG_CUDA(ctx, cudaLaunchKernel((const void*)k, grid, dim3(threads), args, 0, ctx->stream));
    ctx->launches++;
    if (!(flags & RXG_ASYNC)) RXG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return RXG_OK;
}

}  // namespace

namespace rxg {
// rxg_create / rxg_destroy (rxg_api.cu): the per-context NVRTC path and module cache
void delta_ctx_init(const rxg_ctx* ctx) {
    std::lock_guard<std::mutex> lk(g_mu);
    const char* p = getenv("RXG_NVRTC");
    g_ctx[ctx].nvrtc_path = p ? p : "";
}
void delta_ctx_release(const rxg_ctx* ctx) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_ctx.find(ctx);
    if (it == g_ctx.end()) return;
    for (auto& kv : it->second.cache)
        if (kv.second->lib) cudaLibraryUnload(kv.second->lib);
    g_ctx.erase(it);
}
}  // namespace rxg

extern "C" {

int rxg_delta_check_source(const char* source, const char* f_name, const char* g_name, int d, int m, int method,
                           const double ut[3], char* log, size_t log_cap) {
    Spec s;
    std::string msg;
    int rc = check_spec(source, f_name, g_name, d, m, method, ut, s, msg);
    if (rc == RXG_OK) {
        std::lock_guard<std::mutex> lk(g_mu);
        std::vector<char> cubin;
        rc = compile(s, "", cubin, msg);
    }
    copy_log(msg, log, log_cap);
    return rc;
}

int rxg_delta_model_create(rxg_ctx* ctx, const char* source, const char* f_name, const char* g_name, int d, int m,
                           int method, const double ut[3], rxg_delta_model** out, char* log, size_t log_cap) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!out) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_model_create: out is null");
    *out = nullptr;
    copy_log("", log, log_cap);
    Spec s;
    std::string msg;
    int rc = check_spec(source, f_name, g_name, d, m, method, ut, s, msg);
    if (rc != RXG_OK) return rxg::fail(ctx, rc, "%s", msg.c_str());
    const std::string key = key_of(s);
    std::lock_guard<std::mutex> lk(g_mu);
    CtxState& cs = g_ctx[ctx];
    auto it = cs.cache.find(key);
    if (it != cs.cache.end()) {
        *out = it->second.get();
        return RXG_OK;
    }
    std::vector<char> cubin;
    rc = compile(s, cs.nvrtc_path, cubin, msg);
    copy_log(msg, log, log_cap);
    if (rc != RXG_OK) return rxg::fail(ctx, rc, "delta_model_create: %s%s", rc == RXG_ERR_BAD_ARG ? "NVRTC: " : "",
                                       msg.c_str());
    cs.compiles++;
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<rxg_delta_model> mo(new rxg_delta_model());
    mo->d = d; mo->m = m; mo->method = method; mo->has_g = !s.g.empty();
    RXG_CUDA(ctx, cudaLibraryLoadData(&mo->lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0));
    if (cudaLibraryGetKernel(&mo->k_smooth, mo->lib, "rxg_delta_smooth") != cudaSuccess ||
        cudaLibraryGetKernel(&mo->k_filter, mo->lib, "rxg_delta_filter") != cudaSuccess) {
        cudaLibraryUnload(mo->lib);
        return rxg::fail(ctx, RXG_ERR_CUDA, "delta_model_create: the compiled module lacks its kernels");
    }
    *out = mo.get();
    cs.cache[key] = std::move(mo);
    return RXG_OK;
}

long long rxg_delta_compile_count(const rxg_ctx* ctx) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_ctx.find(ctx);
    return it == g_ctx.end() ? 0 : it->second.compiles;
}

int rxg_delta_smooth_f32(rxg_ctx* ctx, const rxg_delta_model* model, int T, int64_t batch, const float* m0,
                         const float* S0, const float* P, const float* B, const float* Q, const float* y,
                         const uint8_t* ymask, float* post_mean, float* post_cov, float* filt_mean, float* filt_cov,
                         int32_t* status, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!model) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_smooth: null model");
    if (flags & ~(unsigned)(RXG_PTR_DEVICE | RXG_ASYNC)) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_smooth: unknown flags");
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "delta_smooth takes device pointers");
    if (T < 1 || batch < 1) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_smooth: T and batch must be >= 1");
    if (!m0 || !S0 || !P || !Q || !y || !post_mean || !post_cov || (!model->has_g && !B) || (!filt_mean != !filt_cov))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_smooth: null pointer argument (B may be null only with g; "
                                               "filt_mean and filt_cov go together)");
    if (!host_spd(S0, model->d) || !host_spd(Q, model->m))
        return rxg::fail(ctx, RXG_ERR_NOT_SPD, "delta_smooth: S0 and Q must be symmetric positive definite");
    rxgd_params_t p;
    pack(p, model, m0, S0, P, model->has_g ? nullptr : B, Q);
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    long long nb = batch;
    void* args[] = {&p, &T, &nb, &y, &ymask, &post_mean, &post_cov, &filt_mean, &filt_cov, &status};
    return launch(ctx, model->k_smooth, batch, args, flags);
}

int rxg_delta_filter_chunk_f32(rxg_ctx* ctx, const rxg_delta_model* model, int T, int64_t batch, const float* P,
                               const float* B, const float* Q, int iters, const float* y, const uint8_t* ymask,
                               float* carry_mean, float* carry_cov, float* carry_tau, float* filt_mean, float* filt_cov,
                               float* filt_tau, int32_t* status, unsigned flags) {
    if (!ctx) return RXG_ERR_BAD_ARG;
    if (!model) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_filter_chunk: null model");
    if (flags & ~(unsigned)(RXG_PTR_DEVICE | RXG_ASYNC))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_filter_chunk: unknown flags");
    if (!(flags & RXG_PTR_DEVICE)) return rxg::fail(ctx, RXG_ERR_UNSUPPORTED, "delta_filter_chunk takes device pointers");
    if (T < 1 || batch < 1) return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_filter_chunk: T and batch must be >= 1");
    if (!P || !y || !carry_mean || !carry_cov || (!filt_mean != !filt_cov))
        return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_filter_chunk: null pointer argument (filt_mean and filt_cov go "
                                               "together)");
    if (carry_tau) {
        if (model->m != 1 || model->has_g || !B || Q || iters < 1)
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_filter_chunk: a Gamma-learned precision (carry_tau) needs m = 1, "
                                                   "a linear observation row B, no Q and iters >= 1");
    } else {
        if (!Q || (!model->has_g && !B) || filt_tau)
            return rxg::fail(ctx, RXG_ERR_BAD_ARG, "delta_filter_chunk: a known noise needs Q (and B without g); "
                                                   "filt_tau belongs to carry_tau");
        if (!host_spd(Q, model->m))
            return rxg::fail(ctx, RXG_ERR_NOT_SPD, "delta_filter_chunk: Q must be symmetric positive definite");
    }
    rxgd_params_t p;
    pack(p, model, nullptr, nullptr, P, model->has_g ? nullptr : B, Q);
    RXG_CUDA(ctx, cudaSetDevice(ctx->device));
    long long nb = batch;
    void* args[] = {&p, &T, &nb, &y, &ymask, &carry_mean, &carry_cov, &carry_tau, &iters, &filt_mean, &filt_cov,
                    &filt_tau, &status};
    return launch(ctx, model->k_filter, batch, args, flags);
}

}  // extern "C"
