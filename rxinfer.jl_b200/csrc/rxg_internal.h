// Internal declarations shared by the translation units of librxgauss (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <string>

#include "../../include/rxgauss.h"

struct rxg_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;
    // grow-only device workspace for gain tables / staging of host-pointer calls
    void* ws = nullptr;
    size_t ws_bytes = 0;
    void* stage = nullptr;
    size_t stage_bytes = 0;
    long long launches = 0;
    int sm_count = 132;
    bool gh_ready = false;
    bool gh_learn_ready = false;    // the Gauss-Hermite table of rxg_hgf_learn.cu uploaded to this device
    // optional per-kernel timing of the last fused sweep (bench.py roofline leg)
    bool profile = false;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};   // gain start, main start, main end, (spare)   // Gauss-Hermite tables uploaded to this device's constant memory
    // host-pointer calls: side streams + events of the sliced H2D | sweep | D2H pipeline
    cudaStream_t s_in = nullptr, s_out = nullptr;
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
    cudaEvent_t ev_start = nullptr;
    // host-pointer calls of a shared model: pinned copy of the [T][d][d] covariance table + its arrival event
    void* h_tab = nullptr;
    size_t h_tab_bytes = 0;
    cudaEvent_t ev_tab = nullptr;
    // side stream for work that overlaps a collective (covariance replication next to the all-gather)
    cudaStream_t s_aux = nullptr;
    cudaEvent_t ev_aux[2] = {nullptr, nullptr};
    // NCCL (dlopen'ed lazily; see rxg_api.cu)
    void* nccl_dl = nullptr;
    void* comm = nullptr;
    int nranks = 1, rank = 0;
    // options (rxg_set_option); the RXG_* environment variables are read ONCE, in rxg_create, as their initial values
    long long opt[RXG_OPT_COUNT_] = {};
    // numerical-failure flag of the chain-independent gain tables (non-SPD model): device word + pinned host mirror
    int* d_bad = nullptr;
    int* h_bad = nullptr;
    bool bad_pending = false;      // a copy d_bad -> h_bad has been enqueued and not yet examined
    // peer-mapped gather (rxg_peer_*): flags of the device-side barrier, one int per rank, in every rank's buffer
    int peer_n = 0, peer_rank = 0;
    int* peer_flags[RXG_MAX_PEERS] = {};     // peer_flags[g] = rank g's flag array as mapped here (own: cudaMalloc'ed)
    unsigned peer_epoch = 0;
    void* d_tmask = nullptr;     // device copy of a shared missing-data pattern (RXG_MASK_SHARED)
    size_t tmask_bytes = 0;
    void* d_useq = nullptr;      // device copy of a shared input sequence (RXG_U_SEQ_SHARED)
    size_t useq_bytes = 0;
    // grow-only scratch of the general-shape front end (padded operands, shifted observations)
    void* aux_buf[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t aux_bytes[4] = {0, 0, 0, 0};
    // persistent host threads of the host-side covariance broadcast
    void* fill_pool = nullptr;
    // grow-only scratch of the prediction post-pass (model copies, per-step tables, forecast buffers)
    void* pred_buf = nullptr;
    size_t pred_bytes = 0;
};

namespace rxg {

int fail(rxg_ctx* ctx, int code, const char* fmt, ...);
int check_cuda(rxg_ctx* ctx, cudaError_t e, const char* what);
// returns device pointer of >= bytes (grow-only); nullptr on failure (error recorded)
void* workspace(rxg_ctx* ctx, size_t bytes);
// host: fp64 Cholesky of the symmetrised (A + A')/2 of an n x n matrix (n <= 16), then its inverse; false if it is not
// symmetric positive definite (or not finite); log det on success
bool host_spd_inv(const float* a, int n, double* inv, double* logdet);
// rxg_hmm.cu: host checks of the HMM entries' probability arrays and Dirichlet parameters
bool stochastic_columns(const float* p, int rows, int K);
bool positive(const float* p, int n);
void* staging(rxg_ctx* ctx, size_t bytes);
// rxg_hgf.cu: the 31 Gauss-Hermite nodes and weights (physicists' convention), fp64
void gauss_hermite_31(double* t, double* w);
void* predict_scratch(rxg_ctx* ctx, size_t bytes);
// device word that gain kernels OR a 1 into when a Cholesky pivot is non-positive (cleared by begin_bad_flag)
int* bad_flag(rxg_ctx* ctx);
int begin_bad_flag(rxg_ctx* ctx);                   // zero the flag on the ctx stream
int end_bad_flag(rxg_ctx* ctx, bool sync_now);      // enqueue the read-back; if sync_now: synchronise and return RXG_ERR_NOT_SPD when set

#define RXG_CUDA(ctx, call)                                         \
    do {                                                            \
        int _rc = ::rxg::check_cuda((ctx), (call), #call);          \
        if (_rc != RXG_OK) return _rc;                              \
    } while (0)

// Extra destinations of the smoothed posteriors of a fused sweep + all-gather: pointers into the PEER ranks'
// gathered buffers (mapped into this process), already offset to this rank's slab.  n = 0: plain sweep.
struct PeerOut {
    float* mean[RXG_MAX_PEERS - 1];
    float* cov[RXG_MAX_PEERS - 1];
    int n_mean;
    int n_cov;
};

struct LgssmCall {
    int d, m, T;
    int64_t batch;
    // shared model: host pointers (row-major); per-chain model: device pointers [..][batch]
    const float *A, *B, *P, *Q, *m0, *S0;
    const float* u;          // transition offset (same pointer space as the model) or null
    // per-step inputs (RXG_U_SEQ_*; then u is null): device sequence, row t at useq + t * d * ustride (ustride = batch
    // for a per-chain sequence [rows][d][batch], 1 for a shared one [rows][d] read with batch stride 0)
    const float* useq = nullptr;
    const float* useq_host = nullptr; // the shared sequence's host copy [rows][d] (large-state trajectory, embedding)
    bool useq_chain = false;
    const float* mean0_chain = nullptr;   // device [d][batch]: per-chain prior mean (streaming carry) or null
    const float* y;          // device
    const uint8_t* ymask;    // device or null
    const uint8_t* tmask = nullptr;   // device [T] or null: missing-data pattern SHARED by all chains (RXG_MASK_SHARED)
    int n_observed = -1;              // number of observed steps of tmask (-1: all T)
    float* mean;             // device
    float* cov;              // device
    float* nle;              // device or null
    int32_t* status;         // device or null
    unsigned flags;
    bool smooth;
    bool tables_only = false;   // compute the gain tables (and the RXG_COV_SHARED_OUT covariance table) and return: no sweep
    PeerOut po = {};            // fused all-gather: peer destinations of the final mean (and covariance) stores
    bool want_cov_table = false; // in: also leave the chain-independent posterior covariance table [T][d][d] in the workspace
    float* cov_table = nullptr;  // out: that table (source of the local covariance replication), or null if the family has none
    cudaEvent_t ev_tables = nullptr;   // recorded on the ctx stream once the gain tables are complete (before the sweep)
    bool fused_peer_stores = false;    // out: the sweep kernel itself stored to c.po (else the caller pushes the slabs)
};

// rxg_hostfill.cpp (plain C++): cov[row][b] = tab[row], non-temporal stores by NUMA-pinned host threads
void host_broadcast_cov(float* cov, const float* tab, int64_t rows, int64_t batch, int nthreads);
// rxg_peer.cu
int launch_replicate_cov(rxg_ctx* ctx, cudaStream_t st, const float* src, int64_t src_stride, float* dst, int64_t rows,
                         int64_t b, int G, int skip);
int ensure_aux_stream(rxg_ctx* ctx);
int stage_shared_mask(rxg_ctx* ctx, int T, const uint8_t* host_mask, LgssmCall& c);    // rxg_api.cu
// rxg_api.cu: validate the RXG_U_SEQ_* flags and set c.u / c.useq* (`rows` rows of the sequence are staged / read)
int stage_inputs(rxg_ctx* ctx, unsigned flags, const float* u, int rows, int d, LgssmCall& c);
// rxg_lgssm_general.cu: any (d, m) in 1..64 (native families, embedding, generic per-chain kernel)
int lgssm_dispatch(rxg_ctx* ctx, LgssmCall& c);
// rxg_lgssm.cu: the register-resident families (d <= 6 shapes)
int lgssm_dispatch_native(rxg_ctx* ctx, LgssmCall& c);
// status[i] = RXG_ERR_NOT_SPD if the ctx's gain-table failure flag is set on the device, else RXG_OK
int fill_status_from_flag(rxg_ctx* ctx, int32_t* status, int64_t n);
bool lgssm_supported(int d, int m);
bool lgssm_native_small(int d, int m);    // a register-resident family shape (keeps its own [T][d][d] covariance table)
// rxg_rules_large.cu: Gaussian rule kernels for state sizes without a register-resident instantiation (d up to 64)
bool rules_small(int d);
bool rules_small2(int dout, int din);
int rules_large_add_cov(rxg_ctx* ctx, int64_t n, int d, const float* mu_in, const float* S_in, const float* Sigma, int shared,
                        float* mu_out, float* S_out);
int rules_large_pair_axpy(rxg_ctx* ctx, int64_t n, int d, const float* v1, const float* M1, const float* v2, const float* M2,
                          float sv, float* vo, float* Mo);
int rules_large_mul_out(rxg_ctx* ctx, int64_t n, int dout, int din, const float* A, const float* mu_in, const float* S_in,
                        float* mu_out, float* S_out);
int rules_large_mul_in(rxg_ctx* ctx, int64_t n, int dout, int din, const float* A, const float* mu_out, const float* S_out,
                       float* xi_in, float* W_in, int32_t* status);
int left_gemm_per_slice(rxg_ctx* ctx, int M, int K, int64_t N, const float* A, const float* X, float* Y, int64_t slices,
                        int64_t x_slice, int64_t y_slice, int accumulate);
int rules_large_convert(rxg_ctx* ctx, int64_t n, int d, int k, const float* const* v_list, const float* const* M_list,
                        float* vo, float* Mo, int32_t* status);
// rxg_predict.cu: predictive distributions of the observations after a smoothing sweep (c = the call as dispatched)
struct PredictArgs {
    int H;
    float *pred_mean, *pred_cov, *fc_mean, *fc_cov;
};
int lgssm_predict_post(rxg_ctx* ctx, const LgssmCall& c, const PredictArgs& p);
// rxg_lgssm_large.cu
int lgssm_large_dispatch(rxg_ctx* ctx, LgssmCall& c);
bool lgssm_large_supported(int d, int m);
// rxg_umma_sweep.cu (d = 16 / 32 / 64 mean recursions on the tensor cores, wgmma)
int launch_umma_sweep(rxg_ctx* ctx, int d, bool smooth, const float* recFE, const float* recG, const float* recK,
                      const float* m0, const float* m0c, const float* y, float* mean, int T, int64_t batch);

}  // namespace rxg
